// smcb_batch.cuh -- what the batched filters (smcb_batch.cu) and the filter bank (smcb_bank.cu) share: the CTA size,
// the padded row length, the resident tier's shared-memory budget and the plain-load CDF helpers.
#pragma once
#include "smcb_step.cuh"

namespace smcb {

constexpr int kBatchBS = 256;

// plain loads (shared or device memory written earlier by this CTA): the multinomial spacings
struct LoadPlain {
    const double *v;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&o)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) o[j] = (i0 + j < n) ? v[i0 + j] : 0.0;
    }
};

// np.searchsorted(cdf, key, 'left') on [0, n) with plain loads
__device__ __forceinline__ int64_t lower_bound_plain(const double *cdf, int64_t n, double key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (cdf[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__host__ __device__ inline int64_t batch_ld(int64_t n) { return (n + 1) & ~(int64_t)1; }

// doubles of shared memory the resident tier needs besides the math tables
__host__ __device__ inline int64_t resident_doubles(int64_t n, int scheme) {
    const int64_t ld = batch_ld(n);
    return 4 * ld + (scheme == SMCB_RS_MULTINOMIAL ? ld + 2 : 0);
}

}  // namespace smcb
