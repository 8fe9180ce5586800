// smcb_search.cuh -- inverse-CDF search (particles/resampling.py:484-509).
//   A[k] = min{ j : cdf[j] >= su[k] }   == np.searchsorted(cdf, su, side='left'),
// clipped to n-1 (the numba loop of the reference has no bounds check).
#pragma once
#ifndef SMCB_MATH_HOST_TEST      // tests/math_host.cpp compiles tile_search for the CPU with its own shim
#include "smcb_common.cuh"
#endif

namespace smcb {

// The search inside a staged CDF tile (the step kernel's multinomial and global-resampling move passes).  s holds
// cdf[sbase, sbase + cnt); the answers of the tile's outputs are known to lie at or after s[l0] (l0 = lo - sbase).
// r0, r1 = the first j in [l0, cnt) with s[j] >= v0, v1 (cnt if none) for one output pair, v0 <= v1.
// v1 lies on average one CDF entry past v0: it walks forward a few entries before it falls back to bisection
// (same result as searchsorted).
__device__ __forceinline__ void tile_search(const double *s, int l0, int cnt, double v0, double v1, int &r0, int &r1) {
    int h0 = cnt;
    while (l0 < h0) { const int mid = (l0 + h0) >> 1; if (s[mid] < v0) l0 = mid + 1; else h0 = mid; }
    int l1 = l0, h1 = cnt;
#pragma unroll
    for (int w = 0; w < 4; w++)
        if (l1 < cnt && s[l1] < v1) l1++;
    if (l1 < cnt && s[l1] < v1) {
        while (l1 < h1) { const int mid = (l1 + h1) >> 1; if (s[mid] < v1) l1 = mid + 1; else h1 = mid; }
    }
    r0 = l0;
    r1 = l1;
}

#ifndef SMCB_MATH_HOST_TEST

// first j in [lo, hi) with cdf[j] >= key, hi if none; cdf non-decreasing
__device__ __forceinline__ int64_t lower_bound(const double *__restrict__ cdf, int64_t lo,
                                               int64_t hi, double key) {
    while (lo < hi) {
        int64_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(cdf + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// same with L2 loads: for a cdf other CTAs wrote earlier in the SAME kernel (the non-coherent path of
// __ldg may serve a stale line)
__device__ __forceinline__ int64_t lower_bound_cg(const double *cdf, int64_t lo, int64_t hi, double key) {
    while (lo < hi) {
        int64_t mid = lo + ((hi - lo) >> 1);
        if (__ldcg(cdf + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Block-cooperative lower_bound over [lo, hi): BLOCK-ary search, each round costs one
// (parallel) probe per thread and one __syncthreads_count -> ceil(log_BLOCK(hi-lo))
// dependent memory round trips instead of log2.  All threads get the result.
template <int BLOCK>
__device__ __forceinline__ int64_t block_lower_bound(const double *__restrict__ cdf, int64_t lo,
                                                     int64_t hi, double key) {
    while (hi - lo > 0) {
        const int64_t span = hi - lo;
        const int64_t step = (span + BLOCK - 1) / BLOCK;          // >= 1
        const int64_t pos = lo + ((int64_t)threadIdx.x + 1) * step - 1;  // last index of my slice
        int pred = 0;
        if (pos < hi) pred = (__ldcg(cdf + pos) < key);
        // monotone cdf => the set of threads with pred == 1 is a prefix of the block
        const int cnt = __syncthreads_count(pred);
        const int64_t nlo = lo + (int64_t)cnt * step;              // all slices before are < key
        if (nlo >= hi) return hi;
        lo = nlo;
        hi = (lo + step - 1 < hi) ? lo + step - 1 : hi;           // slice `cnt`: its last element is >= key
        if (step == 1) return lo;
    }
    return lo;
}

#endif

}  // namespace smcb
