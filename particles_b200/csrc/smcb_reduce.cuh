// smcb_reduce.cuh -- warp reductions and grid-wide deterministic reduction ("last block done").
#pragma once
#include <type_traits>

#include "smcb_common.cuh"

namespace smcb {

// xor butterfly over the 32 lanes, strides 16 -> 1: every lane gets the same bits
template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(kFull, v, m);
    return v;
}
template <class T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) { const T o = __shfl_xor_sync(kFull, v, m); v = o > v ? o : v; }
    return v;
}
// integers only: no kernel takes an fp64 minimum, so none is defined (and none falls back to this NaN-blind form)
template <class T>
__device__ __forceinline__ T warp_min(T v) {
    static_assert(std::is_integral<T>::value, "warp_min: integer types only");
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) { const T o = __shfl_xor_sync(kFull, v, m); v = o < v ? o : v; }
    return v;
}
// fp64 through fmax: a NaN lane gives way to a number
template <>
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, m));
    return v;
}

// Slots of smcb_ctx::counters, the tickets of last_block.  A launch leaves its slot at 0, so kernels that run one
// after the other on the context's stream may share one.
enum TicketSlot : int {
    kTicketLse = 0,             // k_lse, k_max_sum (smcb_api.cu)
    kTicketWmoments = 1,        // k_wmoments
    kTicketMhAccept = 2,        // k_mh_accept (smcb_sampler.cu)
    kTicketCtlMax = 8,          // k_ctl_max
    kTicketCtlRoot = 9,         // k_ctl_root_pass
    kTicketCtlWcov0 = 10,       // k_ctl_wcov, pass 0
    kTicketCtlWcov1 = 11,       // k_ctl_wcov, pass 1
    kTicketNsSelect = 12,       // k_ns_select_pass (smcb_nested.cu)
    kTicketNsLevel = 13,        // k_ns_level
    kTicketNsEvidence = 14,     // k_ns_evidence
    kTicketSlotsUsed
};
constexpr int kTicketSlots = 64;   // counters smcb_create allocates
static_assert(kTicketSlotsUsed <= kTicketSlots, "ticket slots exceed smcb_ctx::counters");

// Called by every thread of every block after the block has written its partials; true in every thread of the one
// block that draws the grid's last ticket, where all other blocks' partials are then visible.  The ticket counter
// wraps back to 0 (atomicInc modulo gridDim.x), so it never needs a memset between launches.
__device__ __forceinline__ bool last_block(unsigned int *ticket) {
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicInc(ticket, gridDim.x - 1) == gridDim.x - 1;
    __syncthreads();
    if (last) __threadfence();
    return last;
}

// Every block deposits K partial triples; the block that draws the last ticket merges
// all partials in a FIXED order (so the result does not depend on block scheduling)
// and returns true with the totals valid in thread 0.
template <int BLOCK, int K>
__device__ __forceinline__ bool grid_merge_lse3(Lse3 (&mine)[K], double *partials /* grid x 4K */,
                                                unsigned int *ticket, Lse3 *smem,
                                                Lse3 (&total)[K]) {
#pragma unroll
    for (int j = 0; j < K; j++) mine[j] = lse3_block_reduce<BLOCK>(mine[j], smem);
    if (threadIdx.x == 0) {
        double *p = partials + (size_t)blockIdx.x * 4 * K;
#pragma unroll
        for (int j = 0; j < K; j++) {
            p[4 * j + 0] = mine[j].m; p[4 * j + 1] = mine[j].s; p[4 * j + 2] = mine[j].q;
        }
    }
    if (!last_block(ticket)) return false;
#pragma unroll
    for (int j = 0; j < K; j++) {
        Lse3 acc = lse3_empty();
        for (int k = threadIdx.x; k < (int)gridDim.x; k += BLOCK) {
            const volatile double *p = partials + (size_t)k * 4 * K + 4 * j;
            acc = lse3_merge(acc, Lse3{p[0], p[1], p[2]});
        }
        total[j] = lse3_block_reduce<BLOCK>(acc, smem);
    }
    return true;
}

// Weights.__init__ scalars from the merged triple (resampling.py:217-226):
//   log_mean = m + log(s / N);  ESS = 1 / sum (w/s)^2 = s^2 / q
// All -inf (m == -inf) or any +inf (m == +inf) give NaN everywhere, as NumPy does.
__device__ __forceinline__ void weights_scalars(const Lse3 &a, double n, double &log_mean,
                                                double &ess) {
    if (a.m == -CUDART_INF || a.m == CUDART_INF || a.m != a.m) {
        log_mean = CUDART_NAN;
        ess = CUDART_NAN;
        return;
    }
    log_mean = a.m + log(a.s / n);
    ess = (a.s * a.s) / a.q;
}

}  // namespace smcb
