// smcb_nested.cu -- the threshold step of nested sampling SMC (NestedSamplingSMC.logG, particles/nested.py:330-351)
// with no host work in between: one call selects the next likelihood level lt, updates the log-evidence, applies the
// stopping rule and writes the new log-weights; the host reads back three doubles.
//
//   lt            np.percentile(llik, 100 (1 - ESSrmin)), bit for bit.  The host gives NumPy's "linear" rule as the
//                 order statistics k0 <= k1 and the weight gamma; the device selects statistic k0 by a radix select
//                 over order-preserving 64-bit keys (6 passes of 11 bits, no sort), statistic k1 is the same value
//                 or the smallest value above it (one more pass), and the two are combined as numpy's _lerp does.
//   evidence      lZt = t log(ESSrmin) - log(n) + LSE(llik[llik <= lt]) and the same with every entry, both by ONE
//                 fixed-order reduction in which an excluded entry enters as -inf: when no entry is above lt the two
//                 sums are the same bits, so the stopping rule |new_evid - new_evid_final| < eps fires, as it does in
//                 the reference (this is also the only case in which no particle survives the cut).
//   lw            0 where llik > lt, -inf elsewhere; all zeros when the run stops (lt = inf).
//
// Every reduction is deterministic: integer counts and integer min / max are order-free, and the floating-point
// sums run grid-stride over a grid that depends on n only, then over the warps and the blocks in a fixed order.
#include "smcb_common.cuh"
#include "smcb_reduce.cuh"

using namespace smcb;

namespace smcb {

constexpr int kNsBlock = 256;
constexpr int kNsDigit = 11;                     // bits per radix pass: 6 passes cover the 64-bit key
constexpr int kNsBins = 1 << kNsDigit;
constexpr int kNsPasses = (64 + kNsDigit - 1) / kNsDigit;
constexpr int kNsBinsPerThread = kNsBins / kNsBlock;

// device-resident state of one call (in the context's workspace)
struct NsState {
    unsigned long long prefix;       // key bits of statistic k0 chosen so far
    unsigned long long rank;         // rank of statistic k0 among the keys that share the prefix
    unsigned long long less;         // keys below the prefix's bucket
    unsigned long long eq;           // keys in the prefix's bucket (after the last pass: equal to statistic k0)
    unsigned long long next_key;     // smallest key above statistic k0 (~0 if none)
    unsigned long long max_key;      // largest key
    unsigned long long cut_key;      // largest key whose value is <= lt (0 if none)
    double lt;
};

// order-preserving map double -> uint64 (llik holds no NaN).  -0.0 sorts just below +0.0: the selected statistic keeps
// the sign of its zero, so a level at a zero has NumPy's bits unless llik holds both -0.0 and +0.0 (which of the two
// NumPy's partition puts at a given index is then unspecified; the value is the same)
__device__ __forceinline__ unsigned long long ns_key(double x) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ double ns_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// one radix-select pass: the histogram of the digit at `shift` over the keys whose bits above the digit equal the
// prefix's; the last block finds the bucket of rank st->rank, extends the prefix and clears the histogram.
// prefix and rank are read once, at the start: every block reads them before the last block (the one that has seen
// every other block's ticket) rewrites them, and within the last block no thread reads them after the write.
__global__ void __launch_bounds__(kNsBlock) k_ns_select_pass(const double *__restrict__ llik, int64_t n, int shift,
                                                            unsigned long long hi_mask, NsState *st,
                                                            unsigned int *hist, unsigned int *ticket) {
    __shared__ unsigned int s_hist[kNsBins];
    __shared__ unsigned long long s_part[kNsBlock];
    for (int b = threadIdx.x; b < kNsBins; b += kNsBlock) s_hist[b] = 0u;
    const unsigned long long prefix = st->prefix, rank = st->rank;
    __syncthreads();
    // log-likelihoods share their sign and top exponent bits, so most keys of a warp fall into the same bin: the lanes
    // with equal bins add their count with one shared atomic (the whole warp steps through the loop together)
    const int lane = threadIdx.x & 31;
    for (int64_t base = (int64_t)blockIdx.x * kNsBlock + (threadIdx.x & ~31); base < n;
         base += (int64_t)gridDim.x * kNsBlock) {
        const int64_t i = base + lane;
        unsigned int bin = kNsBins;                                      // no bin: past n, or another prefix
        if (i < n) {
            const unsigned long long k = ns_key(llik[i]);
            if (((k ^ prefix) & hi_mask) == 0ull) bin = (unsigned int)((k >> shift) & (kNsBins - 1));
        }
        const unsigned int peers = __match_any_sync(0xffffffffu, bin);
        if (bin != kNsBins && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], (unsigned int)__popc(peers));
    }
    __syncthreads();
    for (int b = threadIdx.x; b < kNsBins; b += kNsBlock)
        if (s_hist[b]) atomicAdd(&hist[b], s_hist[b]);
    if (!last_block(ticket)) return;
    // each thread owns kNsBinsPerThread consecutive bins; a serial scan over the threads' sums finds the owner
    unsigned long long own = 0ull;
    unsigned int cnt[kNsBinsPerThread];
#pragma unroll
    for (int j = 0; j < kNsBinsPerThread; j++) {
        cnt[j] = reinterpret_cast<volatile unsigned int *>(hist)[threadIdx.x * kNsBinsPerThread + j];
        own += cnt[j];
    }
    s_part[threadIdx.x] = own;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long acc = 0ull;
        for (int t = 0; t < kNsBlock; t++) { const unsigned long long v = s_part[t]; s_part[t] = acc; acc += v; }
    }
    __syncthreads();
    const unsigned long long before = s_part[threadIdx.x];
    if (rank >= before && rank < before + own) {
        unsigned long long acc = before;
        for (int j = 0; j < kNsBinsPerThread; j++) {
            if (rank < acc + cnt[j]) {
                st->prefix = prefix | ((unsigned long long)(threadIdx.x * kNsBinsPerThread + j) << shift);
                st->rank = rank - acc;
                st->less += acc;
                st->eq = cnt[j];
                break;
            }
            acc += cnt[j];
        }
    }
#pragma unroll
    for (int j = 0; j < kNsBinsPerThread; j++) hist[threadIdx.x * kNsBinsPerThread + j] = 0u;
}

// the smallest key above statistic k0 and the largest key; the last block forms lt (numpy's _lerp, nested.py:332)
__global__ void __launch_bounds__(kNsBlock) k_ns_level(const double *__restrict__ llik, int64_t n, int64_t k1,
                                                      double gamma, NsState *st, unsigned int *ticket) {
    const unsigned long long a_key = st->prefix;
    unsigned long long nx = ~0ull, mx = 0ull;
    for (int64_t i = (int64_t)blockIdx.x * kNsBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kNsBlock) {
        const unsigned long long k = ns_key(llik[i]);
        if (k > a_key && k < nx) nx = k;
        if (k > mx) mx = k;
    }
    nx = warp_min(nx);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) {
        if (nx != ~0ull) atomicMin(&st->next_key, nx);
        atomicMax(&st->max_key, mx);
    }
    if (!last_block(ticket) || threadIdx.x != 0) return;
    const double a = ns_value(a_key);
    const unsigned long long nk = reinterpret_cast<volatile NsState *>(st)->next_key;
    // statistic k1 is statistic k0 while k1 falls inside k0's block of ties
    const double b = ((unsigned long long)k1 < st->less + st->eq || nk == ~0ull) ? a : ns_value(nk);
    const double diff = b - a;                     // numpy _lerp: a + diff g, or b - diff (1 - g) where g >= 0.5
    st->lt = (gamma >= 0.5) ? b - diff * (1.0 - gamma) : a + diff * gamma;
}

// the largest key whose value is <= lt: the shift of the log-sum-exp over llik[llik <= lt]
__global__ void __launch_bounds__(kNsBlock) k_ns_cut_max(const double *__restrict__ llik, int64_t n, NsState *st) {
    const double lt = st->lt;
    unsigned long long mx = 0ull;
    for (int64_t i = (int64_t)blockIdx.x * kNsBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kNsBlock) {
        const double v = llik[i];
        if (v <= lt) { const unsigned long long k = ns_key(v); mx = k > mx ? k : mx; }
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(&st->cut_key, mx);
}

// scipy.special.logsumexp's shift: the maximum, or 0 when it is not finite
__device__ __forceinline__ double ns_shift(unsigned long long key) {
    const double m = key ? ns_value(key) : -CUDART_INF;
    return isfinite(m) ? m : 0.0;
}

__device__ __forceinline__ double log_sum_exp_ab(double a, double b) {      // resampling.py:273-288
    return (a > b) ? a + log1p(exp(b - a)) : b + log1p(exp(a - b));
}

// sum exp(llik - m_cut) over llik <= lt and sum exp(llik - m_all) over all of llik, by one reduction tree; the last
// block forms the two evidence estimates, applies the stopping rule and writes (lt, new_evid, stop)
__global__ void __launch_bounds__(kNsBlock) k_ns_evidence(const double *__restrict__ llik, int64_t n, int t,
                                                         double log_alpha, double log_evid, double eps, NsState *st,
                                                         double *partials, unsigned int *ticket, double *out) {
    __shared__ double s_red[2][kNsBlock / 32];
    const double lt = st->lt, mc = ns_shift(st->cut_key), ma = ns_shift(st->max_key);
    double sc = 0.0, sa = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kNsBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kNsBlock) {
        const double v = llik[i];
        sc += exp(((v <= lt) ? v : -CUDART_INF) - mc);
        sa += exp(v - ma);
    }
    sc = warp_sum(sc);
    sa = warp_sum(sa);
    if ((threadIdx.x & 31) == 0) { s_red[0][threadIdx.x >> 5] = sc; s_red[1][threadIdx.x >> 5] = sa; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double c = 0.0, a = 0.0;
        for (int w = 0; w < kNsBlock / 32; w++) { c += s_red[0][w]; a += s_red[1][w]; }
        partials[2 * blockIdx.x] = c;
        partials[2 * blockIdx.x + 1] = a;
    }
    if (!last_block(ticket) || threadIdx.x != 0) return;
    double c = 0.0, a = 0.0;
    for (unsigned int b = 0; b < gridDim.x; b++) {
        c += reinterpret_cast<volatile double *>(partials)[2 * b];
        a += reinterpret_cast<volatile double *>(partials)[2 * b + 1];
    }
    const double base = (double)t * log_alpha - log((double)n);
    const double lzt = base + (log(c) + mc), lzt_final = base + (log(a) + ma);
    const double new_evid = log_sum_exp_ab(log_evid, lzt), new_evid_final = log_sum_exp_ab(log_evid, lzt_final);
    const bool stop = fabs(new_evid - new_evid_final) < eps;
    if (stop) st->lt = CUDART_INF;
    out[0] = stop ? CUDART_INF : lt;
    out[1] = stop ? new_evid_final : new_evid;
    out[2] = stop ? 1.0 : 0.0;
}

__global__ void __launch_bounds__(kNsBlock) k_ns_weights(const double *__restrict__ llik, int64_t n,
                                                        const NsState *st, double *__restrict__ lw) {
    const double lt = st->lt;            // inf after a stop: every weight is 0
    for (int64_t i = (int64_t)blockIdx.x * kNsBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kNsBlock)
        lw[i] = (lt == CUDART_INF || llik[i] > lt) ? 0.0 : -CUDART_INF;
}

}  // namespace smcb

// NestedSamplingSMC.logG (nested.py:330-351) on the device: see the top of this file and include/smcb.h
extern "C" int smcb_ns_threshold(smcb_ctx *c, const double *llik, int64_t n, int64_t k0, int64_t k1, double gamma,
                                 int t, double log_alpha, double log_evid, double eps, double *lw, double *out) {
    SMCB_REQUIRE(c && llik && lw && out, "smcb_ns_threshold: NULL argument");
    SMCB_REQUIRE(n >= 1 && n <= (int64_t)UINT32_MAX, "smcb_ns_threshold: n = %lld outside [1, 2^32)", (long long)n);
    SMCB_REQUIRE(k0 >= 0 && k0 < n && k1 >= k0 && k1 <= k0 + 1 && k1 < n,
                 "smcb_ns_threshold: order statistics k0 = %lld, k1 = %lld outside [0, %lld)", (long long)k0,
                 (long long)k1, (long long)n);
    SMCB_REQUIRE(gamma >= 0.0 && gamma <= (double)n, "smcb_ns_threshold: gamma must be in [0, n]");
    // workspace: state | block partials (2 per block) | histogram
    NsState *st = reinterpret_cast<NsState *>(c->ws);
    double *partials = c->ws + 64;
    unsigned int *hist = reinterpret_cast<unsigned int *>(c->ws + 64 + 2 * kMaxGrid);
    const NsState init = {0ull, (unsigned long long)k0, 0ull, 0ull, ~0ull, 0ull, 0ull, 0.0};
    SMCB_CUDA(cudaMemcpyAsync(st, &init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    SMCB_CUDA(cudaMemsetAsync(hist, 0, kNsBins * sizeof(unsigned int), c->stream));
    const int grid = grid_for(n, kNsBlock * 4);
    for (int p = 0; p < kNsPasses; p++) {
        const int top = 64 - p * kNsDigit;                               // the digit is bits [shift, top)
        const int shift = top > kNsDigit ? top - kNsDigit : 0;
        const unsigned long long hi_mask = (top == 64) ? 0ull : (~0ull << top);
        SMCB_TRY(launch(c, k_ns_select_pass, grid, kNsBlock, 0, llik, n, shift, hi_mask, st, hist,
                        c->counters + kTicketNsSelect));
    }
    SMCB_TRY(launch(c, k_ns_level, grid, kNsBlock, 0, llik, n, k1, gamma, st, c->counters + kTicketNsLevel));
    SMCB_TRY(launch(c, k_ns_cut_max, grid, kNsBlock, 0, llik, n, st));
    SMCB_TRY(launch(c, k_ns_evidence, grid, kNsBlock, 0, llik, n, t, log_alpha, log_evid, eps, st, partials,
                    c->counters + kTicketNsEvidence, out));
    return launch(c, k_ns_weights, grid, kNsBlock, 0, llik, n, st, lw);
}
