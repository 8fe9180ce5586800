#pragma once
// smcb_step.cuh -- the fused SMC step (particles/core.py:369-383): ONE kernel launch per step.
//
//   k_step(t), every CTA:
//     prologue   merge the per-CTA partials (max, sum exp, sum exp^2 [, sum w x, sum w x^2]) that step
//                t-1 left behind -- every CTA does it redundantly, in the same fixed order, so all of
//                them hold identical bits -- [sharded: exchange the shard totals through the NVLink
//                mailboxes], then compute_summaries of step t-1 (core.py:351-367) and the ESS test of
//                step t (core.py:181-183).  CTA 0 records the (T, 4) summary row, the moments row and the
//                state S_{t-1}.  No "last CTA" serial tail, no separate finish kernel.
//     no resampling:  xp = X_k -> x' ~ M_t(xp) -> lw' = lw + logG -> partials            32 B/particle
//     resampling:     W_i = exp(lw_i - m)/s -> CDF of the CTA's own range (16 B/particle)
//                     -> grid barrier -> su_k -> A_k = search(cdf) -> xp = X[A_k] -> x' -> lw' = logG
//                     -> partials                                                         40 B/particle
//     fused pair (1-D, one device): a streaming step t whose successor is predicted not to resample also runs
//                     step t+1 while the particle sits in registers: x_{t-1}, lw_{t-1} in once, x_t, lw_t out to
//                     buffers t & 1, x_{t+1}, lw_{t+1} out to buffers (t+1) & 1 in place       24 B/particle/step
//                     Launch t+1 then only runs its prologue; if that says "resample", it overwrites the
//                     speculative step t+1 from the intact buffers t & 1.
//   k_tail(t)  (one CTA, once per enqueued batch): the prologue alone, so that the summaries of the last
//              enqueued step exist before the host reads them.  Idempotent with the next k_step.
//
// The step index is a kernel argument (the host mirrors it); everything else a step needs from its
// predecessor is in the partials (four rows per CTA, indexed by step mod 4: a fused launch reads those of t-1 and
// writes those of t and t+1) and in S_{t-2}.
#include <string.h>

#include <new>
#include <type_traits>

#include "smcb_common.cuh"
#include "smcb_dispatch.cuh"
#include "smcb_math.cuh"
#include "smcb_models.cuh"
#include "smcb_scan.cuh"
#include "smcb_search.cuh"

using namespace smcb;

namespace smcb {

constexpr int kPartStride = 16;     // doubles per CTA partial row: w(m,s,q,-) aux(m,s,q,-) sx[4] sxx[4]
constexpr int kMailStride = 32;     // doubles per mailbox slot: the 16 above, then epochs
constexpr int kMailEpoch = 16;      // slot[16] = t + 1 once the sender's statistics of step t are complete
constexpr int kMailScan = 17;       // slot[17] = t + 1 once the sender's CDF of (resampling) step t is complete
constexpr int kMaxStepGrid = 256;   // CTAs of the step kernel: ONE per SM (132 on an H100), each owning a contiguous range
constexpr int kMaxD = 4;
constexpr int kTailBlock = 256;     // threads of the one-CTA helper kernels (>= kMaxStepGrid: one partial row per thread)
constexpr int kPartSlots = 4;       // partial rows per CTA: step s uses row s % 4
#ifndef SMCB_SPECULATE
#define SMCB_SPECULATE 1         // sharded filters: start the streaming pass before the peers' statistics arrive
#endif
template <class M> struct StepCfg {
    // threads per CTA of the step kernel.  One CTA per SM: the warp scheduler favours the oldest CTA / warps (with 3
    // equal CTAs per SM the first retires long before the last, the SM running few warps for the final stretch), so
    // all warps of an SM live in one CTA.  16 warps at up to 128 registers beat 24 warps at 80 (which spill once the
    // prefetch is on).
    static constexpr int BS = 512;
    static constexpr int kU = (M::D == 1) ? 2 : 1;    // pairs in flight per thread in the streaming branch (d-dimensional
                                                      // states: one -- registers, and a finer work unit for the N = 1e6
                                                      // runs they are used at)
    static constexpr int kStage = 8 * BS;             // doubles of CDF staged per output tile (2 BS outputs)
    // dynamic shared memory: the math tables (smcb_tables.h, 64 KB), then two CDF slices (resampling branch) which
    // the streaming branch reuses for its slab records
    static constexpr int kSlabRecords = 128;          // slab records (768 B each): the 96 KB of the CDF staging buffers
    static constexpr int kSlabDoubles = kSlabRecords * 96;   // per-lane slab records of the streaming branch
    static constexpr size_t dyn_smem = kMathTabBytes + (size_t)(2 * kStage > kSlabDoubles ? 2 * kStage : kSlabDoubles) * sizeof(double);
};
constexpr int kScanGroupWarps = 2;  // warps per pipeline group of the resampling scan (scan_scatter_groups)
constexpr int kMovePairs = 2;       // resampling move pass: pairs in flight per thread

// S_t: what is known once step t is finalised; st[t & 1]
struct StepState {
    double logLt, log_mean_w, ess;
    double wm, ws, wq;      // (max, sum exp, sum exp^2) of the inferential weights over ALL particles
    long long t;            // the step this record belongs to
    long long nrs;          // resampling steps among steps 1..t   (grid-barrier epochs)
    int rs;                 // step t resampled
    int rs_next;            // decision for step t + 1
    int pad[2];
};

struct FilterArgs {
    double *X[2];
    double *lw[2];
    long long *A;
    double *cdf;
    double *su;              // multinomial: z = cumsum(-log u), (n + 1)
    const double *data;      // (T, dy)
    const double *sc;        // (T) per-step model constants or NULL
    double *summaries;       // (T, 4)
    double *moments;         // NULL or (T, 2 D): weighted mean and variance per component (collectors.Moments)
    const double *z_in, *u_in;
    StepState *st;           // [2]
    int *sync_timeout;       // a bounded wait expired (diagnostic; results are then invalid)
    double *partials;        // [kPartSlots][kMaxStepGrid][kPartStride]
    // fused pairs of streaming steps (1-D, single device)
    int fuse_mode;           // 0 off, 1 on with the predictor, 2 fuse whenever allowed (SMCB_FUSE)
    int64_t batch_end;       // first step the host has not enqueued yet: step t+1 is only fused below it
    long long *fuse;         // [0] the step the previous launch pre-computed; [1..3] fused pairs, no-op launches,
                             // mispredicted launches (pre-computed step that resampled after all)
    double *fuse_slab;       // grid x StepCfg::kSlabDoubles: the slab records of the second step of a pair
    unsigned long long *bar; // grid-barrier arrivals, never reset
    double *blk_agg;         // multinomial: per-CTA sums of the exponential spacings (grid + 1)
    const double *math_tab;  // smcb_tables.h, built at context creation
    int slab_it;             // iterations per slab of the streaming branch (host: chosen so the records fit)
    int slab_small;          // trailing iterations of a CTA's range handed out as single-iteration slabs
    int slab_lane;           // 1: a slab record holds the 32 lanes' own (m, s, q) (96 doubles); 0: their warp reduction
    int slab_stride;         // doubles per slab record: 4 (+ 4 auxiliary) (+ 2 D moments)
    int64_t n, n_global, index_offset, T;
    int dy;
    int world, rank;
    int grid;
    int64_t chunk;           // pairs of particles per CTA (contiguous ranges)
    double essrmin;
    Philox key;
    // sharded filters: host-driven exchange (NCCL all-gather of local_stats into gathered) ...
    double *local_stats;     // this rank's 16 statistics
    const double *gathered;  // world x 16, rank-major
    // ... or the peer mailboxes: [parity][sender][kMailStride]; mail_peer[p] = rank p's mailbox mapped here
    double *mail_local;
    double *mail_peer[8];
    // exact global resampling: peers' particles and CDFs mapped over NVLink
    int rs_global;
    const double *pX[8][2];
    const double *pcdf[8];
};

__device__ __forceinline__ void wait_epoch(const volatile double *flag, double epoch, int *timeout) {
    const long long t0 = clock64();
    if (*reinterpret_cast<volatile int *>(timeout)) return;   // already broken: do not stall again
    while (*flag < epoch) {
        if (clock64() - t0 > 8000000000ll) { *timeout = 1; break; }    // ~4 s at 2 GHz
    }
    __threadfence_system();
}

__device__ __forceinline__ StepK step_consts(const FilterArgs &a, long long t) {
    StepK k;
    k.t = t;
#pragma unroll
    for (int i = 0; i < kMaxDy; i++) {
        k.yv[i] = (i < a.dy && t >= 0) ? a.data[t * a.dy + i] : 0.0;
        k.yn[i] = (i < a.dy && t + 1 < a.T) ? a.data[(t + 1) * a.dy + i] : 0.0;
    }
    k.y = k.yv[0];
    k.y_next = k.yn[0];
    k.sc0 = (a.sc && t >= 0) ? a.sc[t] : 0.0;
    return k;
}

__device__ __forceinline__ double fix_nan(double v) { return v != v ? -CUDART_INF : v; }  // resampling.py:220

// Weights.__init__ scalars from the merged triple (resampling.py:217-226):
//   log_mean = m + log(s / N);  ESS = 1 / sum (w/s)^2 = s^2 / q
// All -inf (m == -inf) or any +inf (m == +inf) give NaN everywhere, as NumPy does.
__device__ __forceinline__ void weights_scalars(const Lse3 &a, double n, double &log_mean, double &ess) {
    if (a.m == -CUDART_INF || a.m == CUDART_INF || a.m != a.m) {
        log_mean = CUDART_NAN;
        ess = CUDART_NAN;
        return;
    }
    log_mean = a.m + log(a.s / n);
    ess = (a.s * a.s) / a.q;
}

// exp(m - M) for m <= M, 0 for an empty accumulator; NaN when both are +inf (NumPy's inf - inf)
__device__ __forceinline__ double shift_factor(double m, double M) {
    return (m == -CUDART_INF) ? 0.0 : fexp_neg(m - M);
}

// ---------------------------------------------------------------------------
// block-wide fixed-order reductions; every thread receives the result.  Two levels: butterfly inside each warp,
// then warp 0 reduces the per-warp values (lane = warp index) and parks the totals in shared memory -- never
// "every thread walks all warps' values" (with 24 warps that was 7 us of shared-memory traffic per call).
// smem: (BS/32 + 1) x NV doubles.
// ---------------------------------------------------------------------------
__device__ __forceinline__ double nanmax(double a, double b) { return (b > a || b != b) ? b : a; }   // NaN wins

template <int NV, int BS, bool MAX>
__device__ __forceinline__ void block_reduce_all(double (&v)[NV], double *smem) {
    constexpr int NWARP = BS / 32;
    static_assert(NWARP <= 32, "one lane per warp in the second level");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < NV; j++) {
#pragma unroll
        for (int mask = 16; mask > 0; mask >>= 1) {
            const double o = __shfl_xor_sync(0xffffffffu, v[j], mask);
            v[j] = MAX ? nanmax(v[j], o) : v[j] + o;
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < NV; j++) smem[warp * NV + j] = v[j];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int j = 0; j < NV; j++) {
            double x = (lane < NWARP) ? smem[lane * NV + j] : (MAX ? -CUDART_INF : 0.0);
#pragma unroll
            for (int mask = 16; mask > 0; mask >>= 1) {
                const double o = __shfl_xor_sync(0xffffffffu, x, mask);
                x = MAX ? nanmax(x, o) : x + o;
            }
            if (lane == 0) smem[NWARP * NV + j] = x;
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NV; j++) v[j] = smem[NWARP * NV + j];
    __syncthreads();
}
template <int NV, int BS>
__device__ __forceinline__ void block_max_all(double (&v)[NV], double *smem) { block_reduce_all<NV, BS, true>(v, smem); }
template <int NV, int BS>
__device__ __forceinline__ void block_sum_all(double (&v)[NV], double *smem) { block_reduce_all<NV, BS, false>(v, smem); }

// ---------------------------------------------------------------------------
// per-thread accumulators: (max, sum exp, sum exp^2) of the log-weights with ONE exp per value (the
// running shift only moves when a batch maximum exceeds it) and, optionally, sum w x / sum w x^2 per
// component for collectors.Moments (resampling.py:320-338) relative to the same shift.
// Values equal to -inf (masked slots) contribute exactly 0.
// ---------------------------------------------------------------------------
template <int D>
struct Acc {
    Lse3 w;
    double sx[D], sxx[D];
};

template <int D>
__device__ __forceinline__ void acc_init(Acc<D> &a) {
    a.w = lse3_empty();
#pragma unroll
    for (int c = 0; c < D; c++) { a.sx[c] = 0.0; a.sxx[c] = 0.0; }
}

// FINITE: the caller has checked that no value is +-inf / NaN (integer test, nonfinite()): the exponentials then
// need no range select (texp_sat), the maxima no NaN handling, and no slot is masked.  MOM is a template
// parameter so that the moment arithmetic is absent (not predicated off) when nobody collects moments.
template <int NV, int D, bool FINITE, bool MOM>
__device__ __forceinline__ void acc_add_batch_t(Acc<D> &a, const double (&v)[NV], const double (&x)[NV][D]) {
    double mb = v[0];
#pragma unroll
    for (int j = 1; j < NV; j++) mb = FINITE ? (v[j] > mb ? v[j] : mb) : fmax(mb, v[j]);
    if (mb > a.w.m) {                       // also the first time (m = -inf): exp(-inf) = 0
        const double r = texp_neg(a.w.m - mb);
        a.w.s *= r;
        a.w.q *= r * r;
        if (MOM) {
#pragma unroll
            for (int c = 0; c < D; c++) { a.sx[c] *= r; a.sxx[c] *= r; }
        }
        a.w.m = mb;
    }
    if (!FINITE && a.w.m == -CUDART_INF) return;       // nothing but -inf so far
#pragma unroll
    for (int j = 0; j < NV; j++) {
        const double e = FINITE ? texp_sat(v[j] - a.w.m) : texp_neg(v[j] - a.w.m);
        a.w.s += e;
        a.w.q = fma(e, e, a.w.q);
        if (MOM && (FINITE || v[j] != -CUDART_INF)) {
#pragma unroll
            for (int c = 0; c < D; c++) {
                const double ex = e * x[j][c];
                a.sx[c] += ex;
                a.sxx[c] = fma(ex, x[j][c], a.sxx[c]);
            }
        }
    }
}
template <int NV, int D, bool FINITE = false>
__device__ __forceinline__ void acc_add_batch(Acc<D> &a, const double (&v)[NV], const double (&x)[NV][D], bool mom) {
    if (mom) acc_add_batch_t<NV, D, FINITE, true>(a, v, x);
    else acc_add_batch_t<NV, D, FINITE, false>(a, v, x);
}

struct StepSmem {
    double red[32 * 16];
    int next;                 // next slab of the streaming branch
    // pipelined scan (scan_scatter_groups): prefix ring, per-group warp totals / prefixes / heavy-entry queues
    double ringP[32];
    int ringF[32];
    double gwarp[16][8];
    double gpref[16][2];
    int gqn[16];
    long long gq[16][8][3];
    int *timeout_ptr;
    double peer[8][kMailStride];
    double goff[9], gpi[8];
    double pref[2];
    double carry[20];         // prologue_begin -> prologue_end: the shard's statistics and S_{s-1} (not held in registers
                              // across a speculative streaming pass)
};

// exp(m - M) with the table family (inside the step kernels)
__device__ __forceinline__ double shift_factor_t(double m, double M) {
    return (m == -CUDART_INF) ? 0.0 : texp_neg(m - M);
}

__device__ __forceinline__ double warp_max_nan(double v) {
#pragma unroll
    for (int mask = 16; mask > 0; mask >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, v, mask);
        v = (o > v || o != o) ? o : v;
    }
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int mask = 16; mask > 0; mask >>= 1) v += __shfl_xor_sync(0xffffffffu, v, mask);
    return v;
}

// one slab of the streaming branch: the warp's thread accumulators -> one record in shared memory
// [m, s, q, -][aux m, s, q, -][sx[D], sxx[D]]; fixed butterfly order, so the record depends on the slab alone
template <int D, bool APF>
__device__ __forceinline__ void warp_reduce_to_slab(const Acc<D> &sa, const Lse3 &sx, bool mom, double *rec, int lane) {
    const double M = warp_max_nan(sa.w.m);
    const double e = shift_factor_t(sa.w.m, M);
    const double s = warp_sum(sa.w.s * e), q = warp_sum(sa.w.q * (e * e));
    if (lane == 0) { rec[0] = M; rec[1] = s; rec[2] = q; }
    int off = 4;
    if (APF) {
        const double Ma = warp_max_nan(sx.m);
        const double ea = shift_factor_t(sx.m, Ma);
        const double as_ = warp_sum(sx.s * ea), aq = warp_sum(sx.q * (ea * ea));
        if (lane == 0) { rec[4] = Ma; rec[5] = as_; rec[6] = aq; }
        off = 8;
    }
    if (mom) {
#pragma unroll
        for (int c = 0; c < D; c++) {
            const double a1 = warp_sum(sa.sx[c] * e), a2 = warp_sum(sa.sxx[c] * e);
            if (lane == 0) { rec[off + c] = a1; rec[off + D + c] = a2; }
        }
    }
}

// this CTA's row of the partials of step t: the thread accumulators and (streaming branch) the slab records,
// every thread taking a fixed subset of the records in a fixed order.  Two passes -- block maximum first, then one
// exponential per record / accumulator -- instead of pairwise merges with two exponentials each.
template <int D, bool APF, int BS>
__device__ __forceinline__ void write_partial(const FilterArgs &a, long long t, const Acc<D> &acc, const Lse3 &aux,
                                              bool mom, StepSmem &sh, const double *s_slab = nullptr, int n_slab = 0) {
    const bool lane_rec = a.slab_lane != 0;
    const int n_rec = lane_rec ? n_slab * 32 : n_slab;
    auto rec_ptr = [&](int r) {
        return lane_rec ? s_slab + (size_t)(r >> 5) * a.slab_stride + (r & 31) : s_slab + (size_t)r * a.slab_stride;
    };
    const int rs_ = lane_rec ? 32 : 1;                    // distance between m, s, q inside a record
    if (n_slab > 0) __syncthreads();                      // all records are parked
    double mx[2] = {acc.w.m, APF ? aux.m : -CUDART_INF};
    for (int r = threadIdx.x; r < n_rec; r += BS) {
        const double *rec = rec_ptr(r);
        mx[0] = nanmax(mx[0], rec[0]);
        if (APF && !lane_rec) mx[1] = nanmax(mx[1], rec[4]);
    }
    block_max_all<2, BS>(mx, sh.red);
    const double ew = shift_factor_t(acc.w.m, mx[0]);
    const double ea = APF ? shift_factor_t(aux.m, mx[1]) : 0.0;
    double v[4 + 2 * D];
    v[0] = acc.w.s * ew;
    v[1] = acc.w.q * (ew * ew);
    v[2] = APF ? aux.s * ea : 0.0;
    v[3] = APF ? aux.q * (ea * ea) : 0.0;
#pragma unroll
    for (int c = 0; c < D; c++) {
        v[4 + c] = mom ? acc.sx[c] * ew : 0.0;
        v[4 + D + c] = mom ? acc.sxx[c] * ew : 0.0;
    }
    for (int r = threadIdx.x; r < n_rec; r += BS) {
        const double *rec = rec_ptr(r);
        const double e = shift_factor_t(rec[0], mx[0]);
        v[0] += rec[rs_] * e;
        v[1] += rec[2 * rs_] * (e * e);
        if (!lane_rec) {
            if (APF) {
                const double e2 = shift_factor_t(rec[4], mx[1]);
                v[2] += rec[5] * e2;
                v[3] += rec[6] * (e2 * e2);
            }
            if (mom) {
                const int off = APF ? 8 : 4;
#pragma unroll
                for (int c = 0; c < D; c++) { v[4 + c] += rec[off + c] * e; v[4 + D + c] += rec[off + D + c] * e; }
            }
        }
    }
    if (mom) block_sum_all<4 + 2 * D, BS>(v, sh.red);
    else {
        double w4[4] = {v[0], v[1], v[2], v[3]};
        block_sum_all<4, BS>(w4, sh.red);
        v[0] = w4[0]; v[1] = w4[1]; v[2] = w4[2]; v[3] = w4[3];
    }
    if (threadIdx.x == 0) {
        double *p = a.partials + ((size_t)(t % kPartSlots) * kMaxStepGrid + blockIdx.x) * kPartStride;
        p[0] = mx[0]; p[1] = v[0]; p[2] = v[1]; p[3] = 0.0;
        p[4] = APF ? mx[1] : mx[0]; p[5] = APF ? v[2] : v[0]; p[6] = APF ? v[3] : v[1]; p[7] = 0.0;
#pragma unroll
        for (int c = 0; c < kMaxD; c++) {
            p[8 + c] = (c < D) ? v[4 + (c < D ? c : 0)] : 0.0;
            p[12 + c] = (c < D) ? v[4 + D + (c < D ? c : 0)] : 0.0;
        }
    }
}

// merge in a fixed order (a then b); same algebra as Weights.__init__ on the concatenation
__device__ __forceinline__ void merge16(double (&a)[16], const double *b) {
#pragma unroll
    for (int k = 0; k < 2; k++) {           // k = 0: inferential triple (+ moments), k = 1: auxiliary triple
        const double am = a[4 * k], bm = b[4 * k];
        const double M = (bm > am || bm != bm) ? bm : am;
        const double ea = shift_factor(am, M), eb = shift_factor(bm, M);
        a[4 * k] = M;
        a[4 * k + 1] = a[4 * k + 1] * ea + b[4 * k + 1] * eb;
        a[4 * k + 2] = a[4 * k + 2] * (ea * ea) + b[4 * k + 2] * (eb * eb);
        if (k == 0) {
#pragma unroll
            for (int c = 8; c < 16; c++) a[c] = a[c] * ea + b[c] * eb;
        }
    }
}

// this shard's statistics of step s from the per-CTA partial rows (mailbox layout, 16 doubles).  Warp 0 alone merges
// the <= 256 rows -- lane l takes rows l, l + 32, ...; maximum first, then one exponential per row; fixed butterfly
// order -- and parks the 16 numbers in shared memory: one block barrier, and every CTA that runs this holds identical
// bits.
template <bool APF>
__device__ __forceinline__ void shard_totals(const FilterArgs &a, long long s, bool mom, StepSmem &sh, double (&loc)[16]) {
    const int G = a.grid, tid = threadIdx.x;
    if (tid < 32) {
        const double *base = a.partials + (size_t)(s % kPartSlots) * kMaxStepGrid * kPartStride;
        constexpr int kR = kMaxStepGrid / 32;
        double pm[kR], ps[kR], pq[kR], xm[kR], xs[kR], xq[kR];
        double mw = -CUDART_INF, ma = -CUDART_INF;
#pragma unroll
        for (int i = 0; i < kR; i++) {
            const int r = tid + 32 * i;
            pm[i] = -CUDART_INF; ps[i] = 0.0; pq[i] = 0.0; xm[i] = -CUDART_INF; xs[i] = 0.0; xq[i] = 0.0;
            if (r < G) {
                const double *row = base + (size_t)r * kPartStride;
                const double2 r0 = __ldcg(reinterpret_cast<const double2 *>(row));
                pm[i] = r0.x; ps[i] = r0.y; pq[i] = __ldcg(row + 2);
                if (APF) {
                    const double2 r1 = __ldcg(reinterpret_cast<const double2 *>(row + 4));
                    xm[i] = r1.x; xs[i] = r1.y; xq[i] = __ldcg(row + 6);
                }
            }
            mw = nanmax(mw, pm[i]);
            if (APF) ma = nanmax(ma, xm[i]);
        }
        mw = warp_max_nan(mw);
        if (APF) ma = warp_max_nan(ma);
        double v[12];
#pragma unroll
        for (int j2 = 0; j2 < 12; j2++) v[j2] = 0.0;
#pragma unroll
        for (int i = 0; i < kR; i++) {
            const int r = tid + 32 * i;
            const double ew = shift_factor(pm[i], mw);
            v[0] += ps[i] * ew;
            v[1] += pq[i] * (ew * ew);
            if (APF) {
                const double ea = shift_factor(xm[i], ma);
                v[2] += xs[i] * ea;
                v[3] += xq[i] * (ea * ea);
            }
            if (mom && r < G) {
                const double *row = base + (size_t)r * kPartStride + 8;
#pragma unroll
                for (int c = 0; c < 8; c++) v[4 + c] += __ldcg(row + c) * ew;
            }
        }
#pragma unroll
        for (int j2 = 0; j2 < 12; j2++)
            if (j2 < 4 || mom) v[j2] = warp_sum(v[j2]);
        if (tid == 0) {
            double *o = sh.peer[0];               // (not yet in use: the exchange fills it later)
            o[0] = mw; o[1] = v[0]; o[2] = v[1]; o[3] = 0.0;
            o[4] = APF ? ma : mw; o[5] = APF ? v[2] : v[0]; o[6] = APF ? v[3] : v[1]; o[7] = 0.0;
#pragma unroll
            for (int c = 0; c < 8; c++) o[8 + c] = v[4 + c];
        }
    }
    __syncthreads();
#pragma unroll
    for (int j2 = 0; j2 < 16; j2++) loc[j2] = sh.peer[0][j2];
    __syncthreads();
}

// exclusive prefixes P_b, P_{b+1} of this CTA over per-CTA values v (thread b holds v_b, 0 beyond the grid):
// sequential per warp + monotone clamps, the same bits in every CTA
template <int BS>
__device__ __forceinline__ void cta_prefix(double v, StepSmem &sh, double &p_b, double &p_next) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double iw = warp_scan_monotone(v, lane);
    if (lane == 31) sh.red[warp] = iw;
    __syncthreads();
    double woff = 0.0;
    for (int w_ = 0; w_ < BS / 32; w_++)
        if (w_ < warp) woff = woff + sh.red[w_];
    const double incl = woff + iw;                      // P_{tid+1}
    if (tid == 0 && blockIdx.x == 0) sh.pref[0] = 0.0;
    if (tid + 1 == (int)blockIdx.x) sh.pref[0] = incl;
    if (tid == (int)blockIdx.x) sh.pref[1] = incl;
    __syncthreads();
    p_b = sh.pref[0];
    p_next = fmax(sh.pref[1], p_b);
    __syncthreads();
}

struct StepDecision {
    int rs;                   // resample at step t
    long long nrs_prev;       // resampling steps before step t (grid-barrier epochs already passed)
    double reset_c;           // log-weight every resampled particle restarts from (minus logeta[A] for an APF)
    double xm, xs;            // (max, sum exp) of this shard's (auxiliary) weights: the CDF's normalisation
    double p_b, p_next;       // this CTA's range of the CDF
    double ess;               // ESS of step t - 1 (the fused-pair predictor)
};

// compute_summaries of step s = t - 1 (core.py:351-367) + time_to_resample of step t (core.py:181-183),
// by every CTA; the `writer` CTA also records S_s, the summary row and the moments row.
// Two halves.  prologue_begin: this shard's statistics of step s from the partial rows, sent to the peers at once
// (sharded filters), and the shard's OWN resampling test -- the prediction a sharded step kernel speculates on.
// prologue_end: the peers' statistics (the only wait), the global scalars, the decision, the bookkeeping.
struct PrologueCarry {
    bool mom;
};

template <bool APF>
__device__ __forceinline__ bool prologue_begin(const FilterArgs &a, long long t, StepSmem &sh, bool writer,
                                               PrologueCarry &pc) {
    const long long s = t - 1;
    const int tid = threadIdx.x;
    pc.mom = writer && a.moments != nullptr;
    // S_{s-1}: requested first, needed last
    StepState prev;
    prev.logLt = 0.0; prev.log_mean_w = 0.0; prev.nrs = 0; prev.rs_next = 0;
    if (s >= 1) {
        const StepState *pp = a.st + ((s - 1) & 1);
        prev.logLt = __ldcg(&pp->logLt); prev.log_mean_w = __ldcg(&pp->log_mean_w);
        prev.nrs = __ldcg(&pp->nrs); prev.rs_next = __ldcg(&pp->rs_next);
    }
    double loc[16];
    shard_totals<APF>(a, s, pc.mom, sh, loc);
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sh.carry[i] = loc[i];
        sh.carry[16] = prev.logLt; sh.carry[17] = prev.log_mean_w;
        sh.carry[18] = __longlong_as_double(prev.nrs); sh.carry[19] = __longlong_as_double((long long)prev.rs_next);
    }
    if (a.world > 1 && a.mail_local != nullptr) {
        // fused exchange over NVLink peer memory: CTA 0 stores this shard's statistics of step s into every
        // peer's mailbox (one lane per peer), fences, raises the epoch
        if (writer && tid < a.world) {
            double *slot = a.mail_peer[tid] + ((size_t)(s & 1) * a.world + a.rank) * kMailStride;
#pragma unroll
            for (int i = 0; i < 16; i++) slot[i] = loc[i];
            __threadfence_system();
            *reinterpret_cast<volatile double *>(slot + kMailEpoch) = (double)(s + 1);
        }
    }
    // the shard's own ESS test: with ~N / world particles per shard it agrees with the global one except within
    // sampling noise of the threshold
    const Lse3 xl{loc[4], loc[5], loc[6]};
    double lm_l, ess_l;
    weights_scalars(xl, (double)a.n, lm_l, ess_l);
    return (s + 1 < a.T) && (ess_l < (double)a.n * a.essrmin);
}

template <bool APF, int BS>
__device__ __forceinline__ StepDecision prologue_end(const FilterArgs &a, long long t, StepSmem &sh, bool writer,
                                                     bool need_prefix, const PrologueCarry &pc) {
    const long long s = t - 1;
    const int tid = threadIdx.x;
    __syncthreads();                                   // (sh.carry, written by thread 0 in prologue_begin)
    StepState prev;
    double loc[16];
#pragma unroll
    for (int i = 0; i < 16; i++) loc[i] = sh.carry[i];
    prev.logLt = sh.carry[16]; prev.log_mean_w = sh.carry[17];
    prev.nrs = __double_as_longlong(sh.carry[18]); prev.rs_next = (int)__double_as_longlong(sh.carry[19]);
    double glob[16];
#pragma unroll
    for (int j = 0; j < 16; j++) glob[j] = loc[j];
    if (a.world > 1) {
        if (a.mail_local != nullptr) {
            // every CTA waits for `world` epochs in its own mailbox
            const double *box = a.mail_local + (size_t)(s & 1) * a.world * kMailStride;
            if (tid < a.world) {
                wait_epoch(box + (size_t)tid * kMailStride + kMailEpoch, (double)(s + 1), a.sync_timeout);
                for (int i = 0; i < 16; i++)
                    sh.peer[tid][i] = *reinterpret_cast<const volatile double *>(box + (size_t)tid * kMailStride + i);
            }
        } else if (tid < a.world) {
            for (int i = 0; i < 16; i++) sh.peer[tid][i] = __ldcg(a.gathered + (size_t)tid * 16 + i);
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 16; j++) glob[j] = sh.peer[0][j];
        for (int r = 1; r < a.world; r++) merge16(glob, sh.peer[r]);         // rank order: identical bits everywhere
        if (a.rs_global && tid == 0) {
            // shard r's share of the global (auxiliary) weight mass, rank order
            double run = 0.0;
            for (int r = 0; r < a.world; r++) {
                const double pm_ = sh.peer[r][4], ps_ = sh.peer[r][5];
                const double pi = (pm_ == -CUDART_INF) ? 0.0 : ps_ * fexp_neg(pm_ - glob[4]) / glob[5];
                sh.goff[r] = run;
                sh.gpi[r] = pi;
                run = run + pi;
            }
            sh.goff[a.world] = run;
        }
        __syncthreads();
    }
    const Lse3 w{glob[0], glob[1], glob[2]}, x{glob[4], glob[5], glob[6]};
    const Lse3 xl{loc[4], loc[5], loc[6]};
    const double N = (double)a.n_global;
    double log_mean, ess, lm_aux, ess_aux;
    weights_scalars(w, N, log_mean, ess);
    if (APF) weights_scalars(x, N, lm_aux, ess_aux);
    else { lm_aux = log_mean; ess_aux = ess; }
    const int rs_s = prev.rs_next;                                          // did step s resample?
    const bool fresh = (s == 0) || (rs_s != 0);
    const double loglt = fresh ? log_mean : (log_mean - prev.log_mean_w);   // core.py:355-358
    const double logLt = prev.logLt + loglt;
    StepDecision d;
    d.rs = (s + 1 < a.T) && (ess_aux < N * a.essrmin);                      // strict <, NaN -> False
    d.nrs_prev = prev.nrs + (rs_s ? 1 : 0);
    // log-weight every resampled particle restarts from (minus logeta[A] for an APF):
    //   single device, non-APF : 0                        (Weights(), core.py:305)
    //   single device, APF     : log_mean_exp(logetat, W) (core.py:302) = LSE(aux) - LSE(w)
    //   sharded, per shard     : LSE_shard(aux) - LSE_all(w) + log(world): each shard resamples locally and
    //                            carries its share of the mass (SURVEY.md 8e)
    //   sharded, global        : the reference's restart from the global sums
    double rc = 0.0;
    if (a.rs_global) rc = APF ? (log(x.s) + x.m) - (log(w.s) + w.m) : 0.0;
    else if (APF || a.world > 1) rc = (log(xl.s) + xl.m) - (log(w.s) + w.m) + log((double)a.world);
    d.reset_c = rc;
    d.xm = xl.m; d.xs = xl.s;
    d.p_b = 0.0; d.p_next = 0.0;
    d.ess = ess;
    if (writer && tid == 0) {
        double *row = a.summaries + (size_t)s * SMCB_SUMMARY_STRIDE;
        row[0] = ess; row[1] = logLt; row[2] = (double)rs_s; row[3] = log_mean;
        StepState *o = a.st + (s & 1);
        o->logLt = logLt; o->log_mean_w = log_mean; o->ess = ess;
        o->wm = w.m; o->ws = w.s; o->wq = w.q;
        o->t = s; o->nrs = d.nrs_prev; o->rs = rs_s; o->rs_next = d.rs;
        if (a.moments != nullptr) {                                        // wmean_and_var, resampling.py:320-338
            double *mrow = a.moments + (size_t)s * 2 * kMaxD;
#pragma unroll
            for (int c = 0; c < kMaxD; c++) {
                const double mean = glob[8 + c] / w.s;
                mrow[c] = mean;
                mrow[kMaxD + c] = glob[12 + c] / w.s - mean * mean;
            }
        }
    }
    if (d.rs && need_prefix) {
        // The CTAs own contiguous particle ranges, so their partial sums ARE the tile aggregates of the weight
        // scan: exclusive prefixes P_0 = 0 <= P_1 <= ... <= P_G (fixed order, monotone, the same bits in every
        // CTA), and the scan needs no look-back at all.
        double v = 0.0;
        if (tid < a.grid) {                      // row tid of the partials: this CTA's (auxiliary) weight mass
            const double *row = a.partials + ((size_t)(s % kPartSlots) * kMaxStepGrid + tid) * kPartStride + (APF ? 4 : 0);
            v = __ldcg(row + 1) * shift_factor(__ldcg(row), d.xm) / d.xs;
        }
        cta_prefix<BS>(v, sh, d.p_b, d.p_next);
    }
    return d;
}

template <bool APF, int BS>
__device__ __forceinline__ StepDecision step_prologue(const FilterArgs &a, long long t, StepSmem &sh, bool writer,
                                                      bool need_prefix) {
    PrologueCarry pc;
    prologue_begin<APF>(a, t, sh, writer, pc);
    return prologue_end<APF, BS>(a, t, sh, writer, need_prefix, pc);
}

// all CTAs of the (co-resident) grid have arrived; `target` = arrivals expected in total since the filter was made
__device__ __forceinline__ void grid_barrier(const FilterArgs &a, unsigned long long target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(a.bar, 1ull);
        const long long t0 = clock64();
        while (*reinterpret_cast<volatile unsigned long long *>(a.bar) < target) {
            if (clock64() - t0 > 8000000000ll) { *a.sync_timeout = 2; break; }
        }
        __threadfence();
        asm volatile("fence.proxy.async;" ::: "memory");     // the CDF is read by TMA (async proxy) next
    }
    __syncthreads();
}

// the range of pairs this CTA owns
__device__ __forceinline__ void cta_range(const FilterArgs &a, int64_t &pstart, int64_t &pend) {
    const int64_t npairs = (a.n + 1) >> 1;
    pstart = (int64_t)blockIdx.x * a.chunk;
    pend = pstart + a.chunk < npairs ? pstart + a.chunk : npairs;
    if (pstart > npairs) pstart = npairs;
}

// ---------------------------------------------------------------------------
// one pair of particles 2p, 2p + 1: the pair is the unit of the Philox normals and of the paired stores.  k_batch
// (smcb_batch.cu) draws its normals through pair_normals too, so a batched run draws what the single filter draws.
// ---------------------------------------------------------------------------
// the normals of the pair at step t: the table-family Box-Muller of Philox pair counter `pair` ...
template <int NZ>
__device__ __forceinline__ void tab_normals(const Philox &key, uint64_t pair, uint32_t t, double (&z)[2][NZ]) {
#pragma unroll
    for (int c = 0; c < NZ; c++) normal_pair_tab(key, pair, t, (uint32_t)c, z[0][c], z[1][c]);
}
// ... or those of the step's injected (NZ, n) slice zin if it is not NULL; an absent second particle (2p + 1 = n) gets 0
template <int NZ>
__device__ __forceinline__ void pair_normals(const Philox &key, uint64_t pair, uint32_t t, const double *zin, int64_t n,
                                             int64_t p, double (&z)[2][NZ]) {
    if (!zin) return tab_normals<NZ>(key, pair, t, z);
#pragma unroll
    for (int c = 0; c < NZ; c++) {
        z[0][c] = zin[(size_t)c * n + 2 * p];
        z[1][c] = (2 * p + 1 < n) ? zin[(size_t)c * n + 2 * p + 1] : 0.0;
    }
}

// propagate the pair from xp (INIT: generate it; core.py:315-324) and weight it: lw = base + logG (Weights.add,
// resampling.py:241-244; INIT: lw = logG), and for an APF whose step t + 1 exists (`next`) the auxiliary weight
// lw + logeta_t(x).  NaN -> -inf (resampling.py:220).  Returns whether any of these values was +-inf / NaN (integer
// test), so that a caller can accumulate a finite batch with acc_add_batch's FINITE case.
template <class M, int FK, bool INIT>
__device__ __forceinline__ bool move_pair(const M &model, const StepK &k, const double (*xp)[M::D], const double *base,
                                          const double (&z)[2][M::NZ], bool next, double (&x)[2][M::D], double *l,
                                          double *av) {
    constexpr bool APF = FkTraits<FK>::apf;
    bool odd = false;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        double d;
        if (INIT) model_init<M, FK>(model, k, z[j], x[j], d);
        else model_move<M, FK>(model, k, xp[j], z[j], x[j], d);
        l[j] = INIT ? d : base[j] + d;
        odd |= nonfinite(l[j]);
        if (APF) {
            av[j] = next ? l[j] + model_logeta<M>(model, k, x[j]) : -CUDART_INF;
            odd |= nonfinite(av[j]);
        }
    }
    if (odd) {
#pragma unroll
        for (int j = 0; j < 2; j++) { l[j] = fix_nan(l[j]); if (APF) av[j] = fix_nan(av[j]); }
    }
    return odd;
}

// store the pair into SoA buffers of n particles (component stride n).  An odd n's last particle is stored alone, and
// its partner slot is masked (x = 0, lw = av = -inf) so that it contributes exactly 0 to the accumulators.
template <int D, bool APF>
__device__ __forceinline__ void store_pair(double *Xo, double *lwo, int64_t n, int64_t p, bool vec_x, double (&x)[2][D],
                                           double *l, double *av) {
    if (2 * p + 1 < n) {
        if (vec_x) {
#pragma unroll
            for (int c = 0; c < D; c++) st2(Xo + (size_t)c * n + 2 * p, x[0][c], x[1][c]);
        } else {                                      // odd SoA stride: component rows are only 8-byte aligned
#pragma unroll
            for (int c = 0; c < D; c++) { Xo[(size_t)c * n + 2 * p] = x[0][c]; Xo[(size_t)c * n + 2 * p + 1] = x[1][c]; }
        }
        st2(lwo + 2 * p, l[0], l[1]);
    } else {
#pragma unroll
        for (int c = 0; c < D; c++) { Xo[(size_t)c * n + 2 * p] = x[0][c]; x[1][c] = 0.0; }
        lwo[2 * p] = l[0];
        l[1] = -CUDART_INF;
        if (APF) av[1] = -CUDART_INF;
    }
}

// ---------------------------------------------------------------------------
// t = 0: generate_particles + reweight (core.py:315-324, 373-374)
// ---------------------------------------------------------------------------
template <class M, int FK>
__global__ void __launch_bounds__(StepCfg<M>::BS, 1) k_init(M model, FilterArgs a) {
    constexpr bool APF = FkTraits<FK>::apf;
    constexpr int D = M::D, NZ = M::NZ, BS = StepCfg<M>::BS;
    __shared__ StepSmem sh;
    __shared__ __align__(8) uint64_t s_tabbar;
    if (threadIdx.x == 0) mtab_issue(a.math_tab, &s_tabbar);
    __syncthreads();
    mbar_wait(&s_tabbar, 0);
    const StepK k = step_consts(a, 0);
    double *Xo = a.X[0], *lwo = a.lw[0];
    Acc<D> acc;
    acc_init(acc);
    Lse3 aux = lse3_empty();
    const bool mom = a.moments != nullptr;
    const int64_t n = a.n;
    const bool has_next = APF && a.T > 1;
    const bool vec_x = (D == 1) || ((n & 1) == 0);
    int64_t pstart, pend;
    cta_range(a, pstart, pend);
    for (int64_t p = pstart + threadIdx.x; p < pend; p += BS) {
        double z[2][NZ], x[2][D], l[2], av[2];
        pair_normals<NZ>(a.key, (uint64_t)((a.index_offset >> 1) + p), 0u, a.z_in, n, p, z);
        move_pair<M, FK, true>(model, k, nullptr, nullptr, z, has_next, x, l, av);
        store_pair<D, APF>(Xo, lwo, n, p, vec_x, x, l, av);
        acc_add_batch<2, D>(acc, l, x, mom);
        if (APF) lse3_add_batch<2>(aux, av);
    }
    write_partial<D, APF, BS>(a, 0, acc, aux, mom, sh);
}

// ---------------------------------------------------------------------------
// resampling steps: normalised (auxiliary) weights -> CDF   (resampling.py:223-225 + scan)
// ---------------------------------------------------------------------------
template <class M, int FK>
struct LoadWeights {
    const double *lw, *X;
    int64_t ntot;  // particles on this device (SoA component stride)
    double m, s;
    M model;
    StepK kprev;   // step t-1 with y_next = data[t]: what logeta(t-1, X) needs
    struct Raw { double l[8]; double x[8][FkTraits<FK>::apf ? M::D : 1]; };
    // the loads of 8 consecutive particles (log-weights; states too when logeta needs them) ...
    __device__ __forceinline__ void fetch(int64_t i0, int64_t n, Raw &r) const {
        constexpr bool APF = FkTraits<FK>::apf;
        constexpr int D = M::D;
        const bool vec_x = (D == 1) || ((ntot & 1) == 0);
        if (i0 + 8 <= n) {
#pragma unroll
            for (int j = 0; j < 8; j += 2) { double2 t = ld2(lw + i0 + j); r.l[j] = t.x; r.l[j + 1] = t.y; }
            if (APF) {
#pragma unroll
                for (int c = 0; c < D; c++) {
#pragma unroll
                    for (int j = 0; j < 8; j += 2) {
                        if (vec_x) {
                            double2 t = ld2(X + (size_t)c * ntot + i0 + j);
                            r.x[j][APF ? c : 0] = t.x; r.x[j + 1][APF ? c : 0] = t.y;
                        } else {
                            r.x[j][APF ? c : 0] = X[(size_t)c * ntot + i0 + j];
                            r.x[j + 1][APF ? c : 0] = X[(size_t)c * ntot + i0 + j + 1];
                        }
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) {
                r.l[j] = (i0 + j < n) ? lw[i0 + j] : -CUDART_INF;
                if (APF) {
#pragma unroll
                    for (int c = 0; c < D; c++) r.x[j][APF ? c : 0] = (i0 + j < n) ? X[(size_t)c * ntot + i0 + j] : 0.0;
                }
            }
        }
    }
    // ... and their normalised (auxiliary) weights W = exp(lw - m) * (1 / s)  (resampling.py:223-225; the reference
    // divides by s: one rounding apart, and the CDF the ancestors are held to is the device's own)
    __device__ __forceinline__ void weights(const Raw &r, int64_t i0, int64_t n, double (&v)[8]) const {
        constexpr bool APF = FkTraits<FK>::apf;
        const double inv_s = 1.0 / s;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            double e = r.l[j];
            if (APF) e = fix_nan(e + model_logeta<M>(model, kprev, r.x[j]));
            v[j] = (i0 + j < n) ? texp(e - m) * inv_s : 0.0;
        }
    }
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&v)[8]) const {
        Raw r;
        fetch(i0, n, r);
        weights(r, i0, n, v);
    }
};

// inclusive scan of the values load() yields on [e0, e1), written to out[]; starts from p_b and every value is
// clamped into [p_b, p_next], so the result is non-decreasing across CTAs by construction
template <int BS, class LOAD>
__device__ __forceinline__ void scan_range(const LOAD &load, int64_t e0, int64_t e1, double p_b, double p_next,
                                           double *out, double *s_warp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int kTile = BS * kScanItems;
    double carry = 0.0;
    for (int64_t base0 = e0; base0 < e1; base0 += kTile) {
        const int64_t i0 = base0 + (int64_t)tid * kScanItems;
        double r[kScanItems];
        load(i0, e1, r);
#pragma unroll
        for (int j = 1; j < kScanItems; j++) r[j] = r[j - 1] + r[j];
        const double iw = warp_scan_monotone(r[kScanItems - 1], lane);
        if (lane == 31) s_warp[warp] = iw;
        __syncthreads();
        double woff = 0.0, total = 0.0;
#pragma unroll
        for (int w = 0; w < BS / 32; w++) {
            if (w < warp) woff = woff + s_warp[w];
            total = total + s_warp[w];
        }
        const double incl = woff + iw;
        const double up = __shfl_up_sync(0xffffffffu, iw, 1);
        const double excl = (lane == 0) ? woff : (woff + up);
        const double b_i = fmin(p_b + carry, p_next);         // base of this sub-tile
        const double carry_next = carry + total;
        const double b_next = fmin(p_b + carry_next, p_next); // base of the next one
        const double tb = b_i + excl;
        const double cap = fmin(b_i + incl, b_next);
        double o[kScanItems];
#pragma unroll
        for (int j = 0; j < kScanItems; j++) o[j] = fmin(tb + r[j], cap);
        if (i0 + kScanItems <= e1) {
            store_items(out, i0, o);
        } else {
#pragma unroll
            for (int j = 0; j < kScanItems; j++)
                if (i0 + j < e1) out[i0 + j] = o[j];
        }
        carry = carry_next;
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------
// Offspring counting (systematic / stratified; resampling.py:599-610): while a CTA scans its range it also
// scatters the ancestors.  With su_k = (u + k) / N the outputs that select entry j are the k with
// cdf[j-1] < su_k <= cdf[j], i.e. k in [F(cdf[j-1]), F(cdf[j])) where F(c) = #{k : su_k <= c} = floor(c N - u) + 1.
// F is evaluated in fp64 (one FMA + floor), so a boundary output may land one entry off when c N - u sits within
// rounding distance of an integer; the move pass VERIFIES every ancestor against the exact su_k the reference
// computes (the division) and walks to the searchsorted answer, so the result is bit-identical to
// np.searchsorted(cdf, su) -- the scatter only has to be a good hint that leaves no output unassigned.  Coverage is
// gap-free by construction: consecutive threads / tiles / CTAs use the SAME fp64 expression for the shared boundary.
// Stratified uses u = 0 (the hint is searchsorted(cdf, k / N) <= the answer; the move pass walks forward).
// ---------------------------------------------------------------------------
struct Scatter {
    long long *A;
    double Nd, u;
    long long n_out;
    // floor(c N - u) + 1 as rint(c N - u + 1/2) through the magic-number sum (no conversion instruction); the
    // half-way cases differ from the floor -- it is a hint, the move pass decides
    __device__ __forceinline__ long long F(double c) const {
        const double t = fma(c, Nd, 0.5 - u) + kRintMagic;            // c in [0, 1], N < 2^50 (the magic constant's ulp is 1:
                                                                      // it must be added AFTER the fraction is formed)
        const long long k = (long long)(((unsigned long long)(__double2hiint(t) & 0xFFFFF) << 32) |
                                        (unsigned int)__double2loint(t)) - (1ll << 51);
        return k < 0 ? 0 : (k > n_out ? n_out : k);
    }
};

constexpr int kHeavy = 48;          // offspring of one entry above which the whole group fills them cooperatively

// ---------------------------------------------------------------------------
// Scan + scatter of the CTA's range as a PIPELINE of warp groups.  One CTA per SM means one block barrier domain per
// SM: with the whole CTA on one tile every phase of the tile (loads, exponentials, warp scans, the prefix hand-over,
// stores) is exposed -- measured 115 us for 16 B/particle where the three independent 256-thread CTAs of round 1 took
// 52.  So the CTA's warps are split into NG groups of GW warps; group g takes the tiles g, g + NG, ... of the CTA's range, its
// own named barrier (bar.sync g + 1) and its own slice of the hint buffer; the only thing a tile needs from its
// predecessor is the running prefix P_t, handed over through a small shared-memory ring (value + epoch flag) right
// after the group's warp scan -- a decoupled look-back of depth one with a FIXED association order
// (P_{t+1} = min(P_t + total_t, p_next)), so the CDF is deterministic and monotone by construction.
// ---------------------------------------------------------------------------
constexpr int kScanRing = 32;
constexpr int kGroupQ = 8;
__device__ __forceinline__ int *sc_timeout(StepSmem &sh) { return sh.timeout_ptr; }

__device__ __forceinline__ void group_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <int BS, int GW, class LOAD>
__device__ __forceinline__ void scan_scatter_groups(const LOAD &load, int64_t e0, int64_t e1, double p_b, double p_next,
                                                    double *out, const Scatter &sc, bool last_cta, StepSmem &sh,
                                                    int *s_hint_all, int hint_cap_total) {
    constexpr int NG = BS / 32 / GW, GT = GW * 32, kTile = GT * kScanItems;
    static_assert(NG <= 15 && NG <= kScanRing && GW <= 8, "scan_scatter_groups: one named barrier (ids 1..15) and one table row per group");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = warp / GW, gw = warp % GW, gt = tid - grp * GT;
    int *s_hint = s_hint_all + grp * (hint_cap_total / NG);
    const int hint_cap = hint_cap_total / NG;
    volatile double *ringP = sh.ringP;
    volatile int *ringF = sh.ringF;
    if (tid < kScanRing) { sh.ringF[tid] = (tid == 0) ? 1 : 0; if (tid == 0) sh.ringP[0] = p_b; }
    if (tid < NG) sh.gqn[tid] = 0;
    __syncthreads();
    const int64_t nt = (e1 - e0 + kTile - 1) / kTile;
    typename LOAD::Raw nxt;
    if (grp < nt) load.fetch(e0 + (int64_t)grp * kTile + (int64_t)gt * kScanItems, e1, nxt);
    for (int64_t t = grp; t < nt; t += NG) {
        const int64_t base0 = e0 + t * kTile;
        const int64_t i0 = base0 + (int64_t)gt * kScanItems;
        const bool last_tile = (t == nt - 1);
        double r[kScanItems];
        const typename LOAD::Raw cur = nxt;
        if (t + NG < nt) load.fetch(i0 + (int64_t)NG * kTile, e1, nxt);
        load.weights(cur, i0, e1, r);
#pragma unroll
        for (int j = 1; j < kScanItems; j++) r[j] = r[j - 1] + r[j];
        const double iw = warp_scan_monotone(r[kScanItems - 1], lane);
        if (lane == 31) sh.gwarp[grp][gw] = iw;
        group_sync(grp + 1, GT);
        double woff = 0.0, total = 0.0;
#pragma unroll
        for (int w = 0; w < GW; w++) {
            if (w < gw) woff = woff + sh.gwarp[grp][w];
            total = total + sh.gwarp[grp][w];
        }
        if (gt == 0) {                                             // take P_t, hand P_{t+1} to the next tile at once
            const int slot = (int)(t % kScanRing), nslot = (int)((t + 1) % kScanRing);
            const long long t0 = clock64();
            while (ringF[slot] != (int)(t + 1)) {
                if (clock64() - t0 > 4000000000ll) { *sc_timeout(sh) = 3; break; }
            }
            const double Pt = ringP[slot];
            const double Pn = fmin(Pt + total, p_next);
            ringP[nslot] = Pn;
            __threadfence_block();
            ringF[nslot] = (int)(t + 2);
            sh.gpref[grp][0] = Pt;
            sh.gpref[grp][1] = Pn;
        }
        group_sync(grp + 1, GT);
        const double b_i = sh.gpref[grp][0], b_next = sh.gpref[grp][1];
        const double incl = woff + iw;
        const double up = __shfl_up_sync(0xffffffffu, iw, 1);
        const double excl = (lane == 0) ? woff : (woff + up);
        const double tb = b_i + excl;
        const double cap = fmin(b_i + incl, b_next);
        double o[kScanItems];
#pragma unroll
        for (int j = 0; j < kScanItems; j++) o[j] = fmin(tb + r[j], cap);
        if (i0 + kScanItems <= e1) {
            store_items(out, i0, o);
        } else {
#pragma unroll
            for (int j = 0; j < kScanItems; j++)
                if (i0 + j < e1) out[i0 + j] = o[j];
        }
        // ---- scatter.  The tile's entries cover the outputs [K0, K1) = [F(P_t), F(P_{t+1})) (the same fp64
        // expressions the neighbouring tiles / CTAs use, so coverage is gap-free).  Normally that range fits the
        // group's slice of the shared-memory hint buffer: every thread writes the (tile-relative) entry index of each
        // of its outputs there -- 4-byte stores with neighbouring lanes writing neighbouring words -- and the group
        // then copies the buffer to A with fully coalesced stores.  A range too long for the buffer (a few entries
        // with very many offspring) is written directly; entries with more than kHeavy offspring are queued, and the
        // whole group fills them cooperatively.
        const long long K0 = (blockIdx.x == 0 && t == 0) ? 0 : sc.F(b_i);
        const long long K1 = (last_tile && last_cta) ? sc.n_out : sc.F(last_tile ? p_next : b_next);
        const bool staged = (K1 - K0) <= (long long)hint_cap;
        if (i0 < e1) {
            const bool tail_thread = (i0 + kScanItems >= e1);
            long long ks = (gt == 0) ? K0 : sc.F(tb);
            const long long kend = (gt == GT - 1 || tail_thread) ? K1 : sc.F(b_i + incl);
            ks = ks < K0 ? K0 : (ks > K1 ? K1 : ks);
#pragma unroll
            for (int j = 0; j < kScanItems; j++) {
                if (i0 + j < e1) {
                    const bool last_entry = (j == kScanItems - 1) || (i0 + j + 1 >= e1);
                    long long ke = last_entry ? kend : sc.F(o[j]);
                    ke = ke < ks ? ks : (ke > kend ? kend : ke);
                    if (staged) {
                        const int rel = gt * kScanItems + j;
                        for (long long k = ks; k < ke; k++) s_hint[(int)(k - K0)] = rel;
                    } else {
                        if (ke - ks > kHeavy) {
                            const int q = atomicAdd(&sh.gqn[grp], 1);
                            if (q < kGroupQ) { sh.gq[grp][q][0] = ks; sh.gq[grp][q][1] = ke; sh.gq[grp][q][2] = i0 + j; ks = ke; }
                        }
                        for (long long k = ks; k < ke; k++) sc.A[k] = i0 + j;
                    }
                    ks = ke;
                }
            }
        }
        group_sync(grp + 1, GT);
        if (staged) {
            const int cnt = (int)(K1 - K0);
            for (int k = gt; k < cnt; k += GT) sc.A[K0 + k] = base0 + s_hint[k];
        } else {
            const int nq = sh.gqn[grp] < kGroupQ ? sh.gqn[grp] : kGroupQ;
            for (int q = 0; q < nq; q++) {
                const long long ks = sh.gq[grp][q][0], ke = sh.gq[grp][q][1], jj = sh.gq[grp][q][2];
                for (long long k = ks + gt; k < ke; k += GT) sc.A[k] = jj;
            }
        }
        group_sync(grp + 1, GT);
        if (gt == 0) sh.gqn[grp] = 0;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------
// grid points.  Uniforms: injected row uin = (n + 1) of the step, or Philox (purpose kPurposeUniform, pair index, t).
// ---------------------------------------------------------------------------
// systematic resampling's one uniform of step t (resampling.py:609)
__device__ __forceinline__ double systematic_u(const Philox &key, long long t, const double *uin) {
    if (uin) return uin[0];
    double u0, u1;
    uniform_pair(key, 0ull, (uint32_t)t, kPurposeUniform, u0, u1);
    return u0;
}

// su_k of the outputs 2p, 2p + 1 of pair p out of M: systematic (u_sys + k) / M (resampling.py:609) or stratified
// (u_k + k) / M (resampling.py:602) with the uniforms of Philox pair `pair`.  Stratified draws only for a `valid` pair;
// an absent second output (!two) gets u = 0.
template <int SCHEME>
__device__ __forceinline__ void grid_pair(double u_sys, const Philox &key, uint64_t pair, uint32_t t, const double *uin,
                                          int64_t p, bool valid, bool two, double M, double &su0, double &su1) {
    double u0 = u_sys, u1 = u_sys;
    if (SCHEME == SMCB_RS_STRATIFIED) {
        u0 = 0.0; u1 = 0.0;
        if (valid) {
            if (uin) { u0 = uin[2 * p]; u1 = two ? uin[2 * p + 1] : 0.0; }
            else uniform_pair(key, pair, t, kPurposeUniform, u0, u1);
        }
    }
    su0 = (u0 + (double)(2 * p)) / M;
    su1 = (u1 + (double)(2 * p + 1)) / M;
}

// multinomial: the exponential spacings -log u_i, -log u_{i+1} (resampling.py:536-537) for even i; entry i + 1
// exists if i + 1 < e, else it is 0
__device__ __forceinline__ void spacings_pair(const Philox &key, uint32_t t, const double *uin, int64_t i, int64_t e,
                                              double &v0, double &v1) {
    double u0, u1;
    if (uin) { u0 = uin[i]; u1 = (i + 1 < e) ? uin[i + 1] : 1.0; }
    else uniform_pair(key, (uint64_t)(i >> 1), t, kPurposeUniform, u0, u1);
    v0 = -log(u0);                    // u may be 0 or injected: library log
    v1 = (i + 1 < e) ? -log(u1) : 0.0;
}

// multinomial: exponential spacings z = cumsum(-log u), n + 1 of them (resampling.py:536-537), blocked like
// the weights: pass 1 leaves v_i = -log u_i in su[] and the CTA's sum in blk_agg[]; after a grid barrier
// pass 2 scans the CTA's range from the (fixed-order, monotone) prefix of the CTA sums.
__device__ __forceinline__ void spacings_range(const FilterArgs &a, int64_t &e0, int64_t &e1) {
    int64_t pstart, pend;
    cta_range(a, pstart, pend);
    e0 = 2 * pstart;
    e1 = 2 * pend < a.n ? 2 * pend : a.n;
    if (blockIdx.x == gridDim.x - 1) e1 = a.n + 1;                // the last CTA also takes element n
}

struct LoadSpacings {
    const double *su;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&v)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = (i0 + j < n) ? __ldcg(su + i0 + j) : 0.0;
    }
};

template <int BS>
__device__ __forceinline__ void spacings_pass1(const FilterArgs &a, long long t, StepSmem &sh) {
    int64_t e0, e1;
    spacings_range(a, e0, e1);
    const double *uin = a.u_in ? a.u_in + (size_t)t * (a.n + 1) : nullptr;
    double acc[1] = {0.0};
    for (int64_t i = e0 + 2 * (int64_t)threadIdx.x; i < e1; i += 2 * BS) {
        double v0, v1;
        spacings_pair(a.key, (uint32_t)t, uin, i, e1, v0, v1);
        a.su[i] = v0;
        if (i + 1 < e1) a.su[i + 1] = v1;
        acc[0] += v0 + v1;
    }
    block_sum_all<1, BS>(acc, sh.red);
    if (threadIdx.x == 0) a.blk_agg[blockIdx.x] = acc[0];
}

template <int BS>
__device__ __forceinline__ void spacings_pass2(const FilterArgs &a, StepSmem &sh, double *s_warp) {
    const double v = ((int)threadIdx.x < a.grid) ? __ldcg(a.blk_agg + threadIdx.x) : 0.0;
    double p_b, p_next;
    cta_prefix<BS>(v, sh, p_b, p_next);
    int64_t e0, e1;
    spacings_range(a, e0, e1);
    LoadSpacings load{a.su};
    scan_range<BS>(load, e0, e1, p_b, p_next, a.su, s_warp);
}

__device__ __forceinline__ int shard_of(const double *goff, const double *gpi, int world, double su) {
    int k = 0;
    while (k + 1 < world && su >= goff[k + 1]) k++;
    while (k > 0 && !(gpi[k] > 0.0)) k--;
    while (k + 1 < world && !(gpi[k] > 0.0)) k++;
    return k;
}

// what one step of the streaming pass needs besides the particles, and where it writes them
struct StepIo {
    long long t;
    StepK k;
    const double *zin;       // injected normals of step t, (NZ, n), or NULL
    double *Xo, *lwo;        // buffers [t & 1]
    bool last_apf;           // step t + 1 exists (an APF computes its auxiliary weights)
};

__device__ __forceinline__ StepIo step_io(const FilterArgs &a, long long t, int nz) {
    StepIo io;
    io.t = t;
    io.k = step_consts(a, t);
    io.zin = a.z_in ? a.z_in + (size_t)t * nz * a.n : nullptr;
    io.Xo = a.X[t & 1];
    io.lwo = a.lw[t & 1];
    io.last_apf = t + 1 < a.T;
    return io;
}

// what every phase of one k_step launch reads: step t's constants and output buffers, the step that wrote the input
// buffers, and this CTA's range of pairs
struct StepEnv {
    StepIo io;               // step t
    StepK kprev;             // step t - 1, whose weights the resampling branch resamples
    int cur;                 // step t - 1 wrote buffers [cur]
    int64_t n;
    int64_t pstart, pend;    // this CTA's pairs
    bool vec_x;              // SoA component rows are 16-byte aligned
    bool mom;                // moments are collected
};

// propagate + reweight one pair of particles by step io.t; writes x', lw'; returns x', lw' (and the auxiliary
// log-weights of the next step for an APF), -inf in masked slots
template <class M, int FK>
__device__ __forceinline__ void do_pair(const M &model, const FilterArgs &a, const StepIo &io, int64_t n, bool vec_x,
                                        int64_t p, const double (&xp)[2][M::D], const double (&base)[2],
                                        double (&x)[2][M::D], double *l, double *av) {
    double z[2][M::NZ];
    pair_normals<M::NZ>(a.key, (uint64_t)((a.index_offset >> 1) + p), (uint32_t)io.t, io.zin, n, p, z);
    move_pair<M, FK, false>(model, io.k, xp, base, z, io.last_apf, x, l, av);
    store_pair<M::D, FkTraits<FK>::apf>(io.Xo, io.lwo, n, p, vec_x, x, l, av);
}

// The streaming pass: A = arange(N), Xp = X (core.py:335-336).  Step t -- FUSED: and step t + 1 -- over this CTA's
// pairs.  The statistics go to slab records: step t's in s_stage, step t + 1's in the CTA's slice of fuse_slab.
// Returns the number of records.  Work unit = one "iteration" of a warp: kU x 32 consecutive pairs (kU coalesced
// 512-byte rows per array), kU pairs in flight per thread.
template <class M, int FK, bool FUSED>
__device__ __forceinline__ int stream_pass(const M &model, const FilterArgs &a, const StepEnv &e, StepSmem &sh,
                                           double *s_stage) {
    constexpr bool APF = FkTraits<FK>::apf;
    constexpr int D = M::D, NZ = M::NZ;
    constexpr int kU = StepCfg<M>::kU;
    constexpr int kIt = 32 * kU;                                          // pairs per iteration
    const StepIo &io0 = e.io;
    const int64_t n = e.n, pstart = e.pstart, pend = e.pend;
    const bool vec_x = e.vec_x, mom = e.mom;
    const double *__restrict__ Xi = a.X[e.cur];
    const double *__restrict__ lwi = a.lw[e.cur];
    const int lane = threadIdx.x & 31;
    const int npl = (int)(pend - pstart);                                 // pairs of this CTA (< 2^31)
    const int n_iter = (npl + kIt - 1) / kIt;
    // iterations made of complete pairs only run without any bounds test (the odd last particle and the ragged
    // end of the range take the general path)
    const int64_t whole = (n >> 1) < pend ? (n >> 1) : pend;
    const int n_full = whole > pstart ? (int)((whole - pstart) / kIt) : 0;
    const bool fast_ok = (io0.zin == nullptr) && vec_x;
    const double *__restrict__ lwi_c = lwi + 2 * pstart;
    const double *__restrict__ Xi_c = Xi + 2 * pstart;
    const uint64_t gpair0 = (uint64_t)((a.index_offset >> 1) + pstart);
    // one iteration: pairs (relative to pstart) i * kIt + u * 32 + lane.  Loads and arithmetic are separate so
    // that the inputs of the NEXT iteration can be requested before the current one is computed.
    struct In { double base[kU][2]; double xp[kU][2][D]; };
    auto load_full = [&](const double *Xs_c, const double *lws_c, int i, In &in) {
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const int o2 = 2 * (i * kIt + u * 32 + lane);
            const double2 tl = ld2(lws_c + o2);
            in.base[u][0] = tl.x; in.base[u][1] = tl.y;
#pragma unroll
            for (int c = 0; c < D; c++) {
                const double2 tx = ld2(Xs_c + (size_t)c * n + o2);
                in.xp[u][0][c] = tx.x; in.xp[u][1][c] = tx.y;
            }
        }
    };
    auto compute_full = [&](const StepIo &io, int i, const In &in, Acc<D> &ac, Lse3 &ax, double (&l)[2 * kU],
                            double (&x)[2 * kU][D]) {
        double av[APF ? 2 * kU : 1];
        bool odd = false;                                 // some value is +-inf / NaN (integer test)
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const int prel = i * kIt + u * 32 + lane;
            double z[2][NZ];
            tab_normals<NZ>(a.key, gpair0 + (uint64_t)prel, (uint32_t)io.t, z);
            // (move_pair's arithmetic written out: this is the streaming pass's inner loop, and it takes one NaN
            // fix-up per iteration instead of one per pair)
#pragma unroll
            for (int j2 = 0; j2 < 2; j2++) {
                double d;
                model_move<M, FK>(model, io.k, in.xp[u][j2], z[j2], x[2 * u + j2], d);
                l[2 * u + j2] = in.base[u][j2] + d;                   // Weights.add, resampling.py:241-244
                odd |= nonfinite(l[2 * u + j2]);
                if (APF) {
                    av[APF ? 2 * u + j2 : 0] = io.last_apf ? l[2 * u + j2] + model_logeta<M>(model, io.k, x[2 * u + j2])
                                                           : -CUDART_INF;
                    odd |= nonfinite(av[APF ? 2 * u + j2 : 0]);
                }
            }
        }
        if (odd) {                                        // rare: NaN -> -inf (resampling.py:220)
#pragma unroll
            for (int q = 0; q < 2 * kU; q++) {
                l[q] = fix_nan(l[q]);
                if (APF) av[APF ? q : 0] = fix_nan(av[APF ? q : 0]);
            }
        }
        double *const lwo_c = io.lwo + 2 * pstart;
        double *const Xo_c = io.Xo + 2 * pstart;
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const int o2 = 2 * (i * kIt + u * 32 + lane);
#pragma unroll
            for (int c = 0; c < D; c++) st2(Xo_c + (size_t)c * n + o2, x[2 * u][c], x[2 * u + 1][c]);
            st2(lwo_c + o2, l[2 * u], l[2 * u + 1]);
        }
        if (!odd) {
            acc_add_batch<2 * kU, D, true>(ac, l, x, mom);
        } else {
            acc_add_batch<2 * kU, D, false>(ac, l, x, mom);
        }
        if (APF) lse3_add_batch<(APF ? 2 * kU : 1)>(ax, av);
    };
    // general path: ragged end of the range, the odd last particle, injected normals, odd SoA stride
    auto load_general = [&](const double *Xs, const double *lws, int i, In &in) {
        const int64_t qbase = pstart + (int64_t)i * kIt;
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const int64_t p = qbase + u * 32 + lane;
            if (p < pend && 2 * p + 1 < n) {
                double2 tl = ld2(lws + 2 * p);
                in.base[u][0] = tl.x; in.base[u][1] = tl.y;
#pragma unroll
                for (int c = 0; c < D; c++) {
                    if (vec_x) {
                        double2 tx = ld2(Xs + (size_t)c * n + 2 * p);
                        in.xp[u][0][c] = tx.x; in.xp[u][1][c] = tx.y;
                    } else {
                        in.xp[u][0][c] = Xs[(size_t)c * n + 2 * p]; in.xp[u][1][c] = Xs[(size_t)c * n + 2 * p + 1];
                    }
                }
            } else if (p < pend) {
                in.base[u][0] = lws[2 * p]; in.base[u][1] = 0.0;
#pragma unroll
                for (int c = 0; c < D; c++) { in.xp[u][0][c] = Xs[(size_t)c * n + 2 * p]; in.xp[u][1][c] = 0.0; }
            }
        }
    };
    auto compute_general = [&](const StepIo &io, int i, const In &in, Acc<D> &ac, Lse3 &ax, double (&l)[2 * kU],
                               double (&x)[2 * kU][D]) {
        double av[APF ? 2 * kU : 1];
        const int64_t qbase = pstart + (int64_t)i * kIt;
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const int64_t p = qbase + u * 32 + lane;
            if (p < pend) {
                do_pair<M, FK>(model, a, io, n, vec_x, p, in.xp[u], in.base[u],
                               reinterpret_cast<double (&)[2][D]>(x[2 * u]), l + 2 * u, APF ? av + 2 * u : av);
            } else {
                l[2 * u] = l[2 * u + 1] = -CUDART_INF;
                if (APF) av[APF ? 2 * u : 0] = av[APF ? 2 * u + 1 : 0] = -CUDART_INF;
#pragma unroll
                for (int c = 0; c < D; c++) { x[2 * u][c] = 0.0; x[2 * u + 1][c] = 0.0; }
            }
        }
        acc_add_batch<2 * kU, D>(ac, l, x, mom);
        if (APF) lse3_add_batch<(APF ? 2 * kU : 1)>(ax, av);
    };
    // dynamic slabs: a warp takes the next slab of `slab_it` consecutive iterations from a shared counter, so
    // the warps of the SM drift apart (one warp's loads overlap the others' arithmetic) and all retire within
    // one slab of each other whatever the scheduler's priorities.  Determinism: a slab's statistics are parked in
    // shared memory as one record per slab -- the 32 lanes' own (max, sum exp, sum exp^2), or, when auxiliary
    // weights / moments make that too large, their fixed-order reduction over the warp -- and write_partial
    // merges the records in slab order, so the result does not depend on which warp ran which slab.  The tail of
    // the range is cut into single-iteration slabs (short drain).  The records alias the CDF staging buffers,
    // which only the resampling branch uses.
    const int slab_it = a.slab_it;
    const int n_small = a.slab_small < n_iter ? a.slab_small : n_iter;
    const int it_small0 = n_iter - n_small;                               // first single-iteration slab
    const int n_big = (it_small0 + slab_it - 1) / slab_it;                // slabs of (up to) slab_it iterations
    const int n_slab = n_big + n_small;
    const bool lane_rec = a.slab_lane != 0;
    auto grab = [&]() {
        int v = 0;
        if (lane == 0) v = atomicAdd(&sh.next, 1);
        return __shfl_sync(0xffffffffu, v, 0);
    };
    auto first_it = [&](int sl) { return sl < n_big ? sl * slab_it : it_small0 + (sl - n_big); };
    auto park = [&](double *rec, const Acc<D> &sa, const Lse3 &sx) {
        if (lane_rec) { rec[lane] = sa.w.m; rec[32 + lane] = sa.w.s; rec[64 + lane] = sa.w.q; }
        else warp_reduce_to_slab<D, APF>(sa, sx, mom, rec, lane);
    };
    // software pipeline (1-D states): the inputs of the next iteration -- of this slab, or of the slab the warp
    // takes next -- are requested before the current iteration's arithmetic starts (77.5 vs 80.8 us at 512
    // threads; at 768 threads / 80 registers it spills: 120 us)
    constexpr bool PREF = (D == 1);
    // FUSED: every iteration runs step t and then step t + 1 on the values step t has just stored -- exactly what
    // the unfused step t + 1 would load -- with the same slabs, lanes and batches, so both steps' records and
    // partial rows carry the bits of two separate launches.  Step t + 1's records go to the CTA's slice of
    // fuse_slab (the shared-memory buffer holds step t's).  In place: step t + 1 writes buffers [(t+1) & 1] =
    // [(t-1) & 1], the pass's input.  Every element is read once, by the thread that later overwrites it, and its
    // store depends on that load, so no thread ever reads a value another thread wrote; these loads therefore go
    // through plain pointers (no __restrict__, no non-coherent loads).
    // (no prefetch in a fused pair: its two steps of arithmetic per load cover the load latency, and the
    // registers of a prefetched iteration would spill)
    constexpr bool PF = PREF && !FUSED;
    const StepIo io1 = FUSED ? step_io(a, io0.t + 1, NZ) : io0;
    const double *Xs = FUSED ? a.X[e.cur] : Xi;
    const double *lws = FUSED ? a.lw[e.cur] : lwi;
    const double *Xs_c = FUSED ? Xs + 2 * pstart : Xi_c;
    const double *lws_c = FUSED ? lws + 2 * pstart : lwi_c;
    double *const slab1 = FUSED ? a.fuse_slab + (size_t)blockIdx.x * StepCfg<M>::kSlabDoubles : nullptr;
    int sl = grab();
    In pre;
    bool have = false;
    if (PF && sl < n_slab && fast_ok && first_it(sl) < n_full) {
        load_full(Xs_c, lws_c, first_it(sl), pre);
        have = true;
    }
    while (sl < n_slab) {
        const int i0 = first_it(sl);
        const int rem = it_small0 - i0;
        const int cnt = sl < n_big ? (rem < slab_it ? rem : slab_it) : 1;
        Acc<D> sa, sb;
        acc_init(sa);
        Lse3 sx = lse3_empty(), sy = lse3_empty();
        if (FUSED) acc_init(sb);
        int nsl = n_slab;
        for (int k_ = 0; k_ < cnt; k_++) {
            const int i = i0 + k_;
            In cin;
            const bool cur_have = have;
            if (PF && have) cin = pre;
            int inext = -1;
            if (k_ + 1 < cnt) inext = i + 1;
            else { nsl = grab(); if (nsl < n_slab) inext = first_it(nsl); }
            have = false;
            if (PF && inext >= 0 && fast_ok && inext < n_full) { load_full(Xs_c, lws_c, inext, pre); have = true; }
            const bool full = fast_ok && i < n_full;
            if (!(PF && cur_have)) {
                if (full) load_full(Xs_c, lws_c, i, cin);
                else load_general(Xs, lws, i, cin);
            }
            double l[2 * kU], x[2 * kU][D];
            if (full) compute_full(io0, i, cin, sa, sx, l, x);
            else compute_general(io0, i, cin, sa, sx, l, x);
            if (FUSED) {
                In nx;
#pragma unroll
                for (int u = 0; u < kU; u++) {
#pragma unroll
                    for (int j2 = 0; j2 < 2; j2++) {
                        nx.base[u][j2] = l[2 * u + j2];
#pragma unroll
                        for (int c = 0; c < D; c++) nx.xp[u][j2][c] = x[2 * u + j2][c];
                    }
                    // the odd last particle: load_general's (unused) base of the missing partner
                    if (!full && 2 * (pstart + (int64_t)i * kIt + u * 32 + lane) + 1 == n) nx.base[u][1] = 0.0;
                }
                if (full) compute_full(io1, i, nx, sb, sy, l, x);
                else compute_general(io1, i, nx, sb, sy, l, x);
            }
        }
        park(s_stage + (size_t)sl * a.slab_stride, sa, sx);
        if (FUSED) park(slab1 + (size_t)sl * a.slab_stride, sb, sy);
        sl = nsl;
    }
    return n_slab;
}

// A step the prologue says does not resample: the streaming pass (D = 1 and `fuse`: a fused pair).  A speculating
// shard then collects the peers' statistics (`dec`); if the global test says "resample" after all, the pass is
// discarded and this returns true.
template <class M, int FK>
__device__ __forceinline__ bool stream_step(const M &model, const FilterArgs &a, const StepEnv &e, bool fuse,
                                            bool speculate, PrologueCarry &pc, StepDecision &dec, StepSmem &sh,
                                            double *s_stage, int &n_slab) {
    if constexpr (M::D == 1) {
        n_slab = fuse ? stream_pass<M, FK, true>(model, a, e, sh, s_stage) : stream_pass<M, FK, false>(model, a, e, sh, s_stage);
    } else {
        n_slab = stream_pass<M, FK, false>(model, a, e, sh, s_stage);
    }
    if (!speculate) return false;
    // now the peers' statistics: bookkeeping, and was the guess right?
    __syncthreads();
    dec = prologue_end<FkTraits<FK>::apf, StepCfg<M>::BS>(a, e.io.t, sh, blockIdx.x == 0, true, pc);
    if (!dec.rs) return false;
    // no: discard the pass, take the resampling branch
    n_slab = 0;
    if (threadIdx.x == 0) sh.next = 0;
    __syncthreads();
    return true;
}

// The first half of a resampling step, A = resampling(scheme, aux.W, M=N) (core.py:329-333): the CDF of this CTA's
// range -- with the ancestor hints scattered to A when a counting scheme resamples locally -- the multinomial
// spacings, and the grid barrier after which every CTA may read the whole CDF.
template <class M, int FK, int SCHEME>
__device__ __forceinline__ void resample_scan(const M &model, const FilterArgs &a, const StepEnv &e,
                                              const StepDecision &dec, double u_sys, StepSmem &sh, double *s_stage,
                                              double *s_warp) {
    constexpr int BS = StepCfg<M>::BS, kStage = StepCfg<M>::kStage;
    constexpr int kBarriers = (SCHEME == SMCB_RS_MULTINOMIAL) ? 2 : 1;     // grid barriers per resampling step
    const int64_t n = e.n, pstart = e.pstart, pend = e.pend;
    unsigned long long bar_target = (unsigned long long)gridDim.x * ((unsigned long long)dec.nrs_prev * kBarriers);
    constexpr bool kCount = (SCHEME != SMCB_RS_MULTINOMIAL);      // offspring counting (local resampling only)
    const bool count_path = kCount && !a.rs_global;
    {
        LoadWeights<M, FK> load;
        load.lw = a.lw[e.cur];
        load.X = a.X[e.cur];
        load.ntot = n;
        load.m = dec.xm;
        load.s = dec.xs;
        load.model = model;
        load.kprev = e.kprev;
        const int64_t e1 = 2 * pend < n ? 2 * pend : n;
        if (count_path) {
            Scatter sc{a.A, (double)n, (SCHEME == SMCB_RS_SYSTEMATIC) ? u_sys : 0.0, (long long)n};
            if (threadIdx.x == 0) sh.timeout_ptr = a.sync_timeout;
            scan_scatter_groups<BS, kScanGroupWarps>(load, 2 * pstart, e1, dec.p_b, dec.p_next, a.cdf, sc,
                                                     blockIdx.x == gridDim.x - 1, sh, reinterpret_cast<int *>(s_stage),
                                                     4 * kStage);
        } else {
            scan_range<BS>(load, 2 * pstart, e1, dec.p_b, dec.p_next, a.cdf, s_warp);
        }
    }
    if (SCHEME == SMCB_RS_MULTINOMIAL) {
        spacings_pass1<BS>(a, e.io.t, sh);
        bar_target += gridDim.x;
        grid_barrier(a, bar_target);
        spacings_pass2<BS>(a, sh, s_warp);
    }
    bar_target += gridDim.x;
    grid_barrier(a, bar_target);
}

// the shared tail of the move passes: gather the ancestors' states (Xp = X[A]), restart the weights (reset_weights),
// write A, propagate and reweight pair p
template <class M, int FK>
__device__ __forceinline__ void finish_pair(const M &model, const FilterArgs &a, const StepEnv &e, double reset_c,
                                            Acc<M::D> &acc, Lse3 &aux, int64_t p, const double *X0, const double *X1,
                                            int64_t a0, int64_t a1, long long g0, long long g1, bool write_A = true) {
    constexpr bool APF = FkTraits<FK>::apf;
    constexpr int D = M::D, NZ = M::NZ;
    const int64_t n = e.n;
    double *__restrict__ Xo = e.io.Xo;
    double *__restrict__ lwo = e.io.lwo;
    double xp[2][D], base[2], x[2][D];
#pragma unroll
    for (int c = 0; c < D; c++) {                // Xp = X[A], component-wise (SoA)
        xp[0][c] = __ldg(X0 + (size_t)c * n + a0);
        xp[1][c] = __ldg(X1 + (size_t)c * n + a1);
    }
    if (APF) {   // core.py:302: lw = log_mean_exp(logetat, W) - logetat[A]
        base[0] = reset_c - model_logeta<M>(model, e.kprev, xp[0]);
        base[1] = reset_c - model_logeta<M>(model, e.kprev, xp[1]);
    } else {     // Weights() then add(delta): lw = 0 + delta (shard mass if sharded)
        base[0] = reset_c; base[1] = reset_c;
    }
    if (write_A) {
        if (2 * p + 1 < n) *reinterpret_cast<longlong2 *>(a.A + 2 * p) = make_longlong2(g0, g1);
        else a.A[2 * p] = g0;
    }
    double l[2], av[2];
    if (e.io.zin == nullptr && e.vec_x && 2 * p + 1 < n) {       // complete pair, device normals: no bounds tests
        double z[2][NZ];
        tab_normals<NZ>(a.key, (uint64_t)((a.index_offset >> 1) + p), (uint32_t)e.io.t, z);
        const bool odd = move_pair<M, FK, false>(model, e.io.k, xp, base, z, APF && e.io.last_apf, x, l, av);
#pragma unroll
        for (int c = 0; c < D; c++) st2(Xo + (size_t)c * n + 2 * p, x[0][c], x[1][c]);
        st2(lwo + 2 * p, l[0], l[1]);
        if (!odd) acc_add_batch<2, D, true>(acc, l, x, e.mom);
        else acc_add_batch<2, D, false>(acc, l, x, e.mom);
    } else {
        do_pair<M, FK>(model, a, e.io, n, e.vec_x, p, xp, base, x, l, av);
        acc_add_batch<2, D>(acc, l, x, e.mom);
    }
    if (APF) lse3_add_batch<2>(aux, av);
}

// the exact answer of np.searchsorted(cdf, su, 'left') from any starting point a0: gallop to a bracket, then bisect
// (O(log distance) loads)
__device__ __forceinline__ long long settle(const double *cdf, int64_t n, long long a0, double su) {
    a0 = a0 < 0 ? 0 : (a0 > n - 1 ? n - 1 : a0);
    long long lo_, hi_;                                  // answer in [lo_, hi_]: cdf[lo_-1] < su, cdf[hi_] >= su or hi_ = n-1
    if (__ldcg(cdf + a0) < su) {                         // go up
        long long step = 1;
        lo_ = a0 + 1;
        hi_ = a0 + 1;
        while (hi_ < n - 1 && __ldcg(cdf + hi_) < su) { lo_ = hi_ + 1; hi_ += step; step <<= 1; }
        if (hi_ > n - 1) hi_ = n - 1;
    } else {                                             // go down
        long long step = 1;
        hi_ = a0;
        lo_ = a0 - 1;
        while (lo_ >= 0 && __ldcg(cdf + lo_) >= su) { hi_ = lo_; lo_ -= step; step <<= 1; }
        lo_ = lo_ < 0 ? 0 : lo_ + 1;
    }
    while (lo_ < hi_) {                                  // first j in [lo_, hi_] with cdf[j] >= su
        const long long mid = lo_ + ((hi_ - lo_) >> 1);
        if (__ldcg(cdf + mid) < su) lo_ = mid + 1; else hi_ = mid;
    }
    return lo_;
}

// Move pass of the counting schemes (local resampling): every output verifies the scattered ancestor against the
// exact su_k (cdf[a-1] < su_k <= cdf[a], i.e. np.searchsorted's answer), walks if the hint is off, then gathers,
// propagates and reweights.  No tiles, no block barriers: a pair per thread, strided over the CTA's range.
template <class M, int FK, int SCHEME>
__device__ __forceinline__ void move_counted(const M &model, const FilterArgs &a, const StepEnv &e, double reset_c,
                                             double u_sys, const double *uin, Acc<M::D> &acc, Lse3 &aux) {
    constexpr int BS = StepCfg<M>::BS;
    const long long t = e.io.t;
    const int64_t n = e.n, pstart = e.pstart, pend = e.pend;
    const double *__restrict__ Xi = a.X[e.cur];
    const double M_ = (double)n;
    constexpr int kR = kMovePairs;                          // pairs in flight per thread
    // one round = kR pairs per thread, in three parts: the hints (A, written by the scan), the CDF entries that
    // verify them, and verify + repair + gather + propagate
    struct Hints { long long h[kR][2]; };
    struct Cdf { double c0[kR][2], cm[kR][2], c1[kR][(SCHEME == SMCB_RS_STRATIFIED) ? 2 : 1]; };
    auto ld_hints = [&](int64_t p0, Hints &H) {
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int64_t p = p0 + (int64_t)r * BS;
            H.h[r][0] = H.h[r][1] = 0;
            if (p < pend && 2 * p + 1 < n) {
                const longlong2 hh = __ldcg(reinterpret_cast<const longlong2 *>(a.A + 2 * p));
                H.h[r][0] = hh.x; H.h[r][1] = hh.y;
            } else if (p < pend) {
                H.h[r][0] = __ldcg(a.A + 2 * p);
            }
        }
    };
    auto ld_cdf = [&](int64_t p0, const Hints &H, Cdf &Cc) {
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int64_t p = p0 + (int64_t)r * BS;
#pragma unroll
            for (int q = 0; q < 2; q++) {                    // the two CDF entries that decide the hint
                long long hh = H.h[r][q];
                hh = hh < 0 ? 0 : (hh > n - 1 ? n - 1 : hh);
                const bool on = (p < pend) && (q == 0 || 2 * p + 1 < n);
                // (plain loads: this SM touches these lines for the first time in this launch, after the grid
                // barrier, so L1 cannot hold an older copy -- and neighbouring outputs reuse them)
                Cc.c0[r][q] = on ? a.cdf[hh] : 2.0;
                Cc.cm[r][q] = (on && hh > 0) ? a.cdf[hh - 1] : -1.0;
                // stratified: the hint answers k / N and su_k lies up to 1 / N further, so about half of the
                // outputs belong to the NEXT entry -- fetch it with the other two instead of walking
                if (SCHEME == SMCB_RS_STRATIFIED) Cc.c1[r][q] = (on && hh + 1 < n) ? a.cdf[hh + 1] : 2.0;
            }
        }
    };
    auto process = [&](int64_t p0, const Hints &H, const Cdf &Cc) {
        long long h[kR][2];
        double su[kR][2];
        bool valid[kR], two[kR], moved[kR];
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int64_t p = p0 + (int64_t)r * BS;
            moved[r] = false;
            valid[r] = p < pend;
            two[r] = valid[r] && (2 * p + 1 < n);
            grid_pair<SCHEME>(u_sys, a.key, (uint64_t)((a.index_offset >> 1) + p), (uint32_t)t, uin, p, valid[r],
                              two[r], M_, su[r][0], su[r][1]);
#pragma unroll
            for (int q = 0; q < 2; q++) {
                long long hh = H.h[r][q];
                hh = hh < 0 ? 0 : (hh > n - 1 ? n - 1 : hh);
                moved[r] = moved[r] || hh != H.h[r][q];
                h[r][q] = hh;
            }
        }
#pragma unroll
        for (int r = 0; r < kR; r++) {
#pragma unroll
            for (int q = 0; q < 2; q++) {
                const bool on = q == 0 ? valid[r] : two[r];
                bool ok = (Cc.cm[r][q] < su[r][q]) && (su[r][q] <= Cc.c0[r][q] || h[r][q] == n - 1);
                if (SCHEME == SMCB_RS_STRATIFIED) {
                    if (on && !ok && Cc.c0[r][q] < su[r][q] && (su[r][q] <= Cc.c1[r][q] || h[r][q] + 1 == n - 1)) {
                        h[r][q] += 1; moved[r] = true; ok = true;
                    }
                }
                if (on && !ok && Cc.c0[r][q] < su[r][q] && h[r][q] + 1 < n) {
                    // the hint is too low: ONE round trip for the next kWin entries (independent loads, mostly
                    // one line) instead of a chain of dependent ones; the search below only runs past them
                    constexpr int kWin = 6;
                    const long long b = h[r][q] + 1;
                    double wv[kWin];
#pragma unroll
                    for (int i = 0; i < kWin; i++) wv[i] = (b + i < n) ? __ldcg(a.cdf + b + i) : 2.0;
                    int cnt = 0;
#pragma unroll
                    for (int i = 0; i < kWin; i++) cnt += (wv[i] < su[r][q]) ? 1 : 0;   // monotone CDF: a prefix
                    if (cnt < kWin) {
                        long long hn = b + cnt;
                        h[r][q] = hn > n - 1 ? n - 1 : hn;
                        moved[r] = true; ok = true;
                    }
                }
                if (on && !ok) {
                    h[r][q] = settle(a.cdf, n, h[r][q], su[r][q]);
                    moved[r] = true;
                }
            }
            if (!two[r]) h[r][1] = h[r][0];
        }
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int64_t p = p0 + (int64_t)r * BS;
            if (valid[r]) finish_pair<M, FK>(model, a, e, reset_c, acc, aux, p, Xi, Xi, h[r][0], h[r][1], h[r][0], h[r][1],
                                             moved[r]);
        }
    };
    constexpr int64_t kStep = (int64_t)kR * BS;
    for (int64_t p0 = pstart + threadIdx.x; p0 < pend; p0 += kStep) {
        Hints H;
        Cdf Cc;
        ld_hints(p0, H);
        ld_cdf(p0, H, Cc);
        process(p0, H, Cc);
    }
}

// Move pass of the multinomial scheme (local resampling; every other scheme counts offspring when it resamples
// locally): per tile of 2 BS outputs, the CDF slice their ancestors lie in is staged in shared memory by one TMA bulk
// copy (double-buffered) and searched there.
template <class M, int FK>
__device__ __forceinline__ void move_tiles(const M &model, const FilterArgs &a, const StepEnv &e, double reset_c,
                                           Acc<M::D> &acc, Lse3 &aux, double *s_stage, double *s_su, uint64_t *s_bar,
                                           long long &s_hi) {
    constexpr int BS = StepCfg<M>::BS, kStage = StepCfg<M>::kStage;
    const int64_t n = e.n, pstart = e.pstart, pend = e.pend;
    const double *__restrict__ Xi = a.X[e.cur];
    const double zlast = __ldcg(a.su + n);
    int64_t lo = -1;
    if (threadIdx.x == 0) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_init_fence(); }
    __syncthreads();
    uint32_t phase0 = 0, phase1 = 0;
    int buf = 0;
    // thread 0: bring cdf[sb, sb + c) into buffer b (sb = lo_ rounded down to even => 16-byte aligned)
    // by ONE TMA bulk copy (cp.async.bulk + mbarrier); the slice of tile i+1 is in flight while tile i
    // propagates and reweights
    auto issue = [&](int64_t lo_, int b) {
        const int64_t sb = lo_ & ~(int64_t)1;
        const int c = (int)((n - sb) < kStage ? (n - sb) : kStage);
        const uint32_t bytes = (uint32_t)(c & ~1) * 8u;
        double *dst = s_stage + (size_t)b * kStage;
        if (c & 1) dst[c - 1] = __ldcg(a.cdf + sb + c - 1);      // odd tail (n odd, end of the array)
        if (bytes) {
            mbar_arrive_expect_tx(&s_bar[b], bytes);
            tma_bulk_g2s(dst, a.cdf + sb, bytes, &s_bar[b]);
        } else {
            mbar_arrive(&s_bar[b]);
        }
    };
    for (int64_t pbase = pstart; pbase < pend; pbase += BS) {
        const int64_t p = pbase + threadIdx.x;
        const bool active = p < pend;
        const int64_t k0 = 2 * pbase;                                       // first / last output of the tile
        const int64_t ptop = pbase + BS < pend ? pbase + BS : pend;
        const int64_t k1 = (2 * ptop < n ? 2 * ptop : n) - 1;
        double su[2] = {2.0, 2.0};
        if (active) {
            su[0] = __ldcg(a.su + 2 * p) / zlast;                   // resampling.py:537
            su[1] = (2 * p + 1 < n) ? __ldcg(a.su + 2 * p + 1) / zlast : 2.0;
            if (2 * p == k0) s_su[0] = su[0];
            if (2 * p == k1) s_su[1] = su[0];
            if (2 * p + 1 == k1) s_su[1] = su[1];
        }
        __syncthreads();
        const double su_first = s_su[0], su_last = s_su[1];
        if (lo < 0) {                                      // first tile of this block
            lo = block_lower_bound<BS>(a.cdf, 0, n, su_first);
            lo = lo < n - 1 ? lo : n - 1;
            if (threadIdx.x == 0) issue(lo, buf);
            __syncthreads();
        }
        // su is sorted, so the slice starts at `lo`
        const int64_t sbase = lo & ~(int64_t)1;
        const int cnt = (int)((n - sbase) < kStage ? (n - sbase) : kStage);
        mbar_wait(&s_bar[buf], buf ? phase1 : phase0);
        if (buf) phase1 ^= 1u; else phase0 ^= 1u;
        const double *s_cdf = s_stage + (size_t)buf * kStage;
        const bool covered = (sbase + cnt >= n) || (s_cdf[cnt - 1] >= su_last);
        int64_t hi = lo;
        if (!covered) hi = block_lower_bound<BS>(a.cdf, lo, n, su_last);   // rare: sparse mass
        int64_t a0 = 0, a1 = 0;
        if (active) {
            if (covered) {
                int l0, l1;
                tile_search(s_cdf, (int)(lo - sbase), cnt, su[0], su[1], l0, l1);
                a0 = sbase + l0;
                a1 = sbase + l1;
                if (2 * p == k1) s_hi = a0;
                if (2 * p + 1 == k1) s_hi = a1;
            } else {
                const int64_t hi1 = hi < n ? hi + 1 : n;
                a0 = lower_bound_cg(a.cdf, lo, hi1, su[0]);
                a1 = lower_bound_cg(a.cdf, a0, hi1, su[1]);
            }
        }
        __syncthreads();                                   // s_hi published; buffer buf^1 is free
        const int64_t lo_next = covered ? (s_hi < n ? s_hi : n - 1) : (hi < n ? hi : n - 1);
        if (pbase + BS < pend && threadIdx.x == 0) issue(lo_next, buf ^ 1);
        if (active) {
            a0 = a0 < n - 1 ? a0 : n - 1;
            a1 = a1 < n - 1 ? a1 : n - 1;
            finish_pair<M, FK>(model, a, e, reset_c, acc, aux, p, Xi, Xi, a0, a1, a0, a1);
        }
        lo = lo_next;
        buf ^= 1;
    }
}

// Move pass of the exact global resampling over particle shards (SURVEY.md section 8e, mode 2; resampling.py:599-610
// applied to the concatenation of all shards).  Output j of rank r is global offspring index_offset + j: its grid
// point su is located in the global CDF in two levels -- shard k with goff[k] <= su < goff[k+1] (offsets from the
// exchanged statistics, identical bits on every rank), then v = (su - goff[k]) / gpi[k] in shard k's own normalised
// CDF, read over NVLink -- and the ancestor's state is pulled from shard k's particle buffer.
template <class M, int FK, int SCHEME>
__device__ __forceinline__ void move_global(const M &model, const FilterArgs &a, const StepEnv &e, double reset_c,
                                            double u_sys, const double *uin, Acc<M::D> &acc, Lse3 &aux, StepSmem &sh,
                                            double *s_stage, double *s_su, long long &s_hi) {
    constexpr int BS = StepCfg<M>::BS, kStage = StepCfg<M>::kStage;
    const long long t = e.io.t;
    const int cur = e.cur;
    const int64_t n = e.n, pstart = e.pstart, pend = e.pend;
    // First: tell every peer that this shard's CDF of step t is complete, and wait for theirs.
    if (blockIdx.x == 0 && (int)threadIdx.x < a.world) {
        __threadfence_system();
        double *slot = a.mail_peer[threadIdx.x] + ((size_t)(t & 1) * a.world + a.rank) * kMailStride;
        *reinterpret_cast<volatile double *>(slot + kMailScan) = (double)(t + 1);
    }
    if ((int)threadIdx.x < a.world)
        wait_epoch(a.mail_local + ((size_t)(t & 1) * a.world + threadIdx.x) * kMailStride + kMailScan,
                   (double)(t + 1), a.sync_timeout);
    __syncthreads();
    const int world = a.world;
    const double M_ = (double)a.n_global;
    double *s_cdf = s_stage;
    int64_t lo = -1;
    int lo_shard = -1;
    for (int64_t pbase = pstart; pbase < pend; pbase += BS) {
        const int64_t p = pbase + threadIdx.x;
        const bool active = p < pend;                               // sharded filters have even n
        const int64_t k0 = 2 * pbase;
        const int64_t ptop = pbase + BS < pend ? pbase + BS : pend;
        const int64_t k1 = 2 * ptop - 1;
        double su[2] = {2.0, 2.0};
        if (active) {
            const double g0 = (double)(a.index_offset + 2 * p);
            if (SCHEME == SMCB_RS_SYSTEMATIC) {
                su[0] = (u_sys + g0) / M_;
                su[1] = (u_sys + (g0 + 1.0)) / M_;
            } else {
                double u0, u1;
                if (uin) { u0 = uin[2 * p]; u1 = uin[2 * p + 1]; }
                else uniform_pair(a.key, (uint64_t)((a.index_offset >> 1) + p), (uint32_t)t, kPurposeUniform, u0, u1);
                su[0] = (u0 + g0) / M_;
                su[1] = (u1 + (g0 + 1.0)) / M_;
            }
            if (2 * p == k0) s_su[0] = su[0];
            if (2 * p + 1 == k1) s_su[1] = su[1];
        }
        __syncthreads();
        const double su_first = s_su[0], su_last = s_su[1];
        const int kf = shard_of(sh.goff, sh.gpi, world, su_first);
        const int kl = shard_of(sh.goff, sh.gpi, world, su_last);
        int ks[2] = {kf, kf};
        int64_t an[2] = {0, 0};
        if (kf == kl) {
            // the whole tile draws from one shard: staged search on that shard's CDF with the grid
            // points mapped into its local scale
            const double *cdf = a.pcdf[kf];
            const double off = sh.goff[kf], pi = sh.gpi[kf];
            const double v0 = fmin((su[0] - off) / pi, 1.0), v1 = fmin((su[1] - off) / pi, 1.0);
            const double v_first = fmin((su_first - off) / pi, 1.0), v_last = fmin((su_last - off) / pi, 1.0);
            if (lo < 0 || lo_shard != kf) lo = block_lower_bound<BS>(cdf, 0, n, v_first);
            if (lo > n - 1) lo = n - 1;
            lo_shard = kf;
            const int64_t sbase = lo & ~(int64_t)1;
            const int cnt = (int)((n - sbase) < kStage ? (n - sbase) : kStage);
            for (int i = 2 * threadIdx.x; i < cnt; i += 2 * BS) {
                if (i + 1 < cnt) *reinterpret_cast<double2 *>(&s_cdf[i]) = __ldcg(reinterpret_cast<const double2 *>(cdf + sbase + i));
                else s_cdf[i] = __ldcg(cdf + sbase + i);
            }
            __syncthreads();
            const bool covered = (sbase + cnt >= n) || (s_cdf[cnt - 1] >= v_last);
            int64_t hi = lo;
            if (!covered) hi = block_lower_bound<BS>(cdf, lo, n, v_last);
            if (active) {
                if (covered) {
                    int l0, l1;
                    tile_search(s_cdf, (int)(lo - sbase), cnt, v0, v1, l0, l1);
                    an[0] = sbase + l0;
                    an[1] = sbase + l1;
                    if (2 * p + 1 == k1) s_hi = an[1];
                } else {
                    const int64_t hi1 = hi < n ? hi + 1 : n;
                    an[0] = lower_bound_cg(cdf, lo, hi1, v0);
                    an[1] = lower_bound_cg(cdf, an[0], hi1, v1);
                }
            }
            __syncthreads();
            lo = covered ? (s_hi < n ? s_hi : n - 1) : (hi < n ? hi : n - 1);
        } else {
            // the tile straddles a shard boundary (at most world - 1 tiles per rank): plain searches
            if (active) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    ks[j] = shard_of(sh.goff, sh.gpi, world, su[j]);
                    const double v = fmin((su[j] - sh.goff[ks[j]]) / sh.gpi[ks[j]], 1.0);
                    an[j] = lower_bound_cg(a.pcdf[ks[j]], 0, n, v);
                }
            }
            lo = -1;
        }
        if (active) {
            const int64_t a0 = an[0] < n - 1 ? an[0] : n - 1, a1 = an[1] < n - 1 ? an[1] : n - 1;
            // ancestors are GLOBAL particle indices
            finish_pair<M, FK>(model, a, e, reset_c, acc, aux, p, a.pX[ks[0]][cur], a.pX[ks[1]][cur], a0, a1,
                               (long long)ks[0] * n + a0, (long long)ks[1] * n + a1);
        }
        __syncthreads();       // s_su / s_hi / s_cdf are rewritten by the next tile
    }
}

// ---------------------------------------------------------------------------
// the step kernel: resample_move + reweight_particles (+ compute_summaries of the previous step)
// (core.py:323-367)
// ---------------------------------------------------------------------------
template <class M, int FK, int SCHEME>
__global__ void __launch_bounds__(StepCfg<M>::BS, 1) k_step(M model, FilterArgs a, long long t) {
    constexpr bool APF = FkTraits<FK>::apf;
    constexpr int D = M::D, NZ = M::NZ, BS = StepCfg<M>::BS;
    extern __shared__ __align__(128) double s_dyn[];    // math tables | [2][kStage] CDF slices (resampling branch)
    double *const s_stage = s_dyn + kMathTabDoubles;
    __shared__ StepSmem sh;
    __shared__ double s_su[2];
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ __align__(8) uint64_t s_tabbar;
    __shared__ long long s_hi;
    __shared__ double s_warp[BS / 32];
    // the tables are constants: their copy may start before the previous kernel has retired
    if (threadIdx.x == 0) { mtab_issue(a.math_tab, &s_tabbar); sh.next = 0; }
    // everything below reads what the previous kernel of the stream wrote (programmatic dependent launch:
    // this kernel may have been scheduled before its predecessor retired)
    cudaGridDependencySynchronize();
    cudaTriggerProgrammaticLaunchCompletion();
    // Sharded filters with the mailbox exchange SPECULATE: a step whose shard-local ESS test says "no resampling"
    // starts its streaming pass at once and collects the peers' statistics afterwards -- the exchange latency (peer's
    // step end + NVLink store + fence + poll) leaves the critical path.  The pass writes only the other half of the
    // ping-pong buffers, so a wrong guess (global test says "resample": only within sampling noise of the threshold)
    // costs one discarded pass and nothing else.
    PrologueCarry pc;
    const bool pred_rs = prologue_begin<APF>(a, t, sh, blockIdx.x == 0, pc);
    // (not with the exact global resampling: there the peers pull ancestors out of THIS rank's previous generation
    // during their resampling step, and waiting for their end-of-step statistics is what keeps that buffer intact)
    const bool speculate = SMCB_SPECULATE && a.world > 1 && a.mail_local != nullptr && !a.rs_global && !pred_rs;
    StepDecision dec;
    dec.rs = 0; dec.nrs_prev = 0; dec.reset_c = 0.0; dec.xm = 0.0; dec.xs = 1.0; dec.p_b = 0.0; dec.p_next = 0.0;
    dec.ess = 0.0;
    if (!speculate) dec = prologue_end<APF, BS>(a, t, sh, blockIdx.x == 0, true, pc);
    // (no block barrier on the speculative path: CTA 0's sending lanes sit in their system-scope fence for a few
    // microseconds, and the other warps of that CTA start on the slabs meanwhile -- the dynamic slab schedule absorbs it)
    mbar_wait(&s_tabbar, 0);                           // (the prologue's barriers made the init visible)
    const int cur = (int)((t - 1) & 1);                // step s writes buffers [s & 1]
    const bool rs = dec.rs != 0;                       // (a speculative step enters the resampling branch from below)
    if (a.fuse_mode != 0 && __ldcg(a.fuse) == t) {
        // the previous launch ran this step as the second half of a fused pair.  Its x_t, lw_t and partial rows
        // are in place unless step t resamples after all: then the resampling branch below overwrites them from
        // buffers [(t-1) & 1], which the fused pass left intact.
        if (blockIdx.x == 0 && threadIdx.x == 0) a.fuse[rs ? 3 : 2] += 1;
        if (!rs) return;
    }
    // Fuse step t + 1 into this streaming pass?  Only if the host has enqueued it in this batch (a caller that stops
    // after step t reads Xp from buffers [(t-1) & 1]), and -- a step t + 1 that resamples discards the speculative
    // half -- if the ESS extrapolated from steps t - 2 and t - 1 stays above the threshold.  Every CTA decides
    // alike (the prologue's ESS has the same bits everywhere); the choice changes the speed, never the results.
    bool fuse = false;
    if (D == 1 && !rs && a.fuse_mode != 0 && a.world == 1 && t + 1 < a.T && t + 1 < a.batch_end) {
        const double ess2 = (t >= 2) ? __ldcg(&a.st[(t - 2) & 1].ess) : dec.ess;
        fuse = a.fuse_mode == 2 || 2.0 * dec.ess - ess2 >= (double)a.n_global * a.essrmin;
    }
    if (fuse && blockIdx.x == 0 && threadIdx.x == 0) { a.fuse[0] = t + 1; a.fuse[1] += 1; }
    StepEnv e;
    e.io = step_io(a, t, NZ);
    e.kprev = step_consts(a, t - 1);
    e.cur = cur;
    e.n = a.n;
    e.vec_x = (D == 1) || ((a.n & 1) == 0);
    e.mom = a.moments != nullptr;
    cta_range(a, e.pstart, e.pend);

    Acc<D> acc;
    acc_init(acc);
    Lse3 aux = lse3_empty();
    int n_slab = 0;                                    // slab records of the streaming pass
    // the resampling branch: A = resampling(scheme, aux.W, M=N); Xp = X[A]; reset_weights (core.py:329-333).  (One
    // short-circuit condition on purpose: a "resample" flag set in both branches and tested after them costs the
    // bootstrap kernels about 150 more bytes of spills at the 128-register cap.)
    if (rs || stream_step<M, FK>(model, a, e, fuse, speculate, pc, dec, sh, s_stage, n_slab)) {
        const double *uin = a.u_in ? a.u_in + (size_t)t * (a.n + 1) : nullptr;
        const double u_sys = (SCHEME == SMCB_RS_SYSTEMATIC) ? systematic_u(a.key, t, uin) : 0.0;
        resample_scan<M, FK, SCHEME>(model, a, e, dec, u_sys, sh, s_stage, s_warp);
        if (SCHEME != SMCB_RS_MULTINOMIAL && !a.rs_global)
            move_counted<M, FK, SCHEME>(model, a, e, dec.reset_c, u_sys, uin, acc, aux);
        else if (SCHEME == SMCB_RS_MULTINOMIAL && !a.rs_global)
            move_tiles<M, FK>(model, a, e, dec.reset_c, acc, aux, s_stage, s_su, s_bar, s_hi);
        else
            move_global<M, FK, SCHEME>(model, a, e, dec.reset_c, u_sys, uin, acc, aux, sh, s_stage, s_su, s_hi);
    }
    write_partial<D, APF, BS>(a, t, acc, aux, e.mom, sh, s_stage, n_slab);
    if (fuse)   // (acc, aux: still empty -- the streaming pass keeps its statistics in the slab records)
        write_partial<D, APF, BS>(a, t + 1, acc, aux, e.mom, sh, a.fuse_slab + (size_t)blockIdx.x * StepCfg<M>::kSlabDoubles,
                                  n_slab);
}

// the prologue alone (one CTA): finalises the last enqueued step so that the host can read its summaries
template <bool APF>
__global__ void __launch_bounds__(kTailBlock) k_tail(FilterArgs a, long long t) {
    __shared__ StepSmem sh;
    cudaGridDependencySynchronize();
    step_prologue<APF, kTailBlock>(a, t, sh, true, false);
}

// sharded filters with the host-driven exchange (NCCL): this shard's statistics of step s -> local_stats
template <bool APF>
__global__ void __launch_bounds__(kTailBlock) k_publish(FilterArgs a, long long s) {
    __shared__ StepSmem sh;
    double loc[16];
    shard_totals<APF>(a, s, true, sh, loc);
    if (threadIdx.x == 0)
        for (int i = 0; i < 16; i++) a.local_stats[i] = loc[i];
}

}  // namespace smcb

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
struct smcb_filter {
    smcb_ctx *ctx;
    smcb_filter_desc desc;
    FilterArgs args;
    char *mem;            // header (StepState[2], barrier, timeout flag) + partials + block aggregates
    int grid_move;        // CTAs of the step kernel: one per SM (fewer for tiny N)
    int block_size;       // threads per CTA of the step kernel
    size_t dyn_smem;      // its dynamic shared memory (math tables, CDF staging buffers, slab records)
    int slab_doubles;     // doubles of shared memory for the slab records
    int pairs_per_iteration;  // work unit of a warp in the streaming branch
    int64_t t_host;       // steps launched so far (the device needs no other notion of time)
    bool pdl, coop;       // launch attributes in use (programmatic dependent launch, cooperative)
    bool timed;           // inside smcb_filter_step_timed: plain serialised launches
    int (*launch_init)(smcb_filter *);
    int (*launch_step)(smcb_filter *);
    int (*launch_tail)(smcb_filter *);
    int (*launch_publish)(smcb_filter *);
};

template <class... Args>
static int launch_ex(smcb_filter *f, void (*kern)(Args...), int grid, int block, size_t smem, bool coop, bool pdl,
                     Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = f->ctx->stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (coop) { attr[na].id = cudaLaunchAttributeCooperative; attr[na].val.cooperative = 1; na++; }
    if (pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        na++;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    SMCB_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
    f->ctx->launches++;
    return SMCB_OK;
}

template <class M, int FK, int SCHEME>
static int launch_step_t(smcb_filter *f) {
    M model;
    model.load(f->desc.params);
    return launch_ex(f, k_step<M, FK, SCHEME>, f->grid_move, f->block_size, f->dyn_smem, f->coop,
                     f->pdl && !f->timed, model, f->args, (long long)f->t_host);
}

template <class M, int FK>
static int launch_init_t(smcb_filter *f) {
    M model;
    model.load(f->desc.params);
    k_init<M, FK><<<f->grid_move, f->block_size, kMathTabBytes, f->ctx->stream>>>(model, f->args);
    f->ctx->launches++;
    SMCB_CUDA(cudaGetLastError());
    return SMCB_OK;
}

template <int FK>
static int launch_tail_t(smcb_filter *f) {
    return launch_ex(f, k_tail<FkTraits<FK>::apf>, 1, kTailBlock, 0, false, f->pdl && !f->timed, f->args,
                     (long long)f->t_host);
}

template <int FK>
static int launch_publish_t(smcb_filter *f) {
    k_publish<FkTraits<FK>::apf><<<1, kTailBlock, 0, f->ctx->stream>>>(f->args, (long long)(f->t_host - 1));
    f->ctx->launches++;
    SMCB_CUDA(cudaGetLastError());
    return SMCB_OK;
}

template <class M, int FK, int SCHEME>
static int bind_one(smcb_filter *f) {
    f->launch_init = launch_init_t<M, FK>;
    f->launch_step = launch_step_t<M, FK, SCHEME>;
    f->launch_tail = launch_tail_t<FK>;
    f->launch_publish = launch_publish_t<FK>;
    f->block_size = StepCfg<M>::BS;
    f->dyn_smem = StepCfg<M>::dyn_smem;
    f->slab_doubles = StepCfg<M>::kSlabDoubles;
    f->pairs_per_iteration = 32 * StepCfg<M>::kU;
    SMCB_CUDA(cudaFuncSetAttribute(k_step<M, FK, SCHEME>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)StepCfg<M>::dyn_smem));
    SMCB_CUDA(cudaFuncSetAttribute(k_init<M, FK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMathTabBytes));
    int nb = 0;
    SMCB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_step<M, FK, SCHEME>, StepCfg<M>::BS,
                                                            StepCfg<M>::dyn_smem));
    if (nb < 1) {
        set_error("fused filter: the step kernel does not fit on an SM of this device");
        return SMCB_ECUDA;
    }
    return SMCB_OK;
}

template <class M, int FK>
static int bind_scheme(smcb_filter *f) {
    bool fused = false;
    const int rc = with_scheme(f->desc.scheme, [&](auto scheme) {
        fused = true;
        return bind_one<M, FK, decltype(scheme)::value>(f);
    });
    if (!fused)
        set_error("fused filter: resampling scheme %d is not fused (use systematic, stratified or "
                  "multinomial, or the unfused path)", f->desc.scheme);
    return rc;
}

// Binds the kernels of model M.  Each model's kernels are compiled in one translation unit only: smcb_filter.cu
// dispatches on the model id and instantiates StochVol and LinearGauss; the other models' bind_fk<M> are declared
// extern template there and instantiated explicitly in smcb_filter_1d.cu and smcb_filter_nd.cu.
template <class M>
int bind_fk(smcb_filter *f) {
    if (f->desc.fk < SMCB_FK_BOOTSTRAP || f->desc.fk > SMCB_FK_AUXBOOT) {
        set_error("fused filter: unknown Feynman-Kac kind %d", f->desc.fk);
        return SMCB_EINVAL;
    }
    bool offered = false;
    const int rc = with_fk<M>(f->desc.fk, [&](auto fk) {
        offered = true;
        return bind_scheme<M, decltype(fk)::value>(f);
    });
    if (offered) return rc;
    // the reference raises NotImplementedError from StateSpaceModel.proposal / logeta
    set_error("fused filter: model %d implements no proposal/logeta (Feynman-Kac kind %d)",
              f->desc.model, f->desc.fk);
    return SMCB_ENOSYS;
}
