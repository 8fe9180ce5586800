// smcb_hmm.cu -- Baum-Welch forward / backward passes and posterior trajectory draws (particles/hmm.py:150-268) for
// B finite-state HMMs with K <= 128 states:
//   FORWARD    rows [t0, t1) in one launch: pred_t = filt_{t-1} P (sum in j order; init_dist at t = 0),
//              lp = log pred_t + logft_t, logpyt_t = max lp + log sum exp(lp - max), filt_t = exp(lp - logpyt_t);
//   BACKWARD   cost-to-go ctg_k <- LSE_j(log P_kj + logft_{t+1,j} + ctg_j) from t = T-2 down to 0, smth_t =
//              exp_and_normalise(log filt_t + ctg), smth_{T-1} = filt_{T-1};
//   SAMPLE     rows T-2 .. 0 of N trajectories per HMM from the last row the caller drew: a CTA owns a tile of one
//              HMM's trajectories, builds the K column CDFs of x_t | x_{t+1} = j in shared memory once per t and
//              draws #{k : C[j][k] < u} (searchsorted 'left', clipped to K - 1).
// Tiers: K <= 32 runs one warp per HMM (kHmmGroups HMMs per CTA), 33 <= K <= 128 one CTA of ceil(K / 32) warps
// per HMM; the group's transition matrix (or its log, transposed) stays in shared memory for the whole launch.
// Thread k owns state k.  Sums over states: xor butterfly inside a warp, then the warp partials in warp order, so
// the bits depend on the inputs only; sums over j inside one thread run in j order.  exp is the smoothing kernels'
// fexp_neg, log the CUDA fp64 log, and the library is compiled with -fmad=false.
// Randomness (SAMPLE without injected uniforms): Philox keyed by the descriptor's seed, counter (n, t, b,
// kPurposeHmm): the draws do not depend on the tile size or the launch shape.
#include "smcb_math.cuh"
#include "smcb_reduce.cuh"

using namespace smcb;

namespace {

constexpr int kHmmGroups = 4;                  // warp tier: HMMs (one warp each) per CTA
constexpr int kSampleBlock = 256;              // SAMPLE: trajectories per CTA

// The threads that work on one HMM: one warp (kWarp) or the whole CTA.  part: the CTA's warp partials.
template <bool kWarp>
struct Group {
    int nw;
    double *part;

    __device__ __forceinline__ void sync() const {
        if (kWarp) __syncwarp();
        else __syncthreads();
    }
    __device__ __forceinline__ double across_warps(double v, bool is_max) const {
        if (kWarp) return v;
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
        __syncthreads();
        double r = part[0];
        for (int w = 1; w < nw; w++) r = is_max ? fmax(r, part[w]) : r + part[w];
        __syncthreads();
        return r;
    }
    __device__ __forceinline__ double sum(double v) const { return across_warps(warp_sum(v), false); }
    __device__ __forceinline__ double max(double v) const { return across_warps(warp_max(v), true); }
};

// the group of this thread: which HMM, which state, where its shared-memory slab (`per` doubles) starts
template <bool kWarp>
struct Slot {
    int64_t b;
    int k, gi, gs;
    double *base;
};

template <bool kWarp>
__device__ __forceinline__ Slot<kWarp> slot_of(double *smem, int per) {
    Slot<kWarp> s;
    if (kWarp) {
        const int g = threadIdx.x >> 5;
        s.b = (int64_t)blockIdx.x * kHmmGroups + g;
        s.k = s.gi = threadIdx.x & 31;
        s.gs = 32;
        s.base = smem + (size_t)g * per;
    } else {
        s.b = blockIdx.x;
        s.k = s.gi = threadIdx.x;
        s.gs = blockDim.x;
        s.base = smem;
    }
    return s;
}

__host__ __device__ __forceinline__ int slab_doubles(int K) { return K * K + 2 * K + 32; }

// ---------------------------------------------------------------------------
// FORWARD -- hmm.py:176-194
// ---------------------------------------------------------------------------
template <bool kWarp>
__global__ void k_hmm_forward(smcb_hmm_desc d) {
    extern __shared__ double smem[];
    const int K = d.K;
    const Slot<kWarp> s = slot_of<kWarp>(smem, slab_doubles(K));
    if (s.b >= d.B) return;                                   // warp tier only: the whole warp leaves
    double *P = s.base, *f = P + K * K;
    const Group<kWarp> grp{(int)(blockDim.x >> 5), f + 2 * K};
    const double *Pg = d.trans + s.b * d.trans_stride;
    for (int i = s.gi; i < K * K; i += s.gs) P[i] = Pg[i];
    const int64_t row = s.b * d.ld;
    const int k = s.k;
    if (k < K) f[k] = d.t0 == 0 ? d.init[s.b * d.init_stride + k] : d.filt[(row + d.t0 - 1) * K + k];
    grp.sync();
    for (int64_t t = d.t0; t < d.t1; t++) {
        double pred = 0.0, lp = -CUDART_INF;
        if (k < K) {
            if (t == 0) {
                pred = f[k];
            } else {
                for (int j = 0; j < K; j++) pred += f[j] * P[j * K + k];
            }
            lp = log(pred) + d.logft[(row + t) * K + k];
        }
        const double m = grp.max(lp);
        const double sm = grp.sum(k < K ? fexp_neg(lp - m) : 0.0);
        const double lpy = m + log(sm);
        const double fk = fexp_neg(lp - lpy);
        if (k < K) {
            d.pred[(row + t) * K + k] = pred;
            d.filt[(row + t) * K + k] = fk;
        }
        if (k == 0) d.logpyt[row + t] = lpy;
        grp.sync();                                           // every read of f is done
        if (k < K) f[k] = fk;
        grp.sync();
    }
}

// ---------------------------------------------------------------------------
// BACKWARD -- hmm.py:212-236
// ---------------------------------------------------------------------------
template <bool kWarp>
__global__ void k_hmm_backward(smcb_hmm_desc d) {
    extern __shared__ double smem[];
    const int K = d.K;
    const Slot<kWarp> s = slot_of<kWarp>(smem, slab_doubles(K));
    if (s.b >= d.B) return;
    double *LT = s.base, *ft = LT + K * K, *c = ft + K;       // LT[j K + k] = log P[k][j]: conflict-free in k
    const Group<kWarp> grp{(int)(blockDim.x >> 5), c + K};
    const double *Pg = d.trans + s.b * d.trans_stride;
    for (int i = s.gi; i < K * K; i += s.gs) LT[(i % K) * K + i / K] = log(Pg[i]);
    const int64_t row = s.b * d.ld, T = d.t1;
    const int k = s.k;
    if (k < K) {
        c[k] = 0.0;
        d.smth[(row + T - 1) * K + k] = d.filt[(row + T - 1) * K + k];
    }
    for (int64_t t = T - 2; t >= 0; t--) {
        if (k < K) ft[k] = d.logft[(row + t + 1) * K + k];
        grp.sync();
        double ctg = 0.0;
        if (k < K) {
            double mx = -CUDART_INF;
            for (int j = 0; j < K; j++) mx = fmax(mx, (LT[j * K + k] + ft[j]) + c[j]);
            double sm = 0.0;
            for (int j = 0; j < K; j++) sm += fexp_neg(((LT[j * K + k] + ft[j]) + c[j]) - mx);
            ctg = mx + log(sm);
        }
        grp.sync();                                           // every read of c is done
        if (k < K) c[k] = ctg;
        const double lv = k < K ? log(d.filt[(row + t) * K + k]) + ctg : -CUDART_INF;
        const double m = grp.max(lv);
        const double e = k < K ? fexp_neg(lv - m) : 0.0;
        const double sm = grp.sum(e);
        if (k < K) d.smth[(row + t) * K + k] = e / sm;
    }
}

// ---------------------------------------------------------------------------
// SAMPLE -- hmm.py:241-268
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kSampleBlock) k_hmm_sample(smcb_hmm_desc d, Philox key) {
    extern __shared__ double smem[];
    const int K = d.K;
    double *C = smem, *lf = smem + K * K;                     // C[j K + k]: the CDF of x_t given x_{t+1} = j
    const int64_t b = blockIdx.y, N = d.N, T = d.t1;
    const int64_t n = (int64_t)blockIdx.x * kSampleBlock + threadIdx.x;
    const double *Pg = d.trans + b * d.trans_stride;
    const int64_t row = b * d.ld;
    int64_t *paths = d.paths + b * T * N;
    int64_t cur = n < N ? paths[(T - 1) * N + n] : 0;
    for (int64_t t = T - 2; t >= 0; t--) {
        for (int k = threadIdx.x; k < K; k += kSampleBlock) lf[k] = log(d.filt[(row + t) * K + k]);
        __syncthreads();
        for (int j = threadIdx.x; j < K; j += kSampleBlock) {
            double mx = -CUDART_INF;
            for (int k = 0; k < K; k++) mx = fmax(mx, log(Pg[k * K + j]) + lf[k]);
            double sm = 0.0;
            for (int k = 0; k < K; k++) sm += fexp_neg((log(Pg[k * K + j]) + lf[k]) - mx);
            double cs = 0.0;
            for (int k = 0; k < K; k++) {
                cs += fexp_neg((log(Pg[k * K + j]) + lf[k]) - mx) / sm;
                C[j * K + k] = cs;
            }
        }
        __syncthreads();
        if (n < N) {
            double u;
            if (d.U) {
                u = d.U[(b * (T - 1) + t) * N + n];
            } else {
                uint32_t r[4];
                philox4x32_10k((uint32_t)n, (uint32_t)t, (uint32_t)b, kPurposeHmm, key, r);
                u = u53(r[0], r[1]);
            }
            const double *col = C + cur * K;
            int lo = 0, hi = K;                               // the first k with col[k] >= u
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (col[mid] < u) lo = mid + 1;
                else hi = mid;
            }
            cur = lo < K ? lo : K - 1;
            paths[t * N + n] = cur;
        }
        __syncthreads();                                      // the table is rebuilt for t - 1
    }
}

template <bool kWarp>
int launch_groups(smcb_ctx *c, const smcb_hmm_desc &d) {
    const int K = d.K;
    const size_t per = (size_t)slab_doubles(K) * sizeof(double);
    const int block = kWarp ? 32 * kHmmGroups : 32 * ((K + 31) / 32);
    const size_t smem = kWarp ? per * kHmmGroups : per;
    const int64_t grid = kWarp ? (d.B + kHmmGroups - 1) / kHmmGroups : d.B;
    if (d.method == SMCB_HMM_FORWARD) {
        SMCB_TRY(set_smem(k_hmm_forward<kWarp>, smem));
        return launch(c, k_hmm_forward<kWarp>, (unsigned)grid, block, smem, d);
    }
    SMCB_TRY(set_smem(k_hmm_backward<kWarp>, smem));
    return launch(c, k_hmm_backward<kWarp>, (unsigned)grid, block, smem, d);
}

}  // namespace

extern "C" int smcb_hmm(smcb_ctx *c, const smcb_hmm_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_hmm: NULL argument");
    const smcb_hmm_desc &d = *dp;
    SMCB_REQUIRE(d.method == SMCB_HMM_FORWARD || d.method == SMCB_HMM_BACKWARD || d.method == SMCB_HMM_SAMPLE,
                 "smcb_hmm: bad method %d", (int)d.method);
    if (d.K > SMCB_HMM_MAX_K) {
        set_error("smcb_hmm: K = %d states is above the bound of %d", (int)d.K, SMCB_HMM_MAX_K);
        return SMCB_ENOSYS;
    }
    SMCB_REQUIRE(d.K >= 1 && d.B >= 1 && d.B <= 0x7fffffffLL && d.ld >= 1, "smcb_hmm: bad sizes K=%d B=%lld ld=%lld",
                 (int)d.K, (long long)d.B, (long long)d.ld);
    SMCB_REQUIRE(d.trans && d.trans_stride >= 0 && d.filt && d.logft, "smcb_hmm: NULL trans, filt or logft");
    if (d.method == SMCB_HMM_FORWARD) {
        SMCB_REQUIRE(d.init && d.init_stride >= 0 && d.pred && d.logpyt, "smcb_hmm: FORWARD needs init, pred, logpyt");
        SMCB_REQUIRE(d.t0 >= 0 && d.t0 <= d.t1 && d.t1 <= d.ld, "smcb_hmm: bad rows [%lld, %lld) of %lld",
                     (long long)d.t0, (long long)d.t1, (long long)d.ld);
        if (d.t0 == d.t1) return SMCB_OK;
        return d.K <= 32 ? launch_groups<true>(c, d) : launch_groups<false>(c, d);
    }
    if (d.method == SMCB_HMM_BACKWARD) {
        SMCB_REQUIRE(d.smth && d.t1 >= 1 && d.t1 <= d.ld, "smcb_hmm: BACKWARD needs smth and 1 <= T <= ld");
        return d.K <= 32 ? launch_groups<true>(c, d) : launch_groups<false>(c, d);
    }
    SMCB_REQUIRE(d.paths && d.t1 >= 1 && d.t1 <= d.ld && d.N >= 1 && d.N <= 0x7fffffffLL && d.B <= 65535,
                 "smcb_hmm: SAMPLE needs paths, 1 <= T <= ld, 1 <= N < 2^31 and B <= 65535");
    if (d.t1 == 1) return SMCB_OK;
    const size_t smem = ((size_t)d.K * d.K + d.K) * sizeof(double);
    SMCB_TRY(set_smem(k_hmm_sample, smem));
    const dim3 grid((unsigned)((d.N + kSampleBlock - 1) / kSampleBlock), (unsigned)d.B);
    return launch(c, k_hmm_sample, grid, kSampleBlock, smem, d, key_of(d.seed));
}
