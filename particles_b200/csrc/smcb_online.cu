// smcb_online.cu -- one step of the on-line smoothers of additive functionals (particles/collectors.py:345-449):
//   PARIS      one thread per draw j = n * Np + i targeting x_t^n: the first trials alone, the stragglers served by
//              the whole warp (32 consecutive trials per round), then a warp-cooperative exact O(N) draw -- the
//              structure of k_bs_reject (smcb_smooth.cu) over ONE pair of generations;
//   ON2_W      the normalised backward weights of a block of rows, kOnRows rows per CTA: the CTA strides over the
//              ancestors m, computes the transition location of x_{t-1}^m once for its rows, pass 1 an online
//              log-sum-exp per row merged in a fixed order, pass 2 writes omega (coalesced along m);
//   PHI_*      the update of Phi from the draws / weights and the user's psi, in a fixed summation order.
// Randomness: Philox keyed by (seed, t, draw j, trial, purpose): the draws depend on the seed only, never on the
// launch geometry or on other API calls.
#include "smcb_dispatch.cuh"
#include "smcb_smooth.cuh"

using namespace smcb;

namespace {

constexpr int kOnRows = 4;                                    // ON2_W: rows per CTA
constexpr int kOnWarps = kSmBlock / 32;

// X_{t-1} in the layout the shared helpers read (load_x, reject_trial, warp_exact_draw): one generation, index 0
struct PrevGen {
    const double *X[1];
    const double *lw[1];
    int64_t x_stride_n, x_stride_c, N, M, max_trials, cdf_ld;
    const double *cdf;
    const int64_t *prop;
    const double *lu;
};

__device__ __forceinline__ PrevGen prev_gen(const smcb_online_desc &d) {
    PrevGen g;
    g.X[0] = d.X_prev;
    g.lw[0] = d.lw_prev;
    g.x_stride_n = d.x_stride_n;
    g.x_stride_c = d.x_stride_c;
    g.N = d.N;
    g.M = d.N * d.Np;
    g.max_trials = d.max_trials;
    g.cdf_ld = 0;
    g.cdf = d.cdf;
    g.prop = d.prop;
    g.lu = d.lu;
    return g;
}

__device__ __forceinline__ StepK step_of(const smcb_online_desc &d) {
    StepK k{};
    k.t = d.t;
    k.sc0 = d.step_const;
    return k;
}

template <int D>
__device__ __forceinline__ void load_cur(const smcb_online_desc &d, int64_t n, double *x) {
    const double *p = d.X + n * d.x_stride_n;
#pragma unroll
    for (int c = 0; c < D; c++) x[c] = p[c * d.x_stride_c];
}

// ---------------------------------------------------------------------------
// PaRIS draws -- collectors.py:417-444
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_paris(M m, smcb_online_desc d, Philox key, const double *tab) {
    constexpr int D = M::D;
    __shared__ __align__(8) uint64_t s_bar;
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const PrevGen g = prev_gen(d);
    const int lane = threadIdx.x & 31;
    const int64_t j = (int64_t)blockIdx.x * kSmBlock + threadIdx.x;
    const bool live = j < g.M;
    if (__all_sync(kFull, !live)) return;                   // whole warp past N * Np; partial warps stay
    const int64_t mt = d.max_trials;
    const uint64_t call = (uint64_t)d.t;
    TransDensity<M> td;
    td.init(m);
    const StepK k = step_of(d);
    const double bound = d.log_bound;
    double xn[D];
    if (live) {
        load_cur<D>(d, j / d.Np, xn);
    } else {
#pragma unroll
        for (int c = 0; c < D; c++) xn[c] = 0.0;
    }
    bool acc = !live;
    int64_t choice = 0, nprop = 0;
    const int64_t solo = mt < kSoloTrials ? mt : kSoloTrials;
    for (int64_t trial = 0; trial < solo; trial++) {
        if (__all_sync(kFull, acc)) break;
        if (!acc) {
            int64_t prop;
            nprop++;
            if (reject_trial<M>(m, td, g, k, key, call, j, 0, trial, xn, bound, prop)) {
                acc = true;
                choice = prop;
            }
        }
    }
    // the stragglers, one at a time by the whole warp: lane l runs trial base + l, the first accepted trial in
    // trial order wins -- the same draw, proposal and count as running the trials one after another
    unsigned slow = __ballot_sync(kFull, live && !acc && mt > solo);
    while (slow) {
        const int src = __ffs(slow) - 1;
        slow &= slow - 1;
        double xs[D];
#pragma unroll
        for (int c = 0; c < D; c++) xs[c] = __shfl_sync(kFull, xn[c], src);
        const int64_t js = j - lane + src;
        int64_t hit_trial = -1, hit_prop = 0;
        for (int64_t base = solo; base < mt && hit_trial < 0; base += 32) {
            const int64_t trial = base + lane;
            int64_t prop = 0;
            const bool ok = trial < mt && reject_trial<M>(m, td, g, k, key, call, js, 0, trial, xs, bound, prop);
            const unsigned b = __ballot_sync(kFull, ok);
            if (b) {
                const int f = __ffs(b) - 1;
                hit_trial = base + f;
                hit_prop = __shfl_sync(kFull, prop, f);
            }
        }
        if (lane == src) {
            nprop = hit_trial >= 0 ? hit_trial + 1 : mt;
            if (hit_trial >= 0) {
                acc = true;
                choice = hit_prop;
            }
        }
    }
    const long long na = warp_sum((live && acc) ? 1LL : 0LL), np = warp_sum(nprop);
    if (lane == 0) {
        atomicAdd(reinterpret_cast<unsigned long long *>(d.counts), (unsigned long long)na);
        atomicAdd(reinterpret_cast<unsigned long long *>(d.counts + 1), (unsigned long long)np);
    }
    // the exact fallback (collectors.py:437-440), served by the whole warp, one rejected lane at a time
    unsigned need = __ballot_sync(kFull, live && !acc);
    while (need) {
        const int src = __ffs(need) - 1;
        need &= need - 1;
        double xs[D];
#pragma unroll
        for (int c = 0; c < D; c++) xs[c] = __shfl_sync(kFull, xn[c], src);
        const int64_t js = j - lane + src;
        double u, tmp;
        if (d.u_exact) u = d.u_exact[js];
        else smooth_uniforms(key, call, js, 0, 0, kPurposeSmoothExact, u, tmp);
        const int64_t r = warp_exact_draw<M>(m, td, g, k, 0, xs, u, lane);
        if (lane == src) choice = r;
    }
    if (live) d.B[j] = choice;
}

// ---------------------------------------------------------------------------
// ON2 backward weights -- collectors.py:373-383: omega[r, m] = exp_and_normalise(lw_{t-1} + logpt(t, X_{t-1}, x_r))
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_on2_weights(M m, smcb_online_desc d, const double *tab) {
    constexpr int D = M::D;
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ double s_part[2][kOnWarps][kOnRows];
    __shared__ double s_fin[2][kOnRows];
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const PrevGen g = prev_gen(d);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * kOnRows;        // first row of this CTA, relative to d.row0
    const int nr = (int)min((int64_t)kOnRows, d.rows - r0);
    const int64_t N = d.N;
    TransDensity<M> td;
    td.init(m);
    const StepK k = step_of(d);
    double xr[kOnRows][D];
#pragma unroll
    for (int r = 0; r < kOnRows; r++) {
        if (r < nr) {
            load_cur<D>(d, d.row0 + r0 + r, xr[r]);
        } else {
#pragma unroll
            for (int c = 0; c < D; c++) xr[r][c] = 0.0;
        }
    }
    auto loc_of = [&](int64_t i, double *lc) {
        double xp[D];
        load_x<D>(g, 0, i, xp);
        td.loc(m, k, xp, lc);
    };
    // pass 1: per row (max, sum exp) over the thread's ancestors, then a fixed butterfly, then warps in order
    double mx[kOnRows], s[kOnRows];
#pragma unroll
    for (int r = 0; r < kOnRows; r++) { mx[r] = -CUDART_INF; s[r] = 0.0; }
    for (int64_t i = threadIdx.x; i < N; i += kSmBlock) {
        double lc[D];
        loc_of(i, lc);
        const double lw = d.lw_prev[i];
#pragma unroll
        for (int r = 0; r < kOnRows; r++) lse_add<false>(mx[r], s[r], lw + td.lpdf(m, lc, xr[r]));
    }
#pragma unroll
    for (int r = 0; r < kOnRows; r++) {
        warp_lse_merge(mx[r], s[r]);
        if (lane == 0) {
            s_part[0][warp][r] = mx[r];
            s_part[1][warp][r] = s[r];
        }
    }
    __syncthreads();
    if (threadIdx.x < kOnRows) {
        const int r = threadIdx.x;
        double M_ = -CUDART_INF, S = 0.0;
        for (int w = 0; w < kOnWarps; w++) {
            const double mo = s_part[0][w][r], so = s_part[1][w][r];
            const double Mx = fmax(M_, mo);
            if (Mx > -CUDART_INF) {
                S = S * fexp_neg(M_ - Mx) + so * fexp_neg(mo - Mx);
                M_ = Mx;
            }
        }
        s_fin[0][r] = M_;
        s_fin[1][r] = 1.0 / S;
    }
    __syncthreads();
    // pass 2: omega[r, i] = exp(v - max) / sum
    for (int64_t i = threadIdx.x; i < N; i += kSmBlock) {
        double lc[D];
        loc_of(i, lc);
        const double lw = d.lw_prev[i];
#pragma unroll
        for (int r = 0; r < kOnRows; r++) {
            if (r < nr) {
                const double v = lw + td.lpdf(m, lc, xr[r]);
                const double e = (v > -CUDART_INF) ? fexp_neg(v - s_fin[0][r]) : 0.0;
                d.omega[(r0 + r) * N + i] = e * s_fin[1][r];
            }
        }
    }
}

// ---------------------------------------------------------------------------
// Phi updates: PaRIS one thread per row (Np terms in i order, then / Np, as np.average(axis=0));
// ON2 one warp per row (lane-strided sums merged by a fixed butterfly)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_phi_paris(smcb_online_desc d) {
    const int64_t n = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    if (n >= d.N) return;
    const int64_t K = d.k, Np = d.Np;
    for (int64_t c = 0; c < K; c++) {
        double acc = 0.0;
        for (int64_t i = 0; i < Np; i++) {
            const int64_t j = n * Np + i;
            acc += d.phi_prev[d.B[j] * K + c] + d.psi[j * K + c];
        }
        d.phi[n * K + c] = acc / (double)Np;
    }
}

__global__ void __launch_bounds__(kBlock) k_phi_on2(smcb_online_desc d) {
    const int64_t r = ((int64_t)blockIdx.x * kBlock + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= d.rows) return;                                 // whole warps only: kBlock is a multiple of 32
    const int64_t K = d.k, N = d.N;
    const double *w = d.omega + r * N;
    double sw = 0.0;
    for (int64_t i = lane; i < N; i += 32) sw += w[i];
    sw = warp_sum(sw);
    for (int64_t c = 0; c < K; c++) {
        double acc = 0.0;
        for (int64_t i = lane; i < N; i += 32) acc += w[i] * (d.phi_prev[i * K + c] + d.psi[(r * N + i) * K + c]);
        acc = warp_sum(acc);
        if (lane == 0) d.phi[r * K + c] = acc / sw;
    }
}

template <class M>
int run_model(smcb_ctx *c, const smcb_online_desc &d) {
    SMCB_REQUIRE(d.dim == M::D, "smcb_online_smooth: dim %d does not match the model's %d", (int)d.dim, M::D);
    M m;
    m.load(d.params);
    const size_t tab = TransUsesTable<M>::value ? kMathTabBytes : 0;
    if (d.method == SMCB_ONLINE_PARIS) {
        SMCB_TRY(set_smem(k_paris<M>, tab));
        const int grid = (int)((d.N * d.Np + kSmBlock - 1) / kSmBlock);
        return launch(c, k_paris<M>, grid, kSmBlock, tab, m, d, key_of(d.seed ^ kOnlineSeedMix), c->math_tab);
    }
    SMCB_TRY(set_smem(k_on2_weights<M>, tab));
    const int grid = (int)((d.rows + kOnRows - 1) / kOnRows);
    return launch(c, k_on2_weights<M>, grid, kSmBlock, tab, m, d, c->math_tab);
}

}  // namespace

extern "C" int smcb_online_smooth(smcb_ctx *c, const smcb_online_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_online_smooth: NULL argument");
    const smcb_online_desc &d = *dp;
    SMCB_REQUIRE(d.N >= 1 && d.N <= 0x7fffffffLL, "smcb_online_smooth: bad N=%lld", (long long)d.N);
    if (d.method == SMCB_ONLINE_PHI_PARIS || d.method == SMCB_ONLINE_PHI_ON2) {
        SMCB_REQUIRE(d.phi_prev && d.psi && d.phi && d.k >= 1, "smcb_online_smooth: NULL Phi or psi");
        if (d.method == SMCB_ONLINE_PHI_PARIS) {
            SMCB_REQUIRE(d.B && d.Np >= 1, "smcb_online_smooth: PHI_PARIS needs B and Np >= 1");
            return launch(c, k_phi_paris, (int)((d.N + kBlock - 1) / kBlock), kBlock, 0, d);
        }
        SMCB_REQUIRE(d.omega && d.rows >= 1, "smcb_online_smooth: PHI_ON2 needs omega and rows >= 1");
        return launch(c, k_phi_on2, (int)((d.rows * 32 + kBlock - 1) / kBlock), kBlock, 0, d);
    }
    SMCB_REQUIRE(d.method == SMCB_ONLINE_PARIS || d.method == SMCB_ONLINE_ON2_W, "smcb_online_smooth: bad method %d",
                 (int)d.method);
    SMCB_REQUIRE(d.X_prev && d.X && d.lw_prev && d.dim >= 1, "smcb_online_smooth: NULL particles or log-weights");
    if (d.method == SMCB_ONLINE_PARIS) {
        SMCB_REQUIRE(d.Np >= 1 && d.N * d.Np <= 0x7fffffffLL, "smcb_online_smooth: bad Np=%lld", (long long)d.Np);
        SMCB_REQUIRE(d.max_trials >= 0 && d.max_trials < (1LL << 24), "smcb_online_smooth: max_trials out of range");
        SMCB_REQUIRE(d.B && d.counts, "smcb_online_smooth: PaRIS needs B and counts");
        SMCB_REQUIRE(d.max_trials == 0 || d.prop || d.cdf, "smcb_online_smooth: PaRIS needs the CDF");
        SMCB_REQUIRE((d.prop == nullptr) == (d.lu == nullptr), "smcb_online_smooth: prop and lu go together");
    } else {
        SMCB_REQUIRE(d.omega && d.rows >= 1 && d.row0 >= 0 && d.row0 + d.rows <= d.N,
                     "smcb_online_smooth: bad ON2 rows [%lld, +%lld)", (long long)d.row0, (long long)d.rows);
    }
    bool known = false;
    const int rc = with_model(d.model, d.dim, [&](auto m) {
        known = true;
        return run_model<decltype(m)>(c, d);
    });
    if (!known) set_error("smcb_online_smooth: no transition density for model %d, dim %d", (int)d.model, (int)d.dim);
    return rc;
}
