// smcb_twofilter.cu -- two-filter smoothing (particles/smoothing.py:487-566) of a forward generation X_t against an
// information generation Xinfo, one-dimensional states:
//   ON2_ROWS   a block of rows m of Xinfo, kTfRows rows per CTA: the CTA strides over the forward particles n,
//              computes the transition location of X_t[n] once for its rows, and keeps per row an online
//              (max, sum exp, sum exp * psi) that rescales when the max rises -- omega is never stored.  Thread
//              partials merge by a fixed butterfly, then warps in index order, so the bits depend on the inputs only;
//   ON_LOGW    one thread per draw j: the log-weight of the pair (X_t[J_j], Xinfo[I_j]) and the pair itself.
// The draws I, J, the combine across row blocks and the normalisation of omega are existing entries (smcb_resample,
// smcb_exp_and_normalise); the user's phi runs between the launches.
#include "smcb_dispatch.cuh"
#include "smcb_smooth.cuh"

using namespace smcb;

namespace {

constexpr int kTfRows = 4;                                    // ON2_ROWS: rows per CTA
constexpr int kTfWarps = kSmBlock / 32;

__device__ __forceinline__ StepK step_of(const smcb_twofilter_desc &d) {
    StepK k{};
    k.t = d.t + 1;
    k.sc0 = d.step_const;
    return k;
}

// lse_add with a second sum: (mx, s = sum exp(v - mx), a = sum exp(v - mx) psi); -inf and NaN values add nothing
__device__ __forceinline__ void lse_add_psi(double &mx, double &s, double &a, double v, double psi) {
    if (!(v > -CUDART_INF)) return;
    if (v > mx) {
        const double f = fexp_neg(mx - v);
        s = s * f + 1.0;
        a = a * f + psi;
        mx = v;
    } else {
        const double e = fexp_neg(v - mx);
        s += e;
        a += e * psi;
    }
}

// (mo, so, ao) into (mx, s, a): a rescales exactly as s does
__device__ __forceinline__ void lse_merge_psi(double &mx, double &s, double &a, double mo, double so, double ao) {
    double ma = mx;
    lse_merge(ma, a, mo, ao);
    lse_merge(mx, s, mo, so);
}

// ---------------------------------------------------------------------------
// ON2 rows -- smoothing.py:527-547, one block of information particles
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_tf_on2_rows(M m, smcb_twofilter_desc d, const double *tab) {
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ double s_part[3][kTfWarps][kTfRows];
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * kTfRows;        // first row of this CTA, relative to d.row0
    const int nr = (int)min((int64_t)kTfRows, d.rows - r0);
    const int64_t N = d.N;
    TransDensity<M> td;
    td.init(m);
    const StepK k = step_of(d);
    double xr[kTfRows][1];
    const double *psi[kTfRows];
#pragma unroll
    for (int r = 0; r < kTfRows; r++) {
        xr[r][0] = r < nr ? d.Xinfo[(d.row0 + r0 + r) * d.xi_stride] : 0.0;
        psi[r] = d.psi + (r0 + (r < nr ? r : 0)) * N;
    }
    double mx[kTfRows], s[kTfRows], a[kTfRows];
#pragma unroll
    for (int r = 0; r < kTfRows; r++) { mx[r] = -CUDART_INF; s[r] = 0.0; a[r] = 0.0; }
    for (int64_t n = threadIdx.x; n < N; n += kSmBlock) {
        double xp[1], lc[1];
        xp[0] = d.X[n * d.x_stride];
        td.loc(m, k, xp, lc);
        const double lw = d.lw[n];
#pragma unroll
        for (int r = 0; r < kTfRows; r++)
            if (r < nr) lse_add_psi(mx[r], s[r], a[r], lw + td.lpdf(m, lc, xr[r]), psi[r][n]);
    }
#pragma unroll
    for (int r = 0; r < kTfRows; r++) {
#pragma unroll
        for (int mask = 16; mask > 0; mask >>= 1) {
            const double mo = __shfl_xor_sync(kFull, mx[r], mask), so = __shfl_xor_sync(kFull, s[r], mask),
                         ao = __shfl_xor_sync(kFull, a[r], mask);
            lse_merge_psi(mx[r], s[r], a[r], mo, so, ao);
        }
        if (lane == 0) {
            s_part[0][warp][r] = mx[r];
            s_part[1][warp][r] = s[r];
            s_part[2][warp][r] = a[r];
        }
    }
    __syncthreads();
    if (threadIdx.x < nr) {
        const int r = threadIdx.x;
        double M_ = -CUDART_INF, S = 0.0, A = 0.0;
        for (int w = 0; w < kTfWarps; w++) lse_merge_psi(M_, S, A, s_part[0][w][r], s_part[1][w][r], s_part[2][w][r]);
        const int64_t row = d.row0 + r0 + r;
        const bool any = S > 0.0;                             // no positive pair weight: contributes exactly 0
        d.L[row] = any ? M_ + log(S) : -CUDART_INF;
        d.S[row] = any ? A / S : 0.0;
    }
}

// ---------------------------------------------------------------------------
// ON log-weights -- smoothing.py:549-566
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_tf_on_logw(M m, smcb_twofilter_desc d, const double *tab) {
    __shared__ __align__(8) uint64_t s_bar;
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const int64_t j = (int64_t)blockIdx.x * kSmBlock + threadIdx.x;
    if (j >= d.M) return;
    TransDensity<M> td;
    td.init(m);
    const StepK k = step_of(d);
    const int64_t jf = d.J[j], ji = d.I[j];
    double xf[1], xi[1], lc[1];
    xf[0] = d.X[jf * d.x_stride];
    xi[0] = d.Xinfo[ji * d.xi_stride];
    td.loc(m, k, xf, lc);
    double lo = td.lpdf(m, lc, xi);
    if (d.mf) lo -= d.mf[jf];                                 // the reference's order: forward, then information
    if (d.mi) lo -= d.mi[ji];
    d.log_omega[j] = lo;
    d.xf[j] = xf[0];
    d.xi[j] = xi[0];
}

template <class M>
int run_model(smcb_ctx *c, const smcb_twofilter_desc &d) {
    if constexpr (M::D != 1) {
        set_error("smcb_two_filter: two-filter smoothing is not built for %d-dimensional states", M::D);
        return SMCB_ENOSYS;
    } else {
        M m;
        m.load(d.params);
        const size_t tab = TransUsesTable<M>::value ? kMathTabBytes : 0;
        if (d.method == SMCB_TF_ON2_ROWS) {
            SMCB_TRY(set_smem(k_tf_on2_rows<M>, tab));
            const int grid = (int)((d.rows + kTfRows - 1) / kTfRows);
            return launch(c, k_tf_on2_rows<M>, grid, kSmBlock, tab, m, d, c->math_tab);
        }
        SMCB_TRY(set_smem(k_tf_on_logw<M>, tab));
        const int grid = (int)((d.M + kSmBlock - 1) / kSmBlock);
        return launch(c, k_tf_on_logw<M>, grid, kSmBlock, tab, m, d, c->math_tab);
    }
}

}  // namespace

extern "C" int smcb_two_filter(smcb_ctx *c, const smcb_twofilter_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_two_filter: NULL argument");
    const smcb_twofilter_desc &d = *dp;
    SMCB_REQUIRE(d.method == SMCB_TF_ON2_ROWS || d.method == SMCB_TF_ON_LOGW, "smcb_two_filter: bad method %d",
                 (int)d.method);
    SMCB_REQUIRE(d.N >= 1 && d.N <= 0x7fffffffLL && d.Ninfo >= 1 && d.Ninfo <= 0x7fffffffLL,
                 "smcb_two_filter: bad sizes N=%lld Ninfo=%lld", (long long)d.N, (long long)d.Ninfo);
    SMCB_REQUIRE(d.X && d.Xinfo && d.x_stride >= 1 && d.xi_stride >= 1, "smcb_two_filter: NULL or strided-out particles");
    if (d.dim != 1) {
        set_error("smcb_two_filter: two-filter smoothing is not built for %d-dimensional states", (int)d.dim);
        return SMCB_ENOSYS;
    }
    if (d.method == SMCB_TF_ON2_ROWS) {
        SMCB_REQUIRE(d.lw && d.psi && d.L && d.S, "smcb_two_filter: ON2 needs lw, psi, L and S");
        SMCB_REQUIRE(d.rows >= 1 && d.row0 >= 0 && d.row0 + d.rows <= d.Ninfo && d.rows <= 0x7fffffffLL,
                     "smcb_two_filter: bad ON2 rows [%lld, +%lld)", (long long)d.row0, (long long)d.rows);
    } else {
        SMCB_REQUIRE(d.I && d.J && d.log_omega && d.xf && d.xi, "smcb_two_filter: ON needs I, J and the outputs");
        SMCB_REQUIRE(d.M >= 1 && d.M <= 0x7fffffffLL, "smcb_two_filter: bad M=%lld", (long long)d.M);
    }
    bool known = false;
    const int rc = with_model(d.model, d.dim, [&](auto m) {
        known = true;
        return run_model<decltype(m)>(c, d);
    });
    if (!known) set_error("smcb_two_filter: no transition density for model %d, dim %d", (int)d.model, (int)d.dim);
    return rc;
}
