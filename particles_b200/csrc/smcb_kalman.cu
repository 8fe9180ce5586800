// smcb_kalman.cu -- Kalman filter and RTS smoother (particles/kalman.py:169-290, 483-517) for B linear-Gaussian
// models X_t = F X_{t-1} + U, Y_t = G X_t + V with max(dx, dy) <= SMCB_KALMAN_MAX_D:
//   FILTER  rows [t0, t1) in one launch: pred = (mu0, cov0) at t = 0, else (F m, (F Sig) F' + covX);
//           S = (G P) G' + covY, L = chol(S), K' = S^-1 (P G')' through L, filt = (m + K r, P - (K G) P);
//           logpyt = scipy.stats.norm.logpdf's form with scale sqrt(S) (dy = 1) or MvNormal.logpdf's
//           -|L^-1 r|^2 / 2 - sum log L_ii - dy log(2 pi) / 2 (dy > 1);
//   SMOOTH  rows [0, t1) in one launch: J' = P_{t+1}^-1 (Sig_f F')' through chol(P_{t+1}),
//           Sig_s = Sig_f + (J (Sig_s' - P_{t+1})) J', m_s = m_f + J (m_s' - m_{t+1}); smth_{T-1} = filt_{T-1}.
// Tiers: dx = dy = 1 runs one thread per model in registers; otherwise one warp per model, several models per CTA
// (sized from the slab of shared memory one model needs), lane i owning row i of every matrix.  Every sum runs in
// index order inside one thread, from 0.0, and nothing depends on where the model sits in the batch, so a batch row
// is bit-identical to the same model run alone; the library is compiled with -fmad=false.  A non-positive pivot in a
// Cholesky factor becomes NaN, which then fills that model's rows from that step on (no host read, no exception).
#include "smcb_common.cuh"

using namespace smcb;

namespace {

constexpr double kHalfLog2Pi = 0x1.d67f1c864beb4p-1;   // 0.5 log(2 pi) == log(sqrt(2 pi)) in fp64
constexpr int kScalarBlock = 128;                       // scalar tier: models per CTA
constexpr int kMaxGroups = 8;                           // warp tier: at most this many models per CTA
constexpr size_t kSmemBudget = 200 * 1024;              // warp tier: dynamic shared memory per CTA

__device__ __forceinline__ double pivot(double v) { return v > 0.0 ? sqrt(v) : CUDART_NAN; }

// ---------------------------------------------------------------------------
// Scalar tier: dx = dy = 1, one thread per model, the warp tier's operations with d = 1.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kScalarBlock) k_kalman_filter_1(smcb_kalman_desc d) {
    const int64_t b = (int64_t)blockIdx.x * kScalarBlock + threadIdx.x;
    if (b >= d.B) return;
    const double F = d.F[b * d.F_stride], G = d.G[b * d.G_stride];
    const double cX = d.covX[b * d.covX_stride], cY = d.covY[b * d.covY_stride];
    const int64_t row = b * d.ld;
    const double *y = d.y + b * d.y_stride;
    double m = 0.0, S = 0.0;
    if (d.t0 > 0) {
        m = d.filt_mean[row + d.t0 - 1];
        S = d.filt_cov[row + d.t0 - 1];
    }
    for (int64_t t = d.t0; t < d.t1; t++) {
        double pm, P;
        if (t == 0) {
            pm = d.mu0[b * d.mu0_stride];
            P = d.cov0[b * d.cov0_stride];
        } else {
            pm = F * m;
            P = (F * S) * F + cX;
        }
        const double dpm = G * pm;
        const double L = pivot((G * P) * G + cY);
        const double K = ((P * G) / L) / L;
        const double r = y[t] - dpm;
        m = pm + r * K;
        S = P - (K * G) * P;
        const double z = r / L;
        d.pred_mean[row + t] = pm;
        d.pred_cov[row + t] = P;
        d.filt_mean[row + t] = m;
        d.filt_cov[row + t] = S;
        d.logpyt[row + t] = -(z * z) / 2.0 - kHalfLog2Pi - log(L);
    }
}

__global__ void __launch_bounds__(kScalarBlock) k_kalman_smooth_1(smcb_kalman_desc d) {
    const int64_t b = (int64_t)blockIdx.x * kScalarBlock + threadIdx.x;
    if (b >= d.B) return;
    const double F = d.F[b * d.F_stride];
    const int64_t row = b * d.ld, T = d.t1;
    double ms = d.filt_mean[row + T - 1], Ss = d.filt_cov[row + T - 1];
    d.smth_mean[row + T - 1] = ms;
    d.smth_cov[row + T - 1] = Ss;
    for (int64_t t = T - 2; t >= 0; t--) {
        const double Sf = d.filt_cov[row + t], P = d.pred_cov[row + t + 1];
        const double Lp = pivot(P);
        const double J = ((Sf * F) / Lp) / Lp;
        const double dm = ms - d.pred_mean[row + t + 1];
        Ss = Sf + (J * (Ss - P)) * J;
        ms = d.filt_mean[row + t] + dm * J;
        d.smth_mean[row + t] = ms;
        d.smth_cov[row + t] = Ss;
    }
}

// ---------------------------------------------------------------------------
// Warp tier: one warp per model.  Matrices are row-major in shared memory with an odd leading dimension (n | 1),
// so the lanes reading one column of their own rows hit distinct banks.
// ---------------------------------------------------------------------------
__host__ __device__ __forceinline__ int lead(int n) { return n | 1; }

__host__ __device__ __forceinline__ int slab_doubles(int dx, int dy) {
    const int lx = lead(dx), ly = lead(dy);
    const int w = dy * lx > dx * ly ? dy * lx : dx * ly;
    return 5 * dx * lx + dy * lx + 2 * dy * ly + w + 4 * 32;
}

// out[l] = base[l] + s * acc_l for l < n, acc_l = sum_{k < m} a[k] B(k, l) in k order from 0.0, where B(k, l) is
// Bm[k * ldb + l] (kT = false: a B) or Bm[l * ldb + k] (kT = true: a B').  s = 0 drops base; s = -1 is base - acc.
// Four columns run side by side; each keeps its own k-ordered sum.
template <bool kT>
__device__ __forceinline__ void row_prod(const double *a, const double *Bm, int ldb, int n, int m, double *out,
                                         const double *base, int s) {
    for (int l = 0; l < n; l += 4) {
        int c[4];
#pragma unroll
        for (int q = 0; q < 4; q++) c[q] = l + q < n ? l + q : n - 1;
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int k = 0; k < m; k++) {
            const double ak = a[k];
#pragma unroll
            for (int q = 0; q < 4; q++) acc[q] += ak * (kT ? Bm[c[q] * ldb + k] : Bm[k * ldb + c[q]]);
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (l + q < n) out[l + q] = s == 0 ? acc[q] : s > 0 ? base[l + q] + acc[q] : base[l + q] - acc[q];
        }
    }
}

// in-place Cholesky of the n x n matrix A (lower triangle), left-looking, lane i owning row i
__device__ __forceinline__ void chol(double *A, int ld, int n, int i) {
    for (int j = 0; j < n; j++) {
        if (i == j) {
            double acc = 0.0;
            for (int k = 0; k < j; k++) acc += A[j * ld + k] * A[j * ld + k];
            A[j * ld + j] = pivot(A[j * ld + j] - acc);
        }
        __syncwarp();
        if (i > j && i < n) {
            double acc = 0.0;
            for (int k = 0; k < j; k++) acc += A[i * ld + k] * A[j * ld + k];
            A[i * ld + j] = (A[i * ld + j] - acc) / A[j * ld + j];
        }
    }
    __syncwarp();
}

// x <- (L L')^-1 x for one right-hand side x (stride 1), L lower n x n: forward, then backward substitution
__device__ __forceinline__ void chol_solve(const double *L, int ld, int n, double *x) {
    for (int j = 0; j < n; j++) {
        double acc = 0.0;
        for (int k = 0; k < j; k++) acc += L[j * ld + k] * x[k];
        x[j] = (x[j] - acc) / L[j * ld + j];
    }
    for (int j = n - 1; j >= 0; j--) {
        double acc = 0.0;
        for (int k = j + 1; k < n; k++) acc += L[k * ld + j] * x[k];
        x[j] = (x[j] - acc) / L[j * ld + j];
    }
}

// the warp's slab of shared memory and its batch row; a model's row-major (r x c) global matrix to and from it
struct Warp {
    int64_t b;
    int lane;
    double *base;
};

__device__ __forceinline__ Warp warp_of(double *smem, int per) {
    const int g = threadIdx.x >> 5;
    return Warp{(int64_t)blockIdx.x * (blockDim.x >> 5) + g, (int)(threadIdx.x & 31), smem + (size_t)g * per};
}

__device__ __forceinline__ void load(double *dst, int ld, const double *src, int r, int c, int lane) {
    for (int e = lane; e < r * c; e += 32) dst[(e / c) * ld + e % c] = src[e];
}

__device__ __forceinline__ void store(double *dst, const double *src, int ld, int r, int c, int lane) {
    for (int e = lane; e < r * c; e += 32) dst[e] = src[(e / c) * ld + e % c];
}

__global__ void k_kalman_filter_w(smcb_kalman_desc d) {
    extern __shared__ double smem[];
    const int dx = d.dx, dy = d.dy, lx = lead(dx), ly = lead(dy);
    const Warp w = warp_of(smem, slab_doubles(dx, dy));
    if (w.b >= d.B) return;                                   // the whole warp leaves
    const int i = w.lane;
    double *F = w.base, *cX = F + dx * lx, *Sg = cX + dx * lx, *P = Sg + dx * lx, *A = P + dx * lx;
    double *G = A + dx * lx, *cY = G + dy * lx, *L = cY + dy * ly, *W = L + dy * ly;
    double *m = W + (dy * lx > dx * ly ? dy * lx : dx * ly), *pm = m + 32, *r = pm + 32, *z = r + 32;
    const int64_t b = w.b;
    load(F, lx, d.F + b * d.F_stride, dx, dx, i);
    load(cX, lx, d.covX + b * d.covX_stride, dx, dx, i);
    load(G, lx, d.G + b * d.G_stride, dy, dx, i);
    load(cY, ly, d.covY + b * d.covY_stride, dy, dy, i);
    const int64_t row = b * d.ld;
    if (d.t0 > 0) {
        if (i < dx) m[i] = d.filt_mean[(row + d.t0 - 1) * dx + i];
        load(Sg, lx, d.filt_cov + (row + d.t0 - 1) * dx * dx, dx, dx, i);
    }
    const double *y = d.y + b * d.y_stride;
    __syncwarp();
    for (int64_t t = d.t0; t < d.t1; t++) {
        // predict_step
        if (t == 0) {
            if (i < dx) pm[i] = d.mu0[b * d.mu0_stride + i];
            load(P, lx, d.cov0 + b * d.cov0_stride, dx, dx, i);
        } else {
            if (i < dx) {
                row_prod<false>(F + i * lx, m, 1, 1, dx, pm + i, nullptr, 0);
                row_prod<false>(F + i * lx, Sg, lx, dx, dx, A + i * lx, nullptr, 0);
            }
            __syncwarp();
            if (i < dx) row_prod<true>(A + i * lx, F, lx, dx, dx, P + i * lx, cX + i * lx, 1);
        }
        __syncwarp();
        // filter_step: S = (G P) G' + covY (W holds G P), residual r = y - G pm
        if (i < dy) {
            double dpm;
            row_prod<false>(G + i * lx, pm, 1, 1, dx, &dpm, nullptr, 0);
            r[i] = y[t * dy + i] - dpm;
            row_prod<false>(G + i * lx, P, lx, dx, dx, W + i * lx, nullptr, 0);
        }
        __syncwarp();
        if (i < dy) row_prod<true>(W + i * lx, G, lx, dy, dx, L + i * ly, cY + i * ly, 1);
        __syncwarp();
        chol(L, ly, dy, i);
        // gain: lane i solves S k = (P G')[i, :], so W row i becomes row i of K
        if (i < dx) {
            row_prod<true>(P + i * lx, G, lx, dy, dx, W + i * ly, nullptr, 0);
            chol_solve(L, ly, dy, W + i * ly);
        }
        double lp = 0.0;
        if (i == 0) {
            if (dy == 1) {
                const double zz = r[0] / L[0];
                lp = -(zz * zz) / 2.0 - kHalfLog2Pi - log(L[0]);
            } else {                                          // z = L^-1 r, MvNormal.logpdf
                double ssq = 0.0, hld = 0.0;
                for (int j = 0; j < dy; j++) {
                    double acc = 0.0;
                    for (int k = 0; k < j; k++) acc += L[j * ly + k] * z[k];
                    z[j] = (r[j] - acc) / L[j * ly + j];
                }
                for (int j = 0; j < dy; j++) ssq += z[j] * z[j];
                for (int j = 0; j < dy; j++) hld += log(L[j * ly + j]);
                lp = -0.5 * ssq - hld - dy * kHalfLog2Pi;
            }
        }
        __syncwarp();
        // filt = (pm + K r, P - (K G) P); A row i holds row i of K G
        if (i < dx) {
            double kr;
            row_prod<false>(W + i * ly, r, 1, 1, dy, &kr, nullptr, 0);
            m[i] = pm[i] + kr;
            row_prod<false>(W + i * ly, G, lx, dx, dy, A + i * lx, nullptr, 0);
            row_prod<false>(A + i * lx, P, lx, dx, dx, Sg + i * lx, P + i * lx, -1);
        }
        __syncwarp();
        const int64_t o = row + t;
        if (i < dx) {
            d.pred_mean[o * dx + i] = pm[i];
            d.filt_mean[o * dx + i] = m[i];
        }
        store(d.pred_cov + o * dx * dx, P, lx, dx, dx, i);
        store(d.filt_cov + o * dx * dx, Sg, lx, dx, dx, i);
        if (i == 0) d.logpyt[o] = lp;
        __syncwarp();
    }
}

__global__ void k_kalman_smooth_w(smcb_kalman_desc d) {
    extern __shared__ double smem[];
    const int dx = d.dx, lx = lead(dx);
    const Warp w = warp_of(smem, slab_doubles(dx, d.dy));
    if (w.b >= d.B) return;
    const int i = w.lane;
    double *F = w.base, *Sg = F + dx * lx, *P = Sg + dx * lx, *A = P + dx * lx, *Cf = A + dx * lx;
    double *ms = Cf + dx * lx, *pm = ms + 32, *mf = pm + 32, *dm = mf + 32;
    load(F, lx, d.F + w.b * d.F_stride, dx, dx, i);
    const int64_t row = w.b * d.ld, T = d.t1;
    {
        const int64_t o = row + T - 1;
        if (i < dx) {
            ms[i] = d.filt_mean[o * dx + i];
            d.smth_mean[o * dx + i] = ms[i];
        }
        load(Sg, lx, d.filt_cov + o * dx * dx, dx, dx, i);
        for (int e = i; e < dx * dx; e += 32) d.smth_cov[o * dx * dx + e] = d.filt_cov[o * dx * dx + e];
    }
    __syncwarp();
    for (int64_t t = T - 2; t >= 0; t--) {
        const int64_t o = row + t;
        load(Cf, lx, d.filt_cov + o * dx * dx, dx, dx, i);
        load(P, lx, d.pred_cov + (o + 1) * dx * dx, dx, dx, i);
        if (i < dx) {
            mf[i] = d.filt_mean[o * dx + i];
            pm[i] = d.pred_mean[(o + 1) * dx + i];
        }
        __syncwarp();
        // A = Sig_f F'; dm = m_s' - m_{t+1}; Sg becomes D = Sig_s' - P_{t+1}
        if (i < dx) {
            row_prod<true>(Cf + i * lx, F, lx, dx, dx, A + i * lx, nullptr, 0);
            dm[i] = ms[i] - pm[i];
            for (int l = 0; l < dx; l++) Sg[i * lx + l] = Sg[i * lx + l] - P[i * lx + l];
        }
        __syncwarp();
        chol(P, lx, dx, i);
        if (i < dx) chol_solve(P, lx, dx, A + i * lx);        // A row i becomes row i of J
        __syncwarp();
        if (i < dx) row_prod<false>(A + i * lx, Sg, lx, dx, dx, P + i * lx, nullptr, 0);     // P row i: (J D)[i]
        __syncwarp();
        if (i < dx) {
            row_prod<true>(P + i * lx, A, lx, dx, dx, Sg + i * lx, Cf + i * lx, 1);
            double jd;
            row_prod<false>(A + i * lx, dm, 1, 1, dx, &jd, nullptr, 0);
            ms[i] = mf[i] + jd;
            d.smth_mean[o * dx + i] = ms[i];
        }
        __syncwarp();
        store(d.smth_cov + o * dx * dx, Sg, lx, dx, dx, i);
        __syncwarp();
    }
}

// models per CTA of the warp tier
int warp_groups(int dx, int dy) {
    const size_t per = (size_t)slab_doubles(dx, dy) * sizeof(double);
    const size_t g = kSmemBudget / per;
    return g < 1 ? 1 : g > kMaxGroups ? kMaxGroups : (int)g;
}

}  // namespace

extern "C" int smcb_kalman(smcb_ctx *c, const smcb_kalman_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_kalman: NULL argument");
    const smcb_kalman_desc &d = *dp;
    SMCB_REQUIRE(d.method == SMCB_KALMAN_FILTER || d.method == SMCB_KALMAN_SMOOTH, "smcb_kalman: bad method %d",
                 (int)d.method);
    if (d.dx > SMCB_KALMAN_MAX_D || d.dy > SMCB_KALMAN_MAX_D) {
        set_error("smcb_kalman: dx = %d, dy = %d is above the bound of %d", (int)d.dx, (int)d.dy, SMCB_KALMAN_MAX_D);
        return SMCB_ENOSYS;
    }
    SMCB_REQUIRE(d.dx >= 1 && d.dy >= 1 && d.B >= 1 && d.B <= 0x7fffffffLL && d.ld >= 1,
                 "smcb_kalman: bad sizes dx=%d dy=%d B=%lld ld=%lld", (int)d.dx, (int)d.dy, (long long)d.B,
                 (long long)d.ld);
    SMCB_REQUIRE(d.F && d.F_stride >= 0 && d.filt_mean && d.filt_cov && d.pred_mean && d.pred_cov,
                 "smcb_kalman: NULL F, pred or filt");
    if (d.method == SMCB_KALMAN_FILTER) {
        SMCB_REQUIRE(d.G && d.covX && d.covY && d.mu0 && d.cov0 && d.y && d.logpyt && d.G_stride >= 0 &&
                         d.covX_stride >= 0 && d.covY_stride >= 0 && d.mu0_stride >= 0 && d.cov0_stride >= 0 &&
                         d.y_stride >= 0,
                     "smcb_kalman: FILTER needs G, covX, covY, mu0, cov0, y and logpyt");
        SMCB_REQUIRE(d.t0 >= 0 && d.t0 <= d.t1 && d.t1 <= d.ld, "smcb_kalman: bad rows [%lld, %lld) of %lld",
                     (long long)d.t0, (long long)d.t1, (long long)d.ld);
        if (d.t0 == d.t1) return SMCB_OK;
    } else {
        SMCB_REQUIRE(d.smth_mean && d.smth_cov && d.t1 >= 1 && d.t1 <= d.ld,
                     "smcb_kalman: SMOOTH needs smth and 1 <= T <= ld");
    }
    const bool filter = d.method == SMCB_KALMAN_FILTER;
    if (d.dx == 1 && d.dy == 1) {
        const unsigned grid = (unsigned)((d.B + kScalarBlock - 1) / kScalarBlock);
        return launch(c, filter ? k_kalman_filter_1 : k_kalman_smooth_1, grid, kScalarBlock, 0, d);
    }
    const int g = warp_groups(d.dx, d.dy);
    const size_t smem = (size_t)g * slab_doubles(d.dx, d.dy) * sizeof(double);
    const unsigned grid = (unsigned)((d.B + g - 1) / g);
    const auto kern = filter ? k_kalman_filter_w : k_kalman_smooth_w;
    SMCB_TRY(set_smem(kern, smem));
    return launch(c, kern, grid, 32 * g, smem, d);
}
