// smcb_models.cuh -- device restatements of the stock state-space models of the
// reference (the closures that particles builds ProbDist objects from), as structs of
// constants + inline maps, so that PX / PY / proposal / logeta become register math
// inside the fused step kernel (SURVEY.md section 8 row a22).
//
// Every model of the 1-D family exposes (all Normal kernels, as in the reference):
//   init (loc, scale)                     PX0()
//   trans(k, xp) -> (loc, scale)          PX(t, xp)
//   obs_logpdf(k, xp, x)                  PY(t, xp, x).logpdf(data[t])
//   prop0 / prop -> (loc, scale)          proposal0(data) / proposal(t, xp, data)
//   logeta(k, x)                          logeta(t, x, data)   (uses data[t+1])
// `k` carries the per-step scalars (t, y_t, y_{t+1}, host-computed step constants).
// Parameter layout of smcb_filter_desc.params is documented per model below.
#pragma once
#ifndef SMCB_MATH_HOST_TEST      // tests/math_host.cpp compiles this header for the CPU with its own shim
#include "smcb_common.cuh"
#endif
#include "smcb_math.cuh"

namespace smcb {

constexpr int kMaxDy = 4;
struct StepK {
    double y;        // data[t]        (first component; the 1-D models read only this)
    double y_next;   // data[t+1] (0 at the last step; only logeta reads it)
    double sc0;      // host-computed per-step constant (model specific)
    double yv[kMaxDy], yn[kMaxDy];   // vector observation data[t], data[t+1] (d-dimensional models)
    int64_t t;
};

// Normal.logpdf with log(scale) supplied (constant scales: computed once on the host
// with numpy, so the constant is bit-identical to the reference's np.log(scale))
__device__ __forceinline__ double normal_logpdf_ls(double x, double loc, double scale,
                                                   double logscale) {
    double z = (x - loc) / scale;
    return -z * z / 2.0 - kHalfLog2Pi - logscale;
}

// log(sqrt(2 pi)) as scipy.stats.norm.logpdf holds it (np.log of the rounded sqrt): one ulp below the correctly
// rounded kHalfLog2Pi.  The transition density of the backward samplers uses it so that PX.logpdf is bit-identical
// to the reference's.
constexpr double kHalfLog2PiScipy = 0x1.d67f1c864beb4p-1;

// x / c with r = RN(1 / c): the correctly rounded quotient (see MvLinGaussM::div_const)
__host__ __device__ __forceinline__ double div_rn(double x, double c, double r) {
    const double q = x * r;
    return fma(fma(-q, c, x), r, q);
}

// ---------------------------------------------------------------------------
// StochVol -- particles/state_space_models.py:446-498
// params: 0 mu, 1 rho, 2 sigma, 3 sig0, 4 (1-rho)*mu, 5 log(sigma), 6 log(sig0)
// ---------------------------------------------------------------------------
struct StochVolM {
    static constexpr int D = 1, NZ = 1;   // state dimension, normals per particle
    double mu, rho, sigma, sig0, c0, lsigma, lsig0;
    static constexpr bool has_proposal = true;
    __host__ __device__ void load(const double *p) {
        mu = p[0]; rho = p[1]; sigma = p[2]; sig0 = p[3]; c0 = p[4]; lsigma = p[5]; lsig0 = p[6];
    }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = mu; scale = sig0; ls = lsig0;                       // PX0, :462
    }
    __device__ __forceinline__ double ext(double xp) const { return c0 + rho * xp; }  // EXt, :465-467
    __device__ __forceinline__ void trans(const StepK &, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = ext(xp); scale = sigma; ls = lsigma;                // PX, :469-470
    }
    // PY = Normal(0, exp(x/2)), :472-473: z = y / exp(x/2), logpdf = -z^2/2 - log(2 pi)/2 - log(scale).
    // Evaluated with ONE exp: z^2 = y^2 exp(-x) and log(exp(x/2)) = x/2 (differences of a few ulp
    // of the individual terms, < 1e-15 absolute; tolerance of the parity tests is 1e-10).
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double, double x) const {
        const double z2 = (k.y * k.y) * mexp(-x);
        return -0.5 * z2 - kHalfLog2Pi - 0.5 * x;
    }
    __device__ __forceinline__ double xhat(double xst, double sig, double yt) const {  // :475-476
        return xst + 0.5 * (sig * sig) * ((yt * yt) * mexp(-xst) - 1.0);
    }
    __device__ __forceinline__ void prop0(const StepK &k, double &loc, double &scale, double &ls) const {
        loc = xhat(0.0, sig0, k.y); scale = sig0; ls = lsig0;     // :478-482
    }
    __device__ __forceinline__ void prop(const StepK &k, double xp, double &loc, double &scale,
                                         double &ls) const {
        loc = xhat(ext(xp), sigma, k.y); scale = sigma; ls = lsigma;  // :484-488
    }
    __device__ __forceinline__ double logeta(const StepK &k, double x) const {  // :490-498
        double xst = ext(x);
        double xstmmu = xst - mu;
        double e = mexp(-xst);
        double xh = xst + 0.5 * (sigma * sigma) * ((k.y_next * k.y_next) * e - 1.0);
        double xhatmmu = xh - mu;
        return 0.5 / (sigma * sigma) * (xhatmmu * xhatmmu - xstmmu * xstmmu) -
               0.5 * (k.y_next * k.y_next) * e * (1.0 + xstmmu);
    }
};

// ---------------------------------------------------------------------------
// LinearGauss -- particles/kalman.py:397-452; README ToySSM = (rho=1, sigmaX=1, sigma0=1)
// params: 0 rho, 1 sigmaX, 2 sigmaY, 3 sigma0, 4 log sigmaX, 5 log sigmaY, 6 log sigma0,
//         7 sig2post0, 8 sqrt(sig2post0), 9 log sqrt(sig2post0), 10 sig2post, 11 sqrt(sig2post),
//         12 log sqrt(sig2post), 13 sqrt(sX^2+sY^2), 14 log of 13, 15 sigmaX^2, 16 sigmaY^2
// ---------------------------------------------------------------------------
struct LinGaussM {
    static constexpr int D = 1, NZ = 1;   // state dimension, normals per particle
    double rho, sX, sY, s0, lsX, lsY, ls0, s2p0, sp0, lsp0, s2p, sp, lsp, se, lse, sX2, sY2;
    static constexpr bool has_proposal = true;
    __host__ __device__ void load(const double *p) {
        rho = p[0]; sX = p[1]; sY = p[2]; s0 = p[3]; lsX = p[4]; lsY = p[5]; ls0 = p[6];
        s2p0 = p[7]; sp0 = p[8]; lsp0 = p[9]; s2p = p[10]; sp = p[11]; lsp = p[12];
        se = p[13]; lse = p[14]; sX2 = p[15]; sY2 = p[16];
    }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = 0.0; scale = s0; ls = ls0;                          // PX0, :426-427
    }
    __device__ __forceinline__ void trans(const StepK &, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = rho * xp; scale = sX; ls = lsX;                     // PX, :429-430
    }
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double, double x) const {
        return normal_logpdf_ls(k.y, x, sY, lsY);                 // PY, :432-433
    }
    __device__ __forceinline__ void prop0(const StepK &k, double &loc, double &scale, double &ls) const {
        loc = s2p0 * (k.y / sY2); scale = sp0; ls = lsp0;         // :435-438
    }
    __device__ __forceinline__ void prop(const StepK &k, double xp, double &loc, double &scale,
                                         double &ls) const {
        loc = s2p * (rho * xp / sX2 + k.y / sY2); scale = sp; ls = lsp;  // :440-445
    }
    __device__ __forceinline__ double logeta(const StepK &k, double x) const {  // :447-451
        return normal_logpdf_ls(k.y_next, rho * x, se, lse);
    }
};

// ---------------------------------------------------------------------------
// Gordon et al -- particles/state_space_models.py:546-577 (Bootstrap only)
// params: 0 a, 1 b, 2 c, 3 sigmaX, 4 log sigmaX;  step constant sc0 = d*cos(e*(t-1))
// ---------------------------------------------------------------------------
struct GordonM {
    static constexpr int D = 1, NZ = 1;   // state dimension, normals per particle
    double a, b, c, sX, lsX;
    static constexpr bool has_proposal = false;
    __host__ __device__ void load(const double *p) { a = p[0]; b = p[1]; c = p[2]; sX = p[3]; lsX = p[4]; }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = 0.0; scale = 2.0; ls = 0.69314718055994530942;      // Normal(scale=2.), :563-564
    }
    __device__ __forceinline__ void trans(const StepK &k, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = b * xp + c * xp / (1.0 + xp * xp) + k.sc0;          // :566-572
        scale = sX; ls = lsX;
    }
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double, double x) const {
        return normal_logpdf_ls(k.y, a * (x * x), 1.0, 0.0);      // Normal(loc=a x^2), :574-575
    }
    __device__ __forceinline__ void prop0(const StepK &, double &, double &, double &) const {}
    __device__ __forceinline__ void prop(const StepK &, double, double &, double &, double &) const {}
    __device__ __forceinline__ double logeta(const StepK &, double) const { return 0.0; }
};

// ---------------------------------------------------------------------------
// ThetaLogistic -- particles/state_space_models.py:657-689 (Bootstrap)
// params: 0 tau0, 1 tau1, 2 tau2, 3 sigmaX, 4 sigmaY, 5 log sigmaX, 6 log sigmaY
// ---------------------------------------------------------------------------
struct ThetaLogisticM {
    static constexpr int D = 1, NZ = 1;   // state dimension, normals per particle
    double tau0, tau1, tau2, sX, sY, lsX, lsY;
    static constexpr bool has_proposal = false;
    __host__ __device__ void load(const double *p) {
        tau0 = p[0]; tau1 = p[1]; tau2 = p[2]; sX = p[3]; sY = p[4]; lsX = p[5]; lsY = p[6];
    }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = 0.0; scale = 1.0; ls = 0.0;                         // :672-673
    }
    __device__ __forceinline__ void trans(const StepK &, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = xp + tau0 - tau1 * mexp(tau2 * xp); scale = sX; ls = lsX;  // :675-678
    }
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double, double x) const {
        return normal_logpdf_ls(k.y, x, sY, lsY);                 // :680-681
    }
    __device__ __forceinline__ void prop0(const StepK &, double &, double &, double &) const {}
    __device__ __forceinline__ void prop(const StepK &, double, double &, double &, double &) const {}
    __device__ __forceinline__ double logeta(const StepK &, double) const { return 0.0; }
};

// ---------------------------------------------------------------------------
// StochVolLeverage -- particles/state_space_models.py:501-543 (Bootstrap; the reference warns
// that the inherited proposal / logeta are not valid for this model)
// params: StochVol's 0..6, then 7 phi, 8 sqrt(1 - phi^2), 9 log sqrt(1 - phi^2)
// ---------------------------------------------------------------------------
struct StochVolLevM {
    static constexpr int D = 1, NZ = 1;
    static constexpr bool has_proposal = false;
    double mu, rho, sigma, sig0, c0, lsigma, lsig0, phi, sq, lsq;
    __host__ __device__ void load(const double *p) {
        mu = p[0]; rho = p[1]; sigma = p[2]; sig0 = p[3]; c0 = p[4]; lsigma = p[5]; lsig0 = p[6];
        phi = p[7]; sq = p[8]; lsq = p[9];
    }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = mu; scale = sig0; ls = lsig0;
    }
    __device__ __forceinline__ void trans(const StepK &, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = c0 + rho * xp; scale = sigma; ls = lsigma;
    }
    // PY = Normal(s phi u, s sqrt(1 - phi^2)), s = exp(x/2), u = innovation of X_t (:533-543)
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double xp, double x) const {
        const double u = (k.t == 0) ? (x - mu) / sig0 : (x - (c0 + rho * xp)) / sigma;
        const double s = mexp(0.5 * x);
        const double z = (k.y - s * phi * u) / (s * sq);
        return -z * z / 2.0 - kHalfLog2Pi - (0.5 * x + lsq);     // log(s * sq) = x/2 + log sq
    }
    __device__ __forceinline__ void prop0(const StepK &, double &, double &, double &) const {}
    __device__ __forceinline__ void prop(const StepK &, double, double &, double &, double &) const {}
    __device__ __forceinline__ double logeta(const StepK &, double) const { return 0.0; }
};

// ---------------------------------------------------------------------------
// DiscreteCox -- particles/state_space_models.py:611-630: Y_t | X_t ~ Poisson(exp(X_t))
// params: 0 mu, 1 sigma, 2 phi, 3 sig0, 4 log sigma, 5 log sig0;
// step constant sc0 = gammaln(y_t + 1) (host, scipy's term of poisson.logpmf)
// ---------------------------------------------------------------------------
struct DiscreteCoxM {
    static constexpr int D = 1, NZ = 1;
    static constexpr bool has_proposal = false;
    double mu, sigma, phi, sig0, lsigma, lsig0;
    __host__ __device__ void load(const double *p) {
        mu = p[0]; sigma = p[1]; phi = p[2]; sig0 = p[3]; lsigma = p[4]; lsig0 = p[5];
    }
    __device__ __forceinline__ void init(double &loc, double &scale, double &ls) const {
        loc = mu; scale = sig0; ls = lsig0;                         // :622-625
    }
    __device__ __forceinline__ void trans(const StepK &, double xp, double &loc, double &scale,
                                          double &ls) const {
        loc = mu + phi * (xp - mu); scale = sigma; ls = lsigma;     // :627-628
    }
    // Poisson(rate = e^x).logpmf(y) = xlogy(y, rate) - gammaln(y + 1) - rate, log(rate) = x
    __device__ __forceinline__ double obs_logpdf(const StepK &k, double, double x) const {
        const double xl = (k.y == 0.0) ? 0.0 : k.y * x;
        return xl - k.sc0 - mexp(x);
    }
    __device__ __forceinline__ void prop0(const StepK &, double &, double &, double &) const {}
    __device__ __forceinline__ void prop(const StepK &, double, double &, double &, double &) const {}
    __device__ __forceinline__ double logeta(const StepK &, double) const { return 0.0; }
};

// ---------------------------------------------------------------------------
// Feynman-Kac adaptors -- particles/state_space_models.py:299-438
// ---------------------------------------------------------------------------
template <int FK> struct FkTraits {
    static constexpr bool guided = (FK == SMCB_FK_GUIDED || FK == SMCB_FK_APF);
    static constexpr bool apf = (FK == SMCB_FK_APF || FK == SMCB_FK_AUXBOOT);
};

// M0 + logG(0, None, x): Bootstrap :326-327, 332-333; GuidedPF :374-375, 381-386
template <class M, int FK>
__device__ __forceinline__ void fk_init(const M &m, const StepK &k, double z, double &x,
                                        double &delta) {
    double loc, scale, ls;
    if (FkTraits<FK>::guided) {
        m.prop0(k, loc, scale, ls);
        x = loc + scale * z;
        double l0, s0, ls0;
        m.init(l0, s0, ls0);
        delta = normal_logpdf_ls(x, l0, s0, ls0) + m.obs_logpdf(k, x, x) -
                normal_logpdf_ls(x, loc, scale, ls);
    } else {
        m.init(loc, scale, ls);
        x = loc + scale * z;
        delta = m.obs_logpdf(k, x, x);
    }
}

// M(t, xp) + logG(t, xp, x): Bootstrap :329-333; GuidedPF :377-392
template <class M, int FK>
__device__ __forceinline__ void fk_move(const M &m, const StepK &k, double xp, double z, double &x,
                                        double &delta) {
    double loc, scale, ls;
    if (FkTraits<FK>::guided) {
        m.prop(k, xp, loc, scale, ls);
        x = loc + scale * z;
        double lt, st, lst;
        m.trans(k, xp, lt, st, lst);
        delta = normal_logpdf_ls(x, lt, st, lst) + m.obs_logpdf(k, xp, x) -
                normal_logpdf_ls(x, loc, scale, ls);
    } else {
        m.trans(k, xp, loc, scale, ls);
        x = loc + scale * z;
        delta = m.obs_logpdf(k, xp, x);
    }
}

// logG(0, None, x) at a given state x: the delta of fk_init, for a particle that is not drawn (the pinned path of the
// conditional filter, smcb_pmcmc.cu)
template <class M, int FK>
__device__ __forceinline__ double fk_logG0(const M &m, const StepK &k, double x) {
    if (FkTraits<FK>::guided) {
        double loc, scale, ls, l0, s0, ls0;
        m.prop0(k, loc, scale, ls);
        m.init(l0, s0, ls0);
        return normal_logpdf_ls(x, l0, s0, ls0) + m.obs_logpdf(k, x, x) - normal_logpdf_ls(x, loc, scale, ls);
    }
    return m.obs_logpdf(k, x, x);
}

// logG(t, xp, x) at given states xp, x: the delta of fk_move
template <class M, int FK>
__device__ __forceinline__ double fk_logG(const M &m, const StepK &k, double xp, double x) {
    if (FkTraits<FK>::guided) {
        double loc, scale, ls, lt, st, lst;
        m.prop(k, xp, loc, scale, ls);
        m.trans(k, xp, lt, st, lst);
        return normal_logpdf_ls(x, lt, st, lst) + m.obs_logpdf(k, xp, x) - normal_logpdf_ls(x, loc, scale, ls);
    }
    return m.obs_logpdf(k, xp, x);
}

// ---------------------------------------------------------------------------
// d-dimensional models (SoA state): small dense algebra in registers, no tensor cores
// (SURVEY.md section 7 step 7: a 4x4 triangular matvec is 10 FMAs).
// ---------------------------------------------------------------------------

// BearingsOnly -- particles/state_space_models.py:580-608 (Bootstrap only: the reference defines
// no proposal).  State (x0, x1, x2, x3); PX = IndepProd(N(x0, sX), N(x1, sX), Dirac(x0 + x2),
// Dirac(x1 + x3)); PY = Normal(arctan(x3 / x2) [+ pi if x2 < 0], sY).
// params: 0 sigmaX, 1 sigmaY, 2 log sigmaY, 3..6 x0[4], 7 log sigmaX (transition density only)
struct BearingsM {
    static constexpr int D = 4, NZ = 2;
    static constexpr bool has_proposal = false;
    double sX, sY, lsY, x0[4], lsX, isX;
    __host__ __device__ void load(const double *p) {
        sX = p[0]; sY = p[1]; lsY = p[2];
        for (int i = 0; i < 4; i++) x0[i] = p[3 + i];
        lsX = p[7]; isX = 1.0 / sX;
    }
    // PX(t, xp).logpdf(x): IndepProd of N(xp0, sX), N(xp1, sX), Dirac(xp0 + xp2), Dirac(xp1 + xp3), summed in
    // component order (distributions.py IndepProd.logpdf); a Dirac gives 0 where x == loc, -inf elsewhere
    __device__ __forceinline__ void trans_loc(const StepK &, const double *xp, double *lc) const {
        lc[0] = xp[0]; lc[1] = xp[1]; lc[2] = xp[0] + xp[2]; lc[3] = xp[1] + xp[3];
    }
    __device__ __forceinline__ double trans_lpdf(const double *lc, const double *x) const {
        const double z0 = div_rn(x[0] - lc[0], sX, isX), z1 = div_rn(x[1] - lc[1], sX, isX);
        const double a = -z0 * z0 / 2.0 - kHalfLog2PiScipy - lsX, b = -z1 * z1 / 2.0 - kHalfLog2PiScipy - lsX;
        const double c = (x[2] == lc[2]) ? 0.0 : -CUDART_INF, d = (x[3] == lc[3]) ? 0.0 : -CUDART_INF;
        return ((a + b) + c) + d;
    }
    __device__ __forceinline__ double obs(const StepK &k, const double *x) const {   // :603-608
        double angle = atan(x[3] / x[2]);
        if (x[2] < 0.0) angle += 3.14159265358979323846;
        return normal_logpdf_ls(k.yv[0], angle, sY, lsY);
    }
    template <int FK>
    __device__ __forceinline__ void init_nd(const StepK &k, const double *z, double *x, double &d) const {
        x[0] = x0[0] + sX * z[0]; x[1] = x0[1] + sX * z[1]; x[2] = x0[2]; x[3] = x0[3];   // :589-595
        d = obs(k, x);
    }
    template <int FK>
    __device__ __forceinline__ void move_nd(const StepK &k, const double *xp, const double *z, double *x,
                                            double &d) const {
        x[0] = xp[0] + sX * z[0]; x[1] = xp[1] + sX * z[1];                             // :597-603
        x[2] = xp[0] + xp[2]; x[3] = xp[1] + xp[3];
        d = obs(k, x);
    }
    __device__ __forceinline__ double logeta_nd(const StepK &, const double *) const { return 0.0; }
};

// MVLinearGauss -- particles/kalman.py:296-361 (incl. MVLinearGauss_Guarniero_etal, 364-394):
//   X_0 ~ N(mu0, cov0), X_t = F X_{t-1} + U_t, Y_t = G X_t + V_t, optimal proposal and logeta from
//   the Kalman update with the common predictive covariance.  dx = DX (compile time), dy <= 4.
// params (row-major): 0 dy | F[DX*DX] | G[4*DX] | LX[DX*DX] hldX | LY[16] hldY | K[DX*4] |
//   LP[DX*DX] hldP | LE[16] hldE | mu0[DX] | L0[DX*DX] hld0 | loc0p[DX] | LP0[DX*DX] hldP0
// (L* = lower Cholesky factors, hld* = sum log diag; K = Kalman gain; LE = chol of G covX G' + covY)
template <int DX>
struct MvLinGaussM {
    static constexpr int D = DX, NZ = DX;
    static constexpr bool has_proposal = true;
    int dy;
    double F[DX * DX], G[kMaxDy * DX], LX[DX * DX], hldX, LY[kMaxDy * kMaxDy], hldY, K[DX * kMaxDy],
        LP[DX * DX], hldP, LE[kMaxDy * kMaxDy], hldE, mu0[DX], L0[DX * DX], hld0, loc0p[DX],
        LP0[DX * DX], hldP0;
    // reciprocals of the Cholesky diagonals (filled by load()): the triangular solves divide by model constants, and
    // x / c = fma(fma(-q, c, x), r, q) with q = x * r, r = RN(1 / c) is the correctly rounded quotient (Markstein) in 3
    // instructions instead of the ~20-instruction division sequence with its slow-path call
    double iLX[DX], iLY[kMaxDy], iLP[DX], iLE[kMaxDy], iL0[DX], iLP0[DX];
    __host__ __device__ void load(const double *p) {
        dy = (int)p[0]; p += 1;
        auto take = [&](double *dst, int cnt) { for (int i = 0; i < cnt; i++) dst[i] = p[i]; p += cnt; };
        take(F, DX * DX); take(G, kMaxDy * DX); take(LX, DX * DX); take(&hldX, 1);
        take(LY, kMaxDy * kMaxDy); take(&hldY, 1); take(K, DX * kMaxDy); take(LP, DX * DX); take(&hldP, 1);
        take(LE, kMaxDy * kMaxDy); take(&hldE, 1); take(mu0, DX); take(L0, DX * DX); take(&hld0, 1);
        take(loc0p, DX); take(LP0, DX * DX); take(&hldP0, 1);
        for (int i = 0; i < DX; i++) {
            iLX[i] = 1.0 / LX[i * DX + i]; iLP[i] = 1.0 / LP[i * DX + i];
            iL0[i] = 1.0 / L0[i * DX + i]; iLP0[i] = 1.0 / LP0[i * DX + i];
        }
        for (int i = 0; i < kMaxDy; i++) {
            iLY[i] = i < dy ? 1.0 / LY[i * kMaxDy + i] : 0.0;
            iLE[i] = i < dy ? 1.0 / LE[i * kMaxDy + i] : 0.0;
        }
    }
    static __host__ __device__ __forceinline__ double div_const(double x, double c, double r) {
        const double q = x * r;
        return fma(fma(-q, c, x), r, q);
    }
    // The small dense products are written with explicit fma(): the reference evaluates them through BLAS / LAPACK
    // (dgemm, dtrtrs), whose association order and FMA use are not defined, so there is no bit pattern to match
    // (parity for these models is 1e-11 relative, as for the oracle itself) and one instruction per term is half the work.
    // loc + scale * (z @ L.T) with scale = 1 (distributions.py:946-947)
    __device__ __forceinline__ void sample(const double *loc, const double *L, const double *z, double *x) const {
#pragma unroll
        for (int i = 0; i < DX; i++) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j <= i; j++) acc = fma(z[j], L[i * DX + j], acc);
            x[i] = loc[i] + 1.0 * acc;
        }
    }
    // MvNormal.logpdf (distributions.py:949-959), dimension DX
    __device__ __forceinline__ double logpdf_x(const double *x, const double *loc, const double *L, const double *iL,
                                               double hld) const {
        double zz[DX], ss = 0.0;
#pragma unroll
        for (int i = 0; i < DX; i++) {
            double acc = (x[i] - loc[i]) / 1.0;
#pragma unroll
            for (int j = 0; j < i; j++) acc = fma(-L[i * DX + j], zz[j], acc);
            zz[i] = div_const(acc, L[i * DX + i], iL[i]);
            ss = fma(zz[i], zz[i], ss);
        }
        return -0.5 * ss - (0.0 + hld) - (double)DX * kHalfLog2Pi;
    }
    // same in observation space (dimension dy <= 4, runtime)
    __device__ __forceinline__ double logpdf_y(const double *y, const double *loc, const double *L, const double *iL,
                                               double hld) const {
        double zz[kMaxDy], ss = 0.0;
#pragma unroll
        for (int i = 0; i < kMaxDy; i++) {
            if (i < dy) {
                double acc = (y[i] - loc[i]) / 1.0;
#pragma unroll
                for (int j = 0; j < kMaxDy; j++) if (j < i) acc = fma(-L[i * kMaxDy + j], zz[j], acc);
                zz[i] = div_const(acc, L[i * kMaxDy + i], iL[i]);
                ss = fma(zz[i], zz[i], ss);
            }
        }
        return -0.5 * ss - (0.0 + hld) - (double)dy * kHalfLog2Pi;
    }
    __device__ __forceinline__ void matvec_F(const double *xp, double *pm) const {   // xp @ F.T
#pragma unroll
        for (int i = 0; i < DX; i++) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j < DX; j++) acc = fma(xp[j], F[i * DX + j], acc);
            pm[i] = acc;
        }
    }
    __device__ __forceinline__ void matvec_G(const double *x, double *gy) const {    // x @ G.T
#pragma unroll
        for (int i = 0; i < kMaxDy; i++) {
            double acc = 0.0;
            if (i < dy) {
#pragma unroll
                for (int j = 0; j < DX; j++) acc = fma(x[j], G[i * DX + j], acc);
            }
            gy[i] = acc;
        }
    }
    __device__ __forceinline__ double obs(const StepK &k, const double *x) const {   // PY, kalman.py:342-343
        double gy[kMaxDy];
        matvec_G(x, gy);
        return logpdf_y(k.yv, gy, LY, iLY, hldY);
    }
    template <int FK>
    __device__ __forceinline__ void init_nd(const StepK &k, const double *z, double *x, double &d) const {
        if (FkTraits<FK>::guided) {      // proposal0 (kalman.py:351-354); logG(0) state_space_models.py:381-386
            sample(loc0p, LP0, z, x);
            d = logpdf_x(x, mu0, L0, iL0, hld0) + obs(k, x) - logpdf_x(x, loc0p, LP0, iLP0, hldP0);
        } else {                         // PX0 (kalman.py:336-337)
            sample(mu0, L0, z, x);
            d = obs(k, x);
        }
    }
    template <int FK>
    __device__ __forceinline__ void move_nd(const StepK &k, const double *xp, const double *z, double *x,
                                            double &d) const {
        double pm[DX];
        matvec_F(xp, pm);                // PX loc, kalman.py:339-340
        if (FkTraits<FK>::guided) {      // proposal, kalman.py:345-349 -> filter_step 196-229
            double gy[kMaxDy], loc[DX];
            matvec_G(pm, gy);
#pragma unroll
            for (int i = 0; i < DX; i++) {
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < kMaxDy; j++) if (j < dy) acc = fma(k.yv[j] - gy[j], K[i * kMaxDy + j], acc);
                loc[i] = pm[i] + acc;
            }
            sample(loc, LP, z, x);
            d = logpdf_x(x, pm, LX, iLX, hldX) + obs(k, x) - logpdf_x(x, loc, LP, iLP, hldP);
        } else {
            sample(pm, LX, z, x);
            d = obs(k, x);
        }
    }
    __device__ __forceinline__ double logeta_nd(const StepK &k, const double *x) const {   // kalman.py:356-360
        double pm[DX], gy[kMaxDy];
        matvec_F(x, pm);
        matvec_G(pm, gy);
        return logpdf_y(k.yn, gy, LE, iLE, hldE);
    }
    // PX(t, xp).logpdf(x) = MvNormal(F xp, covX).logpdf(x), kalman.py:339-340
    __device__ __forceinline__ void trans_loc(const StepK &, const double *xp, double *lc) const { matvec_F(xp, lc); }
    __device__ __forceinline__ double trans_lpdf(const double *lc, const double *x) const {
        return logpdf_x(x, lc, LX, iLX, hldX);
    }
};

// ---------------------------------------------------------------------------
// transition density PX(t, xp).logpdf(x) (Bootstrap.logpt, state_space_models.py:341-342) for backward sampling
// (csrc/smcb_smooth.cu).  `k` carries the time of x: logpt(t + 1, X_t, x_{t+1}) is evaluated with k.t = t + 1 and
// Gordon's step constant of t + 1.  Split in two so that the O(N^2) sampler computes the per-ancestor part once
// and shares it over every trajectory: loc(k, xp) -> D values, then lpdf(loc, x) per pair.
// ---------------------------------------------------------------------------
// models whose PX calls mexp (the table family): a kernel evaluating their density stages the tables first
template <class M> struct TransUsesTable { static constexpr bool value = false; };
template <> struct TransUsesTable<ThetaLogisticM> { static constexpr bool value = true; };

template <class M>
struct TransDensity {
    double s, is, ls;   // 1-D models: the (constant) scale of PX, its reciprocal and its log
    __device__ __forceinline__ void init(const M &m) {
        if constexpr (M::D == 1) {
            StepK k{};
            double l;
            m.trans(k, 0.0, l, s, ls);
            is = 1.0 / s;
        }
    }
    __device__ __forceinline__ void loc(const M &m, const StepK &k, const double *xp, double *lc) const {
        if constexpr (M::D == 1) {
            double sc, l;
            m.trans(k, xp[0], lc[0], sc, l);
        } else {
            m.trans_loc(k, xp, lc);
        }
    }
    // Normal.logpdf in the reference's order: z = (x - loc) / scale, -z^2/2 - log(2 pi)/2 - log(scale)
    __device__ __forceinline__ double lpdf(const M &m, const double *lc, const double *x) const {
        if constexpr (M::D == 1) {
            const double z = div_rn(x[0] - lc[0], s, is);
            return -z * z / 2.0 - kHalfLog2PiScipy - ls;
        } else {
            return m.trans_lpdf(lc, x);
        }
    }
};

template <class M>
__device__ __forceinline__ double trans_logpdf(const M &m, const StepK &k, const double *xp, const double *x) {
    TransDensity<M> td;
    td.init(m);
    double lc[M::D];
    td.loc(m, k, xp, lc);
    return td.lpdf(m, lc, x);
}

// uniform entry points for the step kernels: scalar Normal-kernel models or vector models
template <class M, int FK>
__device__ __forceinline__ void model_init(const M &m, const StepK &k, const double *z, double *x, double &d) {
    if constexpr (M::D == 1) fk_init<M, FK>(m, k, z[0], x[0], d);
    else m.template init_nd<FK>(k, z, x, d);
}
template <class M, int FK>
__device__ __forceinline__ void model_move(const M &m, const StepK &k, const double *xp, const double *z,
                                           double *x, double &d) {
    if constexpr (M::D == 1) fk_move<M, FK>(m, k, xp[0], z[0], x[0], d);
    else m.template move_nd<FK>(k, xp, z, x, d);
}
template <class M>
__device__ __forceinline__ double model_logeta(const M &m, const StepK &k, const double *x) {
    if constexpr (M::D == 1) return m.logeta(k, x[0]);
    else return m.logeta_nd(k, x);
}

}  // namespace smcb
