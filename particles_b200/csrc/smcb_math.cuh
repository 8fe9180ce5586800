// smcb_math.cuh -- fp64 elementary functions for the step kernel, written for its
// restricted domains.  Why not the CUDA math library: in the step kernel a large share of the
// issued warp-instructions were UMOVs materialising the library's 64-bit polynomial immediates
// and branches around special cases; here the
// coefficients sit in the constant bank (DFMA takes a c[bank][offset] operand directly), the
// domains are restricted and the code is branch-free.  Accuracy: polynomial errors < 5e-18
// (gen_coeffs.py), total error <= ~1.5 ulp; checked against NumPy/mpmath in
// tests/test_gpu_kernels.py::test_device_math.
#pragma once
//
// Two families:
//   f*  polynomial only (coefficients in the constant bank): stand-alone kernels, merges, the sampler;
//   t*  table-assisted, for the step kernels, whose CTAs keep the 64 KB of smcb_tables.h in shared memory: the
//       polynomials shrink to degree 3-5 with coefficients that are fp64 IMMEDIATES (low word zero) wherever the
//       term is small enough, so the streaming loop issues no constant loads and ~half the fp64 instructions.
#ifndef SMCB_MATH_HOST_TEST      // tests/math_host.cpp compiles this header for the CPU with its own shim
#include "smcb_common.cuh"
#endif
#include "smcb_math_coeffs.inc"

#include "smcb_tables.h"

namespace smcb {

constexpr double kRintMagic = 6755399441055744.0;  // 1.5 * 2^52: x + magic rounds x to nearest int

// polynomial evaluation (Horner: N-1 dependent FMAs)
template <int N>
__device__ __forceinline__ double horner(const double (&c)[N], double x) {
    double p = c[N - 1];
#pragma unroll
    for (int i = N - 2; i >= 0; i--) p = fma(p, x, c[i]);
    return p;
}

// exp(x): x <= ~709; returns 0 for x < -708 (incl. -inf; the lost range is < 3e-308),
// +inf for x > 709, NaN for NaN.
__device__ __forceinline__ double fexp(double x) {
    const double t = fma(x, SMCB_LOG2E, kRintMagic);
    const double kd = t - kRintMagic;
    const int k = __double2loint(t);                       // low word of t holds the integer
    double r = fma(kd, -SMCB_LN2_HI, x);
    r = fma(kd, -SMCB_LN2_LO, r);
    const double p = horner(kExpC, r);
    const double scale = __hiloint2double((k + 1023) << 20, 0);   // 2^k, k in [-1022, 1023]
    double res = p * scale;
    res = (x < -708.0) ? 0.0 : res;
    res = (x > 709.0) ? CUDART_INF : res;
    return res;
}

// exp(x) for x <= 0 (weights relative to their maximum): no overflow branch
__device__ __forceinline__ double fexp_neg(double x) {
    const double t = fma(x, SMCB_LOG2E, kRintMagic);
    const double kd = t - kRintMagic;
    const int k = __double2loint(t);
    double r = fma(kd, -SMCB_LN2_HI, x);
    r = fma(kd, -SMCB_LN2_LO, r);
    const double p = horner(kExpC, r);
    const double res = p * __hiloint2double((k + 1023) << 20, 0);
    return (x < -708.0) ? 0.0 : res;
}

// exp(x) for |x| < 700 guaranteed by the caller's domain (no range selects at all); -inf -> NaN!
__device__ __forceinline__ double fexp_mid(double x) {
    const double t = fma(x, SMCB_LOG2E, kRintMagic);
    const double kd = t - kRintMagic;
    const int k = __double2loint(t);
    double r = fma(kd, -SMCB_LN2_HI, x);
    r = fma(kd, -SMCB_LN2_LO, r);
    return horner(kExpC, r) * __hiloint2double((k + 1023) << 20, 0);
}

// log(x) for positive NORMAL x (the 53-bit uniforms of box_muller are >= 2^-54)
__device__ __forceinline__ double flog_pos(double x) {
    int hi = __double2hiint(x), lo = __double2loint(x);
    int e = (hi >> 20) - 1023;
    hi = (hi & 0x000FFFFF) | 0x3FF00000;                   // mantissa in [1, 2)
    const bool big = hi > 0x3FF6A09E;                      // > sqrt(2) (top word compare is enough)
    hi = big ? hi - 0x00100000 : hi;                       // m/2
    e = big ? e + 1 : e;
    const double m = __hiloint2double(hi, lo);
    const double s = (m - 1.0) / (m + 1.0);
    const double z = s * s;
    const double p = horner(kLogC, z);                     // 2 atanh(s) / s
    const double ed = (double)e;
    return fma(ed, SMCB_LN2_HI, fma(s, p, ed * SMCB_LN2_LO));
}

// (sin, cos)(2 pi u) for u in [0, 1)
__device__ __forceinline__ void fsincos2pi(double u, double &s, double &c) {
    const double t4 = u * 4.0;                             // quadrant index = rint(4u) in 0..4
    const double tm = t4 + kRintMagic;
    const double qd = tm - kRintMagic;
    const int q = __double2loint(tm);
    const double r = (t4 - qd) * 0.5;                      // angle = pi (q/2 + r), |r| <= 1/4
    const double z = r * r;
    const double sp = r * horner(kSinPiC, z);              // sin(pi r)
    const double cp = horner(kCosPiC, z);                  // cos(pi r)
    double ss = (q & 1) ? cp : sp;
    double cc = (q & 1) ? sp : cp;
    s = (q & 2) ? -ss : ss;
    c = ((q + 1) & 2) ? -cc : cc;
}

// two N(0,1) from one Philox block (Box-Muller), fast fp64 path
__device__ __forceinline__ void box_muller_fast(const uint32_t r[4], double &z0, double &z1) {
    const double u1 = u53_open(r[0], r[1]);
    const double u2 = u53(r[2], r[3]);
    const double rad = sqrt(-2.0 * flog_pos(u1));
    double s, c;
    fsincos2pi(u2, s, c);
    z0 = rad * c;
    z1 = rad * s;
}

__device__ __forceinline__ void normal_pair_fast(const Philox &key, uint64_t pair, uint32_t t,
                                                 uint32_t comp, double &z0, double &z1) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)pair, (uint32_t)(pair >> 32), t, (comp << 8) | kPurposeNormal, key, r);
    box_muller_fast(r, z0, z1);
}

// ===========================================================================
// table-assisted family (step kernels): tables of smcb_tables.h at the start of dynamic shared memory
// ===========================================================================
#ifdef SMCB_MATH_HOST_TEST
static const double *g_mtab_host = nullptr;
static inline const double *mtab() { return g_mtab_host; }
static inline double rsqrt_approx(double a) {       // what MUFU.RSQ64H delivers: ~22 good bits
    double y = 1.0 / sqrt(a);
    uint64_t b; std::memcpy(&b, &y, 8); b &= 0xFFFFFFFFC0000000ull; std::memcpy(&y, &b, 8);
    return y;
}
#else
__device__ __forceinline__ const double *mtab() {
    extern __shared__ __align__(128) double s_dyn[];
    return s_dyn;
}
__device__ __forceinline__ double rsqrt_approx(double a) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
    return y;
}
// stage the tables: ONE thread arms the barrier and issues the bulk copy; everybody waits before first use
__device__ __forceinline__ void mtab_issue(const double *gsrc, uint64_t *bar) {
    mbar_init(bar, 1);
    mbar_init_fence();
    mbar_arrive_expect_tx(bar, (uint32_t)kMathTabBytes);
    tma_bulk_g2s(const_cast<double *>(mtab()), gsrc, (uint32_t)kMathTabBytes, bar);
}
// stage the tables of a CTA whose dynamic shared memory starts with them: issue, then everybody waits
__device__ __forceinline__ void stage_math_tables(const double *gsrc, uint64_t *bar) {
    if (threadIdx.x == 0) mtab_issue(gsrc, bar);
    __syncthreads();
    mbar_wait(bar, 0);
}
#endif

constexpr double kExpScaleT = (double)kExpTabN * SMCB_LOG2E;
constexpr double kLn2HiT = SMCB_LN2_HI / kExpTabN, kLn2LoT = SMCB_LN2_LO / kExpTabN;   // power-of-two scalings: exact
constexpr double kImmSixth = 0x1.55555p-3;        // 1/6 to 21 bits: an fp64 immediate (term r^3/6 <= 1e-13)
constexpr double kThird = 0.33333333333333333333;
constexpr double kImmFifth = 0x1.99999p-3;        // 1/5 to 21 bits (term r^5/5 <= 1.1e-14 r)
constexpr double kTwoPiOverN = 6.283185307179586476925286766559 / kScTabN;
constexpr double kSinC3 = -0.16666666666666666667;
constexpr double kImmSinC5 = 0x1.11111p-7;        // 1/120 to 21 bits (term d^5/120 <= 2.3e-15 d)
constexpr double kImmCosC4 = 0x1.55555p-5;        // 1/24 to 21 bits (term d^4/24 <= 3.7e-12)

// exp(x) = 2^(k >> 12) T[k & 4095] (1 + r + r^2/2 + r^3/6), x = (k / 4096) ln2 + r, |r| <= ln2 / 8192:
// truncation r^4/24 <= 2.2e-18.  The power of two is applied to the exponent field (integer add).
__device__ __forceinline__ double texp_core(double x) {
    const double t = fma(x, kExpScaleT, kRintMagic);
    const double kd = t - kRintMagic;
    const int k = __double2loint(t);                       // |k| < 2^22 for |x| <= 709
    double r = fma(kd, -kLn2HiT, x);
    r = fma(kd, -kLn2LoT, r);
    const double tj = mtab()[kTabExp + (k & (kExpTabN - 1))];
    const double h = fma(r, kImmSixth, 0.5);
    const double em1 = fma(r * r, h, r);
    const double v = fma(tj, em1, tj);                     // in [1, 2)
    return __hiloint2double(__double2hiint(v) + ((k >> kExpTabBits) << 20), __double2loint(v));
}
// same with the power of two clamped to the normal range (two integer min / max instead of two fp64 selects):
// the result SATURATES at ~2^-1022 / ~2^1024 instead of reaching 0 / +inf; +-inf and a NaN with a zero low word give
// NaN, a NaN with other payloads may give a finite value (see texp).  For arguments that are finite by construction (a
// model's exp of a finite state, a finite log-weight minus its maximum).
__device__ __forceinline__ double texp_sat(double x) {
    const double t = fma(x, kExpScaleT, kRintMagic);
    const double kd = t - kRintMagic;
    const int k = __double2loint(t);
    double r = fma(kd, -kLn2HiT, x);
    r = fma(kd, -kLn2LoT, r);
    const double tj = mtab()[kTabExp + (k & (kExpTabN - 1))];
    const double h = fma(r, kImmSixth, 0.5);
    const double em1 = fma(r * r, h, r);
    const double v = fma(tj, em1, tj);
    // K >> 12 from BOTH words of the magic sum (its mantissa is 2^51 + K): right for |x| up to ~1e9
    int q = (int)__funnelshift_r((unsigned int)k, (unsigned int)__double2hiint(t), kExpTabBits);
    q = q < -1022 ? -1022 : q;
    q = q > 1023 ? 1023 : q;
    return __hiloint2double(__double2hiint(v) + (q << 20), __double2loint(v));
}

// x <= ~709; 0 for x < -708 (incl. -inf), +inf for x > 709, NaN for NaN of any payload.  texp_core adds the power of
// two to the exponent field, so a NaN whose low word is all ones (0x7FFFFFFFFFFFFFFF) comes out of it as DBL_MAX (the
// NaN an H100 makes of -inf - -inf has a zero low word, but a NaN may come from anywhere); the last select passes
// x + inf instead, which is +inf above 709 and NaN for a NaN.
__device__ __forceinline__ double texp(double x) {
    double res = texp_core(x);
    res = (x < -708.0) ? 0.0 : res;
    res = (x <= 709.0) ? res : x + CUDART_INF;
    return res;
}
// x <= 0 (weights relative to their maximum): no overflow select
__device__ __forceinline__ double texp_neg(double x) {
    const double res = texp_core(x);
    return (x < -708.0) ? 0.0 : res;
}

// log(x) for positive NORMAL x: mantissa cell j of m, r = m / c_j - 1 (|r| <= 2^-11),
// log1p(r) = r - r^2/2 + r^3/3 - r^4/4 + r^5/5 (truncation r^6/6 <= 2.3e-21), no division.  Next to 1 the two
// table terms cancel: absolute error <= ~3e-19 there, <= 3 ulp elsewhere (it feeds Box-Muller only)
__device__ __forceinline__ double tlog_pos(double x) {
    const int hi = __double2hiint(x), lo = __double2loint(x);
    const int mant = hi & 0x000FFFFF;
    const int j = mant >> (20 - kLogTabBits);
    const bool big = j >= kLogSplit;
    const int e = (hi >> 20) - 1023 + (big ? 1 : 0);
    const double m = __hiloint2double(mant | (big ? 0x3FE00000 : 0x3FF00000), lo);
    const double *L = mtab() + kTabLog + 2 * j;
    const double inv = L[0], nl = L[1];
    const double r = fma(m, inv, -1.0);
    const double p = fma(r, fma(r, fma(r, kImmFifth, -0.25), kThird), -0.5);
    const double l1p = fma(r * r, p, r);
    const double ed = (double)e;
    return fma(ed, SMCB_LN2_HI, nl + fma(ed, SMCB_LN2_LO, l1p));
}

// sqrt(a), a > 0 normal: reciprocal square root seed + one third-order step, no special-case path (~2 ulp)
__device__ __forceinline__ double tsqrt_pos(double a) {
    const double y0 = rsqrt_approx(a);
    const double e = fma(-a, y0 * y0, 1.0);                // 1 - a y0^2, |e| ~ 2^-21
    const double y = fma(y0 * e, fma(e, 0.375, 0.5), y0);  // y0 (1 + e/2 + 3 e^2/8)
    return a * y;
}

// (sin, cos)(2 pi u), u in [0, 1): angle = 2 pi j / 1024 + d, |d| <= pi / 1024; table rotation by short series
__device__ __forceinline__ void tsincos2pi(double u, double &s, double &c) {
    const double t = fma(u, (double)kScTabN, kRintMagic);
    const double jd = t - kRintMagic;
    const int j = __double2loint(t) & (kScTabN - 1);
    const double d = fma(u, (double)kScTabN, -jd) * kTwoPiOverN;      // the fma is exact
    const double z = d * d;
    const double *S = mtab() + kTabSc + 2 * j;
    const double sj = S[0], cj = S[1];
    const double sd = fma(d * z, fma(z, kImmSinC5, kSinC3), d);      // sin d
    const double cm1 = z * fma(z, kImmCosC4, -0.5);                  // cos d - 1
    s = sj + fma(sj, cm1, cj * sd);
    c = cj + fma(cj, cm1, -(sj * sd));
}

// two N(0,1) from one Philox block (Box-Muller) with the table family
__device__ __forceinline__ void box_muller_tab(const uint32_t r[4], double &z0, double &z1) {
    const double u1 = u53_open(r[0], r[1]);
    const double u2 = u53(r[2], r[3]);
    const double rad = tsqrt_pos(-2.0 * tlog_pos(u1));
    double s, c;
    tsincos2pi(u2, s, c);
    z0 = rad * c;
    z1 = rad * s;
}

__device__ __forceinline__ void normal_pair_tab(const Philox &key, uint64_t pair, uint32_t t,
                                                uint32_t comp, double &z0, double &z1) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)pair, (uint32_t)(pair >> 32), t, (comp << 8) | kPurposeNormal, key, r);
    box_muller_tab(r, z0, z1);
}

// the models' exp (smcb_models.cuh): the table family -- models only run inside the step kernels.  Saturating:
// exp(-x) of a log-volatility beyond +-708 clamps at 2^+-1023, which the weight algebra treats like inf / 0.
__device__ __forceinline__ double mexp(double x) { return texp_sat(x); }

// true iff v is +-inf or NaN (integer test on the exponent field: no fp64 pipe)
__device__ __forceinline__ bool nonfinite(double v) { return (__double2hiint(v) & 0x7FF00000) == 0x7FF00000; }

// ---------------------------------------------------------------------------
// (max, sum exp, sum exp^2) accumulation of a small batch with ONE exp per value:
// the running shift m only moves when the batch maximum exceeds it (one extra exp per
// batch at most, amortised over NV values), instead of a rescale test per value.
// Values equal to -inf (or masked-out slots set to -inf) contribute exactly 0.
// ---------------------------------------------------------------------------
// (table family: step kernels only)
template <int NV>
__device__ __forceinline__ void lse3_add_batch(Lse3 &a, const double (&v)[NV]) {
    double mb = v[0];
#pragma unroll
    for (int j = 1; j < NV; j++) mb = fmax(mb, v[j]);
    if (mb > a.m) {                       // also the first time (a.m = -inf): fexp(-inf) = 0
        const double r = texp_neg(a.m - mb);
        a.s *= r;
        a.q *= r * r;
        a.m = mb;
    }
    if (a.m == -CUDART_INF) return;       // nothing but -inf so far
#pragma unroll
    for (int j = 0; j < NV; j++) {
        const double e = texp_neg(v[j] - a.m);
        a.s += e;
        a.q = fma(e, e, a.q);
    }
}

// the same with the polynomial family (stand-alone kernels: no shared-memory tables)
template <int NV>
__device__ __forceinline__ void lse3_add_batch_f(Lse3 &a, const double (&v)[NV]) {
    double mb = v[0];
#pragma unroll
    for (int j = 1; j < NV; j++) mb = fmax(mb, v[j]);
    if (mb > a.m) {
        const double r = fexp_neg(a.m - mb);
        a.s *= r;
        a.q *= r * r;
        a.m = mb;
    }
    if (a.m == -CUDART_INF) return;
#pragma unroll
    for (int j = 0; j < NV; j++) {
        const double e = fexp_neg(v[j] - a.m);
        a.s += e;
        a.q = fma(e, e, a.q);
    }
}

}  // namespace smcb
