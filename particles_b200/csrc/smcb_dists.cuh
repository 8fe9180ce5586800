// smcb_dists.cuh -- the device log-densities of the univariate laws of distributions.py, and the samplers of those
// whose draws come from here: InvGamma, LogNormal, TruncNormal, Binomial, Geometric, NegativeBinomial,
// DiscreteUniform and Gamma (the sampler InvGamma, NegativeBinomial and Dirichlet draw through) have both; Normal,
// Student, Laplace and Logistic have their log-density here and draw elsewhere.  Every function is
// __host__ __device__: the library's kernels (smcb_dists.cu) and the CPU harness of the tests (tests/dists_host.cpp,
// g++ -ffp-contract=off) compile this same header, so the host build replays the device's values and draws.
//
// Randomness: the draw of element i reads Philox blocks with counter (i lo, block, call lo, (i hi << 8) | purpose)
// under the context's key, `call` = the API call number.  A rejection sampler's k-th trial always reads the same
// blocks, so the draws do not depend on the launch geometry.  Sub-samplers of one element (the Poisson draw of a
// NegativeBinomial) start at block kSubStream.
#pragma once
#ifndef SMCB_DISTS_HOST_TEST
#include "smcb_common.cuh"
#endif

namespace smcb {
namespace dists {

#define SMCB_HD __host__ __device__ __forceinline__

// law codes (include/smcb.h, distributions.py); the codes below kNumSampled have a sampler here
enum : int {
    kInvGamma = 0, kLogNormal = 1, kTruncNormal = 2, kBinomial = 3, kGeometric = 4, kNegBinomial = 5,
    kDiscreteUniform = 6, kGamma = 7, kNormal = 8, kStudent = 9, kLaplace = 10, kLogistic = 11, kNumLaws = 12,
    kNumSampled = 8,
};
SMCB_HD constexpr bool discrete_law(int law) { return law >= kBinomial && law <= kDiscreteUniform; }

constexpr double kLogSqrt2Pi = 0.91893853320467274178;   // log(2 pi) / 2
constexpr double kLog2Pi = 1.8378770664093454836;
constexpr double kSqrtHalf = 0.70710678118654752440;
constexpr double kMaxCount = 9007199254740992.0;           // 2^53: counts above are not integers in fp64
constexpr uint32_t kMaxTrials = 1u << 16;                   // a rejection sampler gives NaN after as many failures
constexpr uint32_t kSubStream = 1u << 24;

SMCB_HD double nan_() { return __builtin_nan(""); }
SMCB_HD double inf_() { return __builtin_inf(); }
SMCB_HD bool is_int(double v) { return floor(v) == v && fabs(v) < inf_(); }

// ---------------------------------------------------------------------------
// counter-based draws
// ---------------------------------------------------------------------------
struct Rng {
    uint32_t k0, k1, call;
    uint64_t elem;
    SMCB_HD void block(uint32_t b, uint32_t r[4]) const {
        philox4x32_10((uint32_t)elem, b, call, ((uint32_t)(elem >> 32) << 8) | kPurposeDists, k0, k1, r);
    }
    SMCB_HD double uniform(uint32_t b) const {        // (0, 1)
        uint32_t r[4];
        block(b, r);
        return u53_open(r[0], r[1]);
    }
    SMCB_HD void uniform2(uint32_t b, double &u, double &v) const {
        uint32_t r[4];
        block(b, r);
        u = u53_open(r[0], r[1]);
        v = u53_open(r[2], r[3]);
    }
    SMCB_HD double normal(uint32_t b) const {         // Box-Muller, cosine branch
        uint32_t r[4];
        block(b, r);
        double s, c;
        sincospi(2.0 * u53(r[2], r[3]), &s, &c);
        return sqrt(-2.0 * log(u53_open(r[0], r[1]))) * c;
    }
};

// ---------------------------------------------------------------------------
// log-densities: scipy.stats' values and conventions (NaN outside the parameter domain or at x = NaN, -inf outside
// the support, -inf at non-integer x for the discrete laws)
// ---------------------------------------------------------------------------
// scipy.stats.invgamma.logpdf(x, a, scale=b)
SMCB_HD double invgamma_logpdf(double x, double a, double b) {
    if (!(a > 0.0) || !(b > 0.0) || x != x) return nan_();
    if (!(x > 0.0) || x == inf_()) return -inf_();
    const double y = x / b;
    return -(a + 1.0) * log(y) - lgamma(a) - 1.0 / y - log(b);
}

// scipy.stats.lognorm.logpdf(x, sigma, scale=exp(mu))
SMCB_HD double lognormal_logpdf(double x, double mu, double sigma) {
    if (!(sigma > 0.0) || x != x || mu != mu) return nan_();
    if (!(x > 0.0) || x == inf_()) return -inf_();
    const double z = (log(x) - mu) / sigma;
    return -0.5 * z * z - log(sigma) - log(x) - kLogSqrt2Pi;
}

// log of the N(0, 1) mass above t >= 0: erfc while it is a normal number, the asymptotic series of the Mills ratio
// beyond (its 10th term is < 1e-19 at t = 25)
SMCB_HD double log_norm_sf(double t) {
    if (t < 25.0) return log(0.5 * erfc(t * kSqrtHalf));
    const double r = 1.0 / (t * t);
    double s = 1.0, term = 1.0;
    for (int k = 1; k <= 10; k++) {
        term *= -(2.0 * k - 1.0) * r;
        s += term;
    }
    return -0.5 * t * t - log(t) - kLogSqrt2Pi + log(s);
}
// log(1 - exp(x)), x <= 0, without cancellation at either end
SMCB_HD double log1mexp(double x) { return x > -0.6931471805599453 ? log(-expm1(x)) : log1p(-exp(x)); }

// log of the N(0, 1) mass of [l, u], l < u, in log space: finite for intervals in either far tail.  A narrow
// interval (w (1 + |c|) < 1e-3) takes the midpoint series phi(c) w (1 + He2(c) w^2 / 24 + He4(c) w^4 / 1920),
// whose next term is < 1e-15: the difference of two tail masses would lose the digits of w.
SMCB_HD double truncnorm_logmass(double l, double u) {
    const double w = u - l, c = 0.5 * (l + u);
    if (w * (1.0 + fabs(c)) < 1e-3) {
        const double c2 = c * c, w2 = w * w;
        return -0.5 * c2 - kLogSqrt2Pi + log(w) +
               log1p((c2 - 1.0) * w2 / 24.0 + ((c2 - 6.0) * c2 + 3.0) * (w2 * w2) / 1920.0);
    }
    if (l >= 0.0) {
        const double ll = log_norm_sf(l);
        return ll + log1mexp(log_norm_sf(u) - ll);
    }
    if (u <= 0.0) {
        const double lu = log_norm_sf(-u);
        return lu + log1mexp(log_norm_sf(-l) - lu);
    }
    return log(0.5 * (erf(u * kSqrtHalf) - erf(l * kSqrtHalf)));
}

// scipy.stats.truncnorm.logpdf(x, (a - mu) / sigma, (b - mu) / sigma, loc=mu, scale=sigma)
SMCB_HD double truncnorm_logpdf(double x, double mu, double sigma, double a, double b) {
    const double l = (a - mu) / sigma, u = (b - mu) / sigma;
    if (!(sigma > 0.0) || !(l < u) || x != x) return nan_();
    const double z = (x - mu) / sigma;
    if (z < l || z > u) return -inf_();
    return -0.5 * z * z - kLogSqrt2Pi - log(sigma) - truncnorm_logmass(l, u);
}

// Loader's saddle-point form of the binomial probability ("Fast and accurate computation of binomial
// probabilities", 2000): no difference of lgamma values, so it keeps its digits at n = 10^6 and beyond.
// stirlerr(k / 2), k = 0 .. 30 (mpmath, 20 digits)
__device__ const double kStirlerrHalves[31] = {
    0.0, 0.15342640972002734529, 0.08106146679532725822, 0.054814121051917653896,
    0.041340695955409294094, 0.033162873519936287485, 0.027677925684998339149,
    0.023746163656297495971, 0.020790672103765093112, 0.018488450532673185231,
    0.016644691189821192163, 0.015134973221917378874, 0.013876128823070747999,
    0.012810465242920226924, 0.011896709945891770095, 0.011104559758206917327,
    0.010411265261972096497, 0.0097994161261588032984, 0.0092554621827127329177,
    0.008768700134139385463, 0.0083305634333628712565, 0.0079341145643140205472,
    0.007573675487951840795, 0.0072445543013203831795, 0.0069428401072095298657,
    0.0066652470327076824424, 0.0064089941880042070684, 0.0061717122630394576475,
    0.0059513701127588477356, 0.005746216513010115682, 0.005554733551962801371};
// stirlerr(n) = log(n!) - log(sqrt(2 pi n) (n / e)^n)
SMCB_HD double stirlerr(double n) {
    constexpr double S0 = 1.0 / 12.0, S1 = 1.0 / 360.0, S2 = 1.0 / 1260.0, S3 = 1.0 / 1680.0, S4 = 1.0 / 1188.0;
    if (n <= 15.0) {
        const double nn = n + n;
#if defined(__CUDA_ARCH__) || defined(SMCB_DISTS_HOST_TEST)     // (nvcc's host pass never runs it)
        if (nn == floor(nn)) return kStirlerrHalves[(int)nn];        // a global (L1-cached) read: the index varies
#endif
        return lgamma(n + 1.0) - (n + 0.5) * log(n) + n - kLogSqrt2Pi;
    }
    const double r = 1.0 / n, r2 = r * r;                            // one division
    if (n > 500.0) return (S0 - S1 * r2) * r;
    if (n > 80.0) return (S0 - (S1 - S2 * r2) * r2) * r;
    if (n > 35.0) return (S0 - (S1 - (S2 - S3 * r2) * r2) * r2) * r;
    return (S0 - (S1 - (S2 - (S3 - S4 * r2) * r2) * r2) * r2) * r;
}
// bd0(x, np) = x log(x / np) + np - x, by its series where the two terms cancel
SMCB_HD double bd0(double x, double np) {
    if (fabs(x - np) < 0.1 * (x + np)) {
        double v = (x - np) / (x + np);
        double s = (x - np) * v;
        double ej = 2.0 * x * v;
        v = v * v;
        for (int j = 1; j < 1000; j++) {
            ej *= v;
            const double s1 = s + ej / (2 * j + 1);
            if (s1 == s) return s1;
            s = s1;
        }
        return s;
    }
    return x * log(x / np) + np - x;
}
// log of the binomial probability of x successes in n trials, q = 1 - p (x, n need not be integers)
SMCB_HD double binom_raw_log(double x, double n, double p, double q) {
    if (p == 0.0) return x == 0.0 ? 0.0 : -inf_();
    if (q == 0.0) return x == n ? 0.0 : -inf_();
    if (x == 0.0) {
        if (n == 0.0) return 0.0;
        return p < 0.1 ? -bd0(n, n * q) - n * p : n * log(q);
    }
    if (x == n) return q < 0.1 ? -bd0(n, n * p) - n * q : n * log(p);
    if (x < 0.0 || x > n) return -inf_();
    const double lc = stirlerr(n) - stirlerr(x) - stirlerr(n - x) - bd0(x, n * p) - bd0(n - x, n * q);
    const double lf = kLog2Pi + log(x) + log1p(-x / n);
    return lc - 0.5 * lf;
}

// scipy.stats.binom.logpmf(x, n, p)
SMCB_HD double binomial_logpmf(double x, double n, double p) {
    if (!(n >= 0.0) || !is_int(n) || !(p >= 0.0 && p <= 1.0) || x != x) return nan_();
    if (!is_int(x) || x < 0.0 || x > n) return -inf_();
    return binom_raw_log(x, n, p, 1.0 - p);
}

// scipy.stats.geom.logpmf(x, p): support 1, 2, ...
SMCB_HD double geometric_logpmf(double x, double p) {
    if (!(p > 0.0 && p <= 1.0) || x != x) return nan_();
    if (!is_int(x) || x < 1.0) return -inf_();
    return (x == 1.0 ? 0.0 : (x - 1.0) * log1p(-p)) + log(p);
}

// scipy.stats.nbinom.logpmf(x, n, p): the number of failures before the n-th success, n > 0 real
SMCB_HD double nbinom_logpmf(double x, double n, double p) {
    if (!(n > 0.0) || n == inf_() || !(p > 0.0 && p <= 1.0) || x != x) return nan_();
    if (x == inf_()) return nan_();                                     // scipy's value at +inf
    if (!is_int(x) || x < 0.0) return -inf_();
    return log(n / (n + x)) + binom_raw_log(n, x + n, p, 1.0 - p);
}

// scipy.stats.randint.logpmf(x, lo, hi): lo, ..., hi - 1
SMCB_HD double discrete_uniform_logpmf(double x, double lo, double hi) {
    if (!is_int(lo) || !is_int(hi) || !(hi > lo) || x != x) return nan_();
    if (!is_int(x) || x < lo || x >= hi) return -inf_();
    return -log(hi - lo);
}

// The laws of state-space models' PX / PY: scipy's formulas without its parameter checks.  Their lgamma terms come
// from the host as c0 (scipy's gammaln), not from the device's lgamma.
// scipy.stats.norm.logpdf(x, loc, scale), in the operation order of SURVEY.md section 9 item 2
SMCB_HD double normal_logpdf(double x, double loc, double scale) {
    const double z = (x - loc) / scale;
    return -z * z / 2.0 - kLogSqrt2Pi - log(scale);
}

// scipy.stats.t.logpdf(x, df, loc, scale); c0 = gammaln((df + 1) / 2) - gammaln(df / 2) - log(df pi) / 2
SMCB_HD double student_logpdf(double x, double df, double loc, double scale, double c0) {
    const double z = (x - loc) / scale;
    return c0 - 0.5 * (df + 1.0) * log1p(z * z / df) - log(scale);
}

// scipy.stats.gamma.logpdf(x, a, scale=1 / b); c0 = -gammaln(a).  scipy's xlogy(a - 1, x): the term is 0 when
// a == 1, also at x = 0 and x = +inf; at x = 0 it is +inf for a < 1 and -inf for a > 1, and x = +inf gives -inf for
// a <= 1 and NaN (inf - inf) for a > 1
SMCB_HD double gamma_logpdf(double x, double a, double b, double c0) {
    const double xl = (a == 1.0) ? 0.0 : (a - 1.0) * log(x);
    return (x != x) ? x : (x >= 0.0) ? a * log(b) + c0 + xl - b * x : -inf_();
}

// scipy.stats.laplace.logpdf(x, loc, scale)
SMCB_HD double laplace_logpdf(double x, double loc, double scale) {
    return -log(2.0 * scale) - fabs(x - loc) / scale;
}

// scipy.stats.logistic.logpdf(x, loc, scale) in scipy's symmetric form: exp(-|z|) cannot overflow
SMCB_HD double logistic_logpdf(double x, double loc, double scale) {
    const double y = -fabs((x - loc) / scale);
    return y - 2.0 * log1p(exp(y)) - log(scale);
}

SMCB_HD double law_logpdf(int law, double x, double p0, double p1, double p2, double p3) {
    switch (law) {
        case kInvGamma: return invgamma_logpdf(x, p0, p1);
        case kLogNormal: return lognormal_logpdf(x, p0, p1);
        case kTruncNormal: return truncnorm_logpdf(x, p0, p1, p2, p3);
        case kBinomial: return binomial_logpmf(x, p0, p1);
        case kGeometric: return geometric_logpmf(x, p0);
        case kNegBinomial: return nbinom_logpmf(x, p0, p1);
        case kDiscreteUniform: return discrete_uniform_logpmf(x, p0, p1);
        case kGamma: return gamma_logpdf(x, p0, p1, p2);
        case kNormal: return normal_logpdf(x, p0, p1);
        case kStudent: return student_logpdf(x, p0, p1, p2, p3);
        case kLaplace: return laplace_logpdf(x, p0, p1);
        default: return logistic_logpdf(x, p0, p1);
    }
}

// ---------------------------------------------------------------------------
// samplers (blocks from `base` on)
// ---------------------------------------------------------------------------
// Gamma(a, rate b): Marsaglia & Tsang (2000); a < 1 draws Gamma(a + 1) and multiplies by U^(1/a).  Trial k reads
// blocks base + 2k (the normal) and base + 2k + 1 (the acceptance uniform, words 0-1); the boost uniform is words
// 2-3 of block base + 1, which no trial reads.
// The Marsaglia-Tsang draw of Gamma(aa, 1), aa >= 1
SMCB_HD double mt_gamma(const Rng &g, uint32_t base, double aa) {
    const double d = aa - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
    for (uint32_t k = 0; k < kMaxTrials; k++) {
        const double z = g.normal(base + 2 * k);
        const double t = 1.0 + c * z;
        if (t <= 0.0) continue;
        const double v = t * t * t;
        const double u = g.uniform(base + 2 * k + 1);
        if (log(u) < 0.5 * z * z + d - d * v + d * log(v)) return d * v;
    }
    return nan_();
}
// the boost uniform of a < 1
SMCB_HD double gamma_boost_u(const Rng &g, uint32_t base) {
    uint32_t r[4];
    g.block(base + 1, r);
    return u53_open(r[2], r[3]);
}
SMCB_HD double gamma_rvs(const Rng &g, uint32_t base, double a, double b) {
    if (!(a > 0.0) || !(b > 0.0)) return nan_();
    double x = mt_gamma(g, base, a < 1.0 ? a + 1.0 : a);
    if (a < 1.0) x *= pow(gamma_boost_u(g, base), 1.0 / a);
    return x / b;
}
// log of the same Gamma(a, 1) draw, in log space throughout: finite where the draw itself underflows to 0 (the
// boost U^(1/a) of a ~ 1e-3 is below 1e-308 for most U)
SMCB_HD double gamma_log_rvs(const Rng &g, uint32_t base, double a) {
    if (!(a > 0.0)) return nan_();
    double lx = log(mt_gamma(g, base, a < 1.0 ? a + 1.0 : a));
    if (a < 1.0) lx += log(gamma_boost_u(g, base)) / a;
    return lx;
}

// Poisson(lam): inversion below lam = 10, PTRS (Hoermann 1993, "The transformed rejection method for generating
// Poisson random variables") above, one block per trial
SMCB_HD double poisson_rvs(const Rng &g, uint32_t base, double lam) {
    if (!(lam >= 0.0) || lam == inf_()) return nan_();
    if (lam == 0.0) return 0.0;
    if (lam < 10.0) {
        const double u = g.uniform(base);
        double p = exp(-lam), F = p, k = 0.0;
        while (u > F) {
            k += 1.0;
            p *= lam / k;
            if (p == 0.0) break;
            F += p;
        }
        return k;
    }
    const double slam = sqrt(lam), loglam = log(lam);
    const double b = 0.931 + 2.53 * slam, a = -0.059 + 0.02483 * b;
    const double invalpha = 1.1239 + 1.1328 / (b - 3.4), vr = 0.9277 - 3.6224 / (b - 2.0);
    for (uint32_t t = 0; t < kMaxTrials; t++) {
        double U, V;
        g.uniform2(base + t, U, V);
        U -= 0.5;
        const double us = 0.5 - fabs(U);
        const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
        if (us >= 0.07 && V <= vr) return k;
        if (k < 0.0 || (us < 0.013 && V > us)) continue;
        if (log(V) + log(invalpha) - log(a / (us * us) + b) <= -lam + k * loglam - lgamma(k + 1.0)) return k;
    }
    return nan_();
}

// Binomial(n, p): inversion from 0 while n min(p, q) < 10, BTRS (Hoermann 1993, "The generation of binomial random
// variates") otherwise; on min(p, q), reflected for p > 1/2
SMCB_HD double binomial_rvs(const Rng &g, double n, double p) {
    if (!(n >= 0.0) || !is_int(n) || !(p >= 0.0 && p <= 1.0)) return nan_();
    if (n == 0.0 || p == 0.0) return 0.0;
    if (p == 1.0) return n;
    const bool flip = p > 0.5;
    const double pp = flip ? 1.0 - p : p, q = 1.0 - pp;
    double k = nan_();
    if (n * pp < 10.0) {
        const double u = g.uniform(0);
        const double r = pp / q;
        double pk = exp(n * log1p(-pp)), F = pk;
        k = 0.0;
        while (u > F && k < n) {
            pk *= (n - k) / (k + 1.0) * r;
            k += 1.0;
            if (pk == 0.0) break;
            F += pk;
        }
    } else {
        const double spq = sqrt(n * pp * q);
        const double b = 1.15 + 2.53 * spq, a = -0.0873 + 0.0248 * b + 0.01 * pp, c = n * pp + 0.5;
        const double vr = 0.92 - 4.2 / b, alpha = (2.83 + 5.1 / b) * spq, lpq = log(pp / q);
        const double m = floor((n + 1.0) * pp), h = lgamma(m + 1.0) + lgamma(n - m + 1.0);
        for (uint32_t t = 0; t < kMaxTrials; t++) {
            double U, V;
            g.uniform2(t, U, V);
            U -= 0.5;
            const double us = 0.5 - fabs(U);
            const double kk = floor((2.0 * a / us + b) * U + c);
            if (kk < 0.0 || kk > n) continue;
            if (us >= 0.07 && V <= vr) { k = kk; break; }
            const double lv = log(V * alpha / (a / (us * us) + b));
            if (lv <= h - lgamma(kk + 1.0) - lgamma(n - kk + 1.0) + (kk - m) * lpq) { k = kk; break; }
        }
    }
    return flip ? n - k : k;
}

// N(0, 1) restricted to [l, u], exact (Robert 1995, "Simulation of truncated normal variables"): an interval that
// holds 0 by normal rejection (or uniform proposals when it is shorter than sqrt(2 pi)); an interval on one side of
// 0 by uniform proposals when (u^2 - l^2) / 2 < 1, whose acceptance is then > 1/e whatever its width, and by the
// translated-exponential proposal with Robert's optimal rate otherwise.  Only exp and log of finite arguments: finite
// in either far tail, and a narrow interval keeps its digits.  One block per trial.
SMCB_HD double truncnorm_std_rvs(const Rng &g, double l, double u) {
    const bool neg = u <= 0.0;
    if (neg) {
        const double t = l;
        l = -u;
        u = -t;
    }
    for (uint32_t k = 0; k < kMaxTrials; k++) {
        double z;
        if (l < 0.0) {
            if (u - l >= 2.5066282746310002) {
                z = g.normal(k);
                if (z < l || z > u) continue;
            } else {
                double a, v;
                g.uniform2(k, a, v);
                z = l + a * (u - l);
                if (v > exp(-0.5 * z * z)) continue;
            }
        } else if ((u - l) * (u + l) < 2.0) {
            double a, v;
            g.uniform2(k, a, v);
            z = l + a * (u - l);
            if (v > exp(-0.5 * (z - l) * (z + l))) continue;
        } else {
            const double alpha = 0.5 * (l + sqrt(l * l + 4.0));
            double a, v;
            g.uniform2(k, a, v);
            z = l - log(a) / alpha;
            if (z > u) continue;
            const double e = z - alpha;
            if (v > exp(-0.5 * e * e)) continue;
        }
        return neg ? -z : z;
    }
    return nan_();
}

SMCB_HD double truncnorm_rvs(const Rng &g, double mu, double sigma, double a, double b) {
    const double l = (a - mu) / sigma, u = (b - mu) / sigma;
    if (!(sigma > 0.0) || !(l < u)) return nan_();
    const double x = mu + sigma * truncnorm_std_rvs(g, l, u);
    return fmin(fmax(x, a), b);      // rounding of mu + sigma z never leaves [a, b]
}

SMCB_HD double law_rvs(int law, const Rng &g, double p0, double p1, double p2, double p3) {
    switch (law) {
        case kInvGamma: {                                       // b / Gamma(a, 1)
            if (!(p1 > 0.0)) return nan_();
            return p1 / gamma_rvs(g, 0, p0, 1.0);
        }
        case kLogNormal:
            if (!(p1 > 0.0)) return nan_();
            return exp(p0 + p1 * g.normal(0));
        case kTruncNormal: return truncnorm_rvs(g, p0, p1, p2, p3);
        case kBinomial: return binomial_rvs(g, p0, p1);
        case kGeometric: {                                      // ceil(log U / log(1 - p))
            if (!(p0 > 0.0 && p0 <= 1.0)) return nan_();
            if (p0 == 1.0) return 1.0;
            return fmin(fmax(ceil(log(g.uniform(0)) / log1p(-p0)), 1.0), kMaxCount);
        }
        case kNegBinomial: {                                    // Poisson(Gamma(n, scale (1 - p) / p)), as NumPy
            if (!(p0 > 0.0) || !(p1 > 0.0 && p1 <= 1.0)) return nan_();
            if (p1 == 1.0) return 0.0;
            return fmin(poisson_rvs(g, kSubStream, gamma_rvs(g, 0, p0, p1 / (1.0 - p1))), kMaxCount);
        }
        case kDiscreteUniform: {                                // lo + floor(U (hi - lo))
            if (!is_int(p0) || !is_int(p1) || !(p1 > p0)) return nan_();
            uint32_t r[4];
            g.block(0, r);
            return fmin(p0 + floor(u53(r[0], r[1]) * (p1 - p0)), p1 - 1.0);
        }
        default: return gamma_rvs(g, 0, p0, p1);
    }
}

#undef SMCB_HD
}  // namespace dists
}  // namespace smcb
