"""The laws of particles_b200/csrc/smcb_dists.cuh compiled for the CPU by tests/dists_host.cpp: log-densities against
scipy.stats (and mpmath where scipy itself loses digits), samplers by Kolmogorov-Smirnov / chi-square tests on 10^6
draws from the library's Philox counters, and the host-side parts of the new laws of particles_b200.distributions
(posterior formulas, Cond in a StructDist, the NegativeBinomial deviation from the reference)."""
import ctypes as C
import os
import subprocess

import mpmath as mp
import numpy as np
import pytest
from scipy import stats
from scipy.special import gammaln

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_build")
INVGAMMA, LOGNORMAL, TRUNCNORMAL, BINOMIAL, GEOMETRIC, NEGBINOMIAL, DUNIFORM, GAMMA = range(8)
NORMAL, STUDENT, LAPLACE, LOGISTIC = range(8, 12)
SEED = 20261018

_lib = None


def build_dists_host():
    """g++ build of tests/dists_host.cpp (smcb_dists.cuh compiled for the host)."""
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "libdists_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "dists_host.cpp"), "-o", so])
        _lib = C.CDLL(so)
        _lib.dh_rvs.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_long] + [C.c_void_p] * 5 + [C.c_long]
        _lib.dh_dirichlet_rvs.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_int, C.c_void_p, C.c_long]
    return _lib


def _arr(v, n):
    return None if v is None else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (n,)))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def host_logpdf(law, x, *params):
    x = np.atleast_1d(np.asarray(x, dtype=np.float64))
    n = max([x.size] + [np.size(p) for p in params])
    ps = [_arr(p, n) for p in params] + [None] * (4 - len(params))
    xs, out = _arr(x, n), np.empty(n)
    build_dists_host().dh_logpdf(law, _p(xs), *[_p(a) for a in ps], _p(out), C.c_long(n))
    return out


def host_rvs(law, n, *params, seed=SEED, call=0, offset=0):
    ps = [_arr(p, n) for p in params] + [None] * (4 - len(params))
    out = np.empty(n)
    build_dists_host().dh_rvs(law, seed, call, offset, *[_p(a) for a in ps], _p(out), n)
    return out


def host_dirichlet_rvs(alpha, n, seed=SEED, call=0):
    alpha = np.ascontiguousarray(alpha, dtype=np.float64)
    out = np.empty((n, alpha.size))
    build_dists_host().dh_dirichlet_rvs(seed, call, _p(alpha), alpha.size, _p(out), n)
    return out


def close(got, ref, rtol=1e-12, atol=1e-12):
    """relative rtol, absolute atol near zero; NaN / inf must sit at the same places with the same sign"""
    got, ref = np.broadcast_arrays(np.asarray(got, float), np.asarray(ref, float))
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (got[np.isnan(got) != np.isnan(ref)], ref)
    assert np.array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)])
    err = np.abs(got[fin] - ref[fin])
    ok = err <= np.maximum(rtol * np.abs(ref[fin]), atol)
    assert ok.all(), (got[fin][~ok][:5], ref[fin][~ok][:5])


# ----------------------------------------------------------------------------------------------------- log-densities
def test_invgamma_lognormal_logpdf():
    x = np.concatenate([[-1.0, 0.0, np.nan, np.inf, 1e-300, 1e300], np.geomspace(1e-6, 1e4, 400)])
    for a, b in [(0.3, 1.0), (1.0, 1.0), (2.5, 0.7), (40.0, 3.0)]:
        close(host_logpdf(INVGAMMA, x, a, b), stats.invgamma.logpdf(x, a, scale=b))
    for mu, s in [(0.0, 1.0), (-2.0, 0.3), (5.0, 2.5)]:
        with np.errstate(divide="ignore"):
            close(host_logpdf(LOGNORMAL, x, mu, s), stats.lognorm.logpdf(x, s, scale=np.exp(mu)))
    # per-element parameters, and parameters outside the domain: NaN as scipy
    r = np.random.RandomState(1)
    xs, a, b = r.gamma(2.0, 1.0, 1000), r.uniform(0.2, 9.0, 1000), r.uniform(0.1, 5.0, 1000)
    close(host_logpdf(INVGAMMA, xs, a, b), stats.invgamma.logpdf(xs, a, scale=b))
    close(host_logpdf(LOGNORMAL, xs, a - 4.0, b), stats.lognorm.logpdf(xs, b, scale=np.exp(a - 4.0)))
    assert np.isnan(host_logpdf(INVGAMMA, [1.0, 1.0], [0.0, 1.0], [1.0, -1.0])).all()
    assert np.isnan(host_logpdf(LOGNORMAL, [1.0], 0.0, 0.0)).all()


def student_c0(df):
    """the host-computed constant of Student's log-density (its lgamma terms)"""
    return gammaln(0.5 * (df + 1.0)) - gammaln(0.5 * df) - 0.5 * np.log(df * np.pi)


def test_normal_student_gamma_laplace_logistic_logpdf():
    """the laws of state-space models' PX / PY against scipy: NaN, +-inf, 0, negative x (Gamma's xlogy cases at
    a < 1, a == 1, a > 1), |z| near 700 (Logistic's exp(-|z|) form), scalar and per-element parameters"""
    x = np.concatenate([[-np.inf, -700.0, -3.0, -0.0, 0.0, 1e-300, np.inf, np.nan, 699.5, 700.5, 710.0],
                        np.linspace(-8.0, 12.0, 81)])
    mid = x[~(np.abs(x) > 600.0)]          # scipy's laplace.logpdf is the log of its pdf: -inf once that underflows
    with np.errstate(all="ignore"):
        for loc, s in [(0.0, 1.0), (0.5, 2.0), (-3.0, 0.1)]:
            close(host_logpdf(NORMAL, x, loc, s), stats.norm.logpdf(x, loc, s))
            close(host_logpdf(LAPLACE, mid, loc, s), stats.laplace.logpdf(mid, loc, s))
            close(host_logpdf(LOGISTIC, x, loc, s), stats.logistic.logpdf(x, loc, s))
            for df in (1.0, 2.5, 30.0):
                close(host_logpdf(STUDENT, x, df, loc, s, student_c0(df)), stats.t.logpdf(x, df, loc, s))
        for a, b in [(0.4, 2.0), (1.0, 1.0), (1.0, 0.3), (3.5, 2.0), (40.0, 5.0)]:
            close(host_logpdf(GAMMA, x, a, b, -gammaln(a)), stats.gamma.logpdf(x, a, scale=1.0 / b))
    r = np.random.RandomState(7)
    n = 2000
    xs, loc, s, df = r.normal(0.0, 3.0, n), r.normal(size=n), r.uniform(0.1, 4.0, n), r.uniform(0.5, 50.0, n)
    close(host_logpdf(NORMAL, xs, loc, s), stats.norm.logpdf(xs, loc, s))
    close(host_logpdf(STUDENT, xs, df, loc, s, student_c0(df)), stats.t.logpdf(xs, df, loc, s))
    close(host_logpdf(LAPLACE, xs, loc, s), stats.laplace.logpdf(xs, loc, s))
    close(host_logpdf(LOGISTIC, xs, loc, s), stats.logistic.logpdf(xs, loc, s))
    a, b, g = r.uniform(0.2, 9.0, n), r.uniform(0.1, 5.0, n), r.gamma(2.0, 1.0, n)
    close(host_logpdf(GAMMA, g, a, b, -gammaln(a)), stats.gamma.logpdf(g, a, scale=1.0 / b))


def _truncnorm_mp(x, mu, s, a, b):
    """log-density of N(mu, s^2) on [a, b] in 50-digit arithmetic"""
    with mp.workdps(50):
        x, mu, s, a, b = (mp.mpf(float(v)) for v in (x, mu, s, a, b))
        if x < a or x > b:
            return -np.inf
        l, u = (a - mu) / s, (b - mu) / s
        mass = (mp.ncdf(u) - mp.ncdf(l)) if l < 0 else (mp.erfc(l / mp.sqrt(2)) - mp.erfc(u / mp.sqrt(2))) / 2
        z = (x - mu) / s
        return float(-z * z / 2 - mp.log(mp.sqrt(2 * mp.pi)) - mp.log(s) - mp.log(mass))


def test_truncnorm_logpdf_tails_and_narrow():
    cases = [(0.0, 1.0, a, np.inf) for a in (0.0, 3.0, 8.0, 30.0, 40.0)]
    cases += [(0.0, 1.0, -np.inf, -a) for a in (0.0, 3.0, 8.0, 30.0, 35.0, 40.0)]          # mirrored
    cases += [(0.0, 1.0, -1.0, 2.0), (1.0, 2.0, -3.0, 0.5), (0.5, 0.5, -1.0, 1.0), (0.0, 1.0, 30.0, 31.0)]
    cases += [(0.0, 1.0, a, a + 1e-8) for a in (-1.0, 0.0, 2.0, 9.0, 35.0)]                   # b - a = 1e-8
    cases += [(0.0, 1.0, a, a + 1e-4) for a in (0.3, 4.0, 20.0)]
    for mu, s, a, b in cases:
        lo = a if np.isfinite(a) else (b - 12.0 * s if not np.isfinite(a) else a)
        hi = b if np.isfinite(b) else a + 12.0 * s
        x = np.concatenate([np.linspace(lo, hi, 25), [a - 1e-3 if np.isfinite(a) else -1e300, np.nan]])
        x = x[np.isfinite(x) | np.isnan(x)]
        ref = np.array([np.nan if np.isnan(v) else _truncnorm_mp(v, mu, s, a, b) for v in x])
        close(host_logpdf(TRUNCNORMAL, x, mu, s, a, b), ref)
    # agrees with scipy where scipy itself is exact, per-element parameters included
    r = np.random.RandomState(2)
    mu, s = r.normal(size=500), r.uniform(0.2, 3.0, 500)
    a, b = mu - r.uniform(0.1, 3.0, 500) * s, mu + r.uniform(0.1, 3.0, 500) * s
    x = a + r.rand(500) * (b - a)
    close(host_logpdf(TRUNCNORMAL, x, mu, s, a, b), stats.truncnorm.logpdf(x, (a - mu) / s, (b - mu) / s, mu, s))
    assert np.isnan(host_logpdf(TRUNCNORMAL, [0.5, 0.5], 0.0, [1.0, -1.0], [1.0, 0.0], [0.0, 1.0])).all()


def test_discrete_logpmf_edges():
    x = np.array([-1.0, 0.0, 0.5, 1.0, 2.0, 3.0, 7.0, 10.0, 11.0, 50.0, np.nan, np.inf, 2.0000001])
    for n, p in [(10, 0.3), (10, 0.0), (10, 1.0), (0, 0.5), (50, 0.999), (3, 1e-9)]:
        with np.errstate(divide="ignore", invalid="ignore"):
            close(host_logpdf(BINOMIAL, x, n, p), stats.binom.logpmf(x, n, p))
    for p in (0.3, 1.0, 1e-6, 0.999):
        with np.errstate(divide="ignore", invalid="ignore"):
            close(host_logpdf(GEOMETRIC, x, p), stats.geom.logpmf(x, p))
    for n, p in [(1.0, 0.5), (3.5, 0.3), (0.2, 0.9), (20.0, 1.0), (7.0, 1e-3)]:
        with np.errstate(divide="ignore", invalid="ignore"):
            close(host_logpdf(NEGBINOMIAL, x, n, p), stats.nbinom.logpmf(x, n, p))
    for lo, hi in [(0, 2), (-3, 11), (2, 3)]:
        close(host_logpdf(DUNIFORM, x, lo, hi), stats.randint.logpmf(x, lo, hi))
    # parameters outside the domain: NaN, as scipy
    for law, pars in [(BINOMIAL, (2.5, 0.5)), (BINOMIAL, (5, 1.5)), (GEOMETRIC, (0.0,)), (NEGBINOMIAL, (0.0, 0.5)),
                      (NEGBINOMIAL, (2.0, 0.0)), (DUNIFORM, (3, 3))]:
        assert np.isnan(host_logpdf(law, [1.0], *pars)).all()
    # per-element parameters
    r = np.random.RandomState(3)
    n, p = r.randint(0, 200, 2000).astype(float), r.rand(2000)
    k = np.floor(r.rand(2000) * (n + 1))
    close(host_logpdf(BINOMIAL, k, n, p), stats.binom.logpmf(k, n, p))
    nn = r.uniform(0.1, 40.0, 2000)
    close(host_logpdf(NEGBINOMIAL, k, nn, p), stats.nbinom.logpmf(k, nn, p))


def test_binomial_negbinomial_large_n_against_mpmath():
    def binom_mp(k, n, p):
        with mp.workdps(40):
            k, n, p = mp.mpf(k), mp.mpf(n), mp.mpf(p)
            return float(mp.loggamma(n + 1) - mp.loggamma(k + 1) - mp.loggamma(n - k + 1) + k * mp.log(p)
                         + (n - k) * mp.log1p(-p))

    def nbinom_mp(k, n, p):
        with mp.workdps(40):
            k, n, p = mp.mpf(k), mp.mpf(n), mp.mpf(p)
            return float(mp.loggamma(n + k) - mp.loggamma(k + 1) - mp.loggamma(n) + n * mp.log(p)
                         + k * mp.log1p(-p))

    for n, p in [(1e6, 0.5), (1e6, 0.01), (1e6, 0.999), (123457, 0.3)]:
        m = n * p
        ks = np.unique(np.clip(np.round(m + np.array([-5, -1, 0, 1, 2, 5, 50]) * np.sqrt(m * (1 - p) + 1)), 0, n))
        got = host_logpdf(BINOMIAL, ks, n, p)
        np.testing.assert_allclose(got, [binom_mp(k, n, p) for k in ks], rtol=0, atol=1e-9)
    for n, p in [(1e6, 0.5), (2.5e5 + 0.5, 0.9), (3.7, 1e-4)]:
        m = n * (1 - p) / p
        ks = np.unique(np.clip(np.round(m + np.array([-3, -1, 0, 1, 4]) * np.sqrt(m / p + 1)), 0, None))
        got = host_logpdf(NEGBINOMIAL, ks, n, p)
        np.testing.assert_allclose(got, [nbinom_mp(k, n, p) for k in ks], rtol=0, atol=1e-9)


# ---------------------------------------------------------------------------------------------------------- samplers
N_GOF = 1_000_000
P_MIN = 1e-4


def ks_p(u):
    """KS p-value of values that should be U(0, 1)"""
    return stats.kstest(u, "uniform").pvalue


def chi2_p(draws, pmf_of, support_lo):
    """chi-square p-value of integer draws against the pmf of a law whose support starts at support_lo: bins from
    there up, those with fewer than 20 expected merged into the two tails (the upper one takes all the mass above)"""
    draws = draws.astype(np.int64)
    assert draws.min() >= support_lo
    ks = np.arange(support_lo, int(draws.max()) + 1)
    expct = pmf_of(ks) * draws.size
    obs = np.bincount(draws - support_lo, minlength=ks.size).astype(float)
    keep = expct >= 20
    first, last = np.argmax(keep), ks.size - 1 - np.argmax(keep[::-1])
    e = expct[first:last + 1].copy()
    o = obs[first:last + 1].copy()
    e[0] += expct[:first].sum()
    o[0] += obs[:first].sum()
    e[-1] += draws.size - expct[:last + 1].sum()
    o[-1] += obs[last + 1:].sum()
    return stats.chisquare(o, e).pvalue


@pytest.mark.parametrize("a", [0.3, 1.0, 4.5, 150.0])
def test_gamma_sampler_ks(a):
    x = host_rvs(GAMMA, N_GOF, a, 2.0)
    assert np.isfinite(x).all() and (x > 0).all()
    assert ks_p(stats.gamma.cdf(x, a, scale=0.5)) > P_MIN


def test_continuous_samplers_ks():
    x = host_rvs(INVGAMMA, N_GOF, 2.5, 1.5, call=1)
    assert ks_p(stats.invgamma.cdf(x, 2.5, scale=1.5)) > P_MIN
    x = host_rvs(LOGNORMAL, N_GOF, -1.0, 0.7, call=2)
    assert ks_p(stats.lognorm.cdf(x, 0.7, scale=np.exp(-1.0))) > P_MIN
    # per-element parameters: the probability-integral transform F_i(x_i)
    r = np.random.RandomState(4)
    a, b = r.uniform(0.2, 6.0, N_GOF), r.uniform(0.1, 4.0, N_GOF)
    x = host_rvs(INVGAMMA, N_GOF, a, b, call=3)
    assert ks_p(stats.invgamma.cdf(x, a, scale=b)) > P_MIN


@pytest.mark.parametrize("mu,s,a,b", [(0.0, 1.0, 0.0, np.inf), (0.0, 1.0, -1.0, 2.0), (0.0, 1.0, 3.0, 3.5),
                                      (0.0, 1.0, 8.0, np.inf), (0.0, 1.0, 40.0, np.inf), (0.0, 1.0, -np.inf, -38.0),
                                      (2.0, 0.5, 1.0, 1.0 + 1e-8), (0.0, 1.0, -0.2, 0.1), (1.0, 3.0, -np.inf, 1.5)])
def test_truncnorm_sampler_ks(mu, s, a, b):
    x = host_rvs(TRUNCNORMAL, N_GOF, mu, s, a, b, call=5)
    assert np.isfinite(x).all() and (x >= a).all() and (x <= b).all()
    l, u = (a - mu) / s, (b - mu) / s
    z = (x - mu) / s
    if l > 5:            # far right tail: the exact conditional cdf of the excess, in closed form via log sf ratios
        with mp.workdps(30):
            sfl = mp.erfc(l / mp.sqrt(2))
            cdf = np.array([float(1 - mp.erfc(v / mp.sqrt(2)) / sfl) for v in z[:20000]])
        assert ks_p(cdf) > P_MIN
    elif u < -5:
        with mp.workdps(30):
            cu = mp.erfc(-u / mp.sqrt(2))
            cdf = np.array([float(mp.erfc(-v / mp.sqrt(2)) / cu) for v in z[:20000]])
        assert ks_p(cdf) > P_MIN
    elif b - a < 1e-6:   # narrow interval: the draws are uniform across it to first order
        assert ks_p((x - a) / (b - a)) > P_MIN
    else:
        assert ks_p(stats.truncnorm.cdf(x, l, u, mu, s)) > P_MIN


@pytest.mark.parametrize("n,p", [(10, 0.3), (30, 0.3), (34, 0.3), (1000, 0.02), (1000, 0.5), (50, 0.9),
                                 (10**6, 0.4), (7, 0.999)])
def test_binomial_sampler_chi2(n, p):
    x = host_rvs(BINOMIAL, N_GOF, n, p, call=6)
    assert (x >= 0).all() and (x <= n).all() and (x == np.floor(x)).all()
    assert chi2_p(x, lambda k: stats.binom.pmf(k, n, p), 0) > P_MIN


@pytest.mark.parametrize("n,p", [(1.0, 0.5), (3.5, 0.3), (0.4, 0.05), (25.0, 0.2), (1000.0, 0.9)])
def test_negbinomial_sampler_chi2(n, p):
    x = host_rvs(NEGBINOMIAL, N_GOF, n, p, call=7)
    assert (x >= 0).all() and (x == np.floor(x)).all()
    assert chi2_p(x, lambda k: stats.nbinom.pmf(k, n, p), 0) > P_MIN


def test_geometric_discrete_uniform_samplers_chi2():
    x = host_rvs(GEOMETRIC, N_GOF, 0.2, call=8)
    assert x.min() >= 1 and chi2_p(x, lambda k: stats.geom.pmf(k, 0.2), 1) > P_MIN
    x = host_rvs(DUNIFORM, N_GOF, -3, 17, call=9)
    assert x.min() >= -3 and x.max() <= 16 and chi2_p(x, lambda k: stats.randint.pmf(k, -3, 17), -3) > P_MIN


def test_dirichlet_sampler_marginals():
    alpha = np.array([0.5, 2.0, 3.5])
    x = host_dirichlet_rvs(alpha, 300_000)
    np.testing.assert_allclose(x.sum(1), 1.0, rtol=1e-14)
    for j in range(3):       # marginals are Beta(alpha_j, sum - alpha_j)
        assert ks_p(stats.beta.cdf(x[:, j], alpha[j], alpha.sum() - alpha[j])) > P_MIN


def test_harness_philox_matches_reference_generator():
    """the harness's restatement of the library's Philox4x32-10, 53-bit uniforms and Box-Muller normal, block by
    block, against tests/philox_ref.py (the counters of smcb_dists.cuh: (elem lo, block, call, (elem hi << 8) | 8))"""
    import philox_ref as pr
    lib = build_dists_host()
    lib.dh_block.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.dh_block_draws.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
    for seed, call, elem, block in [(0, 0, 0, 0), (SEED, 3, 12345, 7), (2**64 - 1, 2**31, 2**40 + 5, 2**24 + 1),
                                    (77, 0, 199_999, 131073)]:
        got = np.empty(4, dtype=np.uint32)
        lib.dh_block(seed, call, elem, block, _p(got))
        ref = pr.philox4x32_10(elem & 0xFFFFFFFF, block, call & 0xFFFFFFFF, ((elem >> 32) << 8) | 8,
                               seed & 0xFFFFFFFF, seed >> 32)
        assert np.array_equal(got, np.array([int(np.asarray(v)) for v in ref], dtype=np.uint32))
        draws = np.empty(2)
        lib.dh_block_draws(seed, call, elem, block, _p(draws))
        r = [np.asarray(v, dtype=np.uint32) for v in ref]
        assert draws[0] == pr.u53_open(r[0], r[1])
        z = np.sqrt(-2.0 * np.log(pr.u53_open(r[0], r[1]))) * np.cos(2 * np.pi * pr.u53(r[2], r[3]))
        np.testing.assert_allclose(draws[1], z, rtol=1e-12, atol=1e-15)


def test_dirichlet_small_alphas_stay_finite():
    """rows of alpha = 1e-3, whose Gamma draws all underflow, are normalised in log space: finite, on the simplex,
    and with the Beta(a_j, sum - a_j) marginals"""
    alpha = np.array([1e-3, 1e-3, 2e-3])
    x = host_dirichlet_rvs(alpha, 200_000, call=13)
    assert np.isfinite(x).all()
    np.testing.assert_allclose(x.sum(1), 1.0, rtol=1e-14)
    # almost every row puts all its mass on one coordinate, with probability a_j / sum(a)
    top = np.argmax(x, axis=1)
    np.testing.assert_allclose(np.bincount(top, minlength=3) / x.shape[0], alpha / alpha.sum(), atol=5e-3)


def test_draws_depend_on_counters_only():
    """element i's draw is the same whatever the other elements are, and changes with the call number"""
    a = host_rvs(BINOMIAL, 1000, 50, 0.4, call=11)
    b = host_rvs(BINOMIAL, 10, 50, 0.4, call=11, offset=500)
    assert np.array_equal(a[500:510], b)
    assert not np.array_equal(a, host_rvs(BINOMIAL, 1000, 50, 0.4, call=12))


# --------------------------------------------------------------------------------------- host side of the new laws
def test_posteriors_match_reference_formulas():
    from particles_b200 import distributions as D
    r = np.random.RandomState(5)
    x = r.normal(1.0, 2.0, 37)
    post = D.Normal(loc=0.5, scale=2.0).posterior(x, sigma=1.5)
    pr0, prd = 1 / 4.0, 37 / 1.5 ** 2
    varp = 1 / (pr0 + prd)
    np.testing.assert_allclose([post.loc, post.scale], [varp * (pr0 * 0.5 + prd * x.mean()), np.sqrt(varp)],
                               rtol=1e-15)
    g = D.Gamma(a=2.0, b=3.0).posterior(x)
    assert (g.a, g.b) == (2.0 + 0.5 * 37, 3.0 + 0.5 * np.sum(x ** 2))
    ig = D.InvGamma(a=2.0, b=3.0).posterior(x)
    assert isinstance(ig, D.InvGamma) and (ig.a, ig.b) == (2.0 + 0.5 * 37, 3.0 + 0.5 * np.sum(x ** 2))
    tn = D.TruncNormal(mu=0.5, sigma=0.5, a=-1.0, b=1.0).posterior(x, s=2.0)
    pr0, prd = 4.0, 37 / 4.0
    varp = 1 / (pr0 + prd)
    np.testing.assert_allclose([tn.mu, tn.sigma], [varp * (pr0 * 0.5 + prd * x.mean()), np.sqrt(varp)], rtol=1e-15)
    assert (tn.a, tn.b) == (-1.0, 1.0)
    X = r.normal(size=(20, 2))
    cov, Sig = np.array([[2.0, 0.3], [0.3, 1.0]]), np.array([[1.0, 0.2], [0.2, 0.5]])
    mv = D.MvNormal(loc=np.array([0.1, -0.2]), cov=cov).posterior(X, Sigma=Sig)
    Sp = np.linalg.inv(np.linalg.inv(cov) + 20 * np.linalg.inv(Sig))
    mp_ = Sp @ (np.array([0.1, -0.2]) @ np.linalg.inv(cov) + np.linalg.inv(Sig) @ X.sum(0))
    np.testing.assert_allclose(mv.cov, Sp, rtol=1e-12)
    np.testing.assert_allclose(mv.loc, mp_, rtol=1e-12)
    with pytest.raises(ValueError):
        D.MvNormal(loc=np.zeros(2), scale=2.0, cov=cov).posterior(X)


def test_cond_in_structdist_dtype():
    from particles_b200 import distributions as D
    law = D.StructDist({"rho": D.Uniform(0.0, 1.0), "sigma": D.Cond(lambda th: D.Gamma(b=1.0 / th["rho"]))})
    assert law.dtype == [("rho", float), ("sigma", float)]
    c = D.Cond(lambda th: D.Normal(), dim=1, dtype="float64")
    assert (c.dim, c.dtype) == (1, "float64") and isinstance(c(None), D.Normal)
    assert issubclass(D.Poisson, D.DiscreteDist) and issubclass(D.Categorical, D.DiscreteDist)
    for cls in (D.Binomial, D.Geometric, D.NegativeBinomial, D.DiscreteUniform):
        assert issubclass(cls, D.DiscreteDist) and cls.dtype == np.int64


def test_negbinomial_deviation_from_reference():
    """The reference's NegativeBinomial.logpdf is nbinom.logpmf(x, p, n): it does not describe its own draws
    (numpy's negative_binomial(n, p)); this package's logpdf is nbinom.logpmf(x, n, p), which does."""
    n, p = 3.5, 0.3
    draws = np.random.RandomState(6).negative_binomial(n, p, size=400_000)
    ks = np.arange(0, 60)
    freq = np.bincount(draws, minlength=ks.size)[:ks.size] / draws.size
    ours = np.exp(host_logpdf(NEGBINOMIAL, ks, n, p))
    with np.errstate(all="ignore"):
        theirs = np.exp(stats.nbinom.logpmf(ks, p, n))
    assert np.abs(freq - ours).max() < 3e-3
    assert np.abs(freq - np.nan_to_num(theirs)).max() > 0.05
    close(np.log(ours), stats.nbinom.logpmf(ks, n, p))
