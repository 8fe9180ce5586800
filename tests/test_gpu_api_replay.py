"""The stand-alone kernels of ``csrc/smcb_api.cu`` against their long-double replay (tests/api_replay.py): the weight
reductions at every grid and batch-loop edge, ``wmean_and_var`` at every component-chunk edge up to d = 32, every
resampling scheme at M << N and on NS-like weights (the search's unstaged branch), the log-densities at their tails
and edges, and the device's own draws restated from their Philox counters.  Each case asserts the branch or regime
it is meant to reach."""
import functools

import numpy as np
import pytest

import api_replay as ar

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SEED = 0x5EED0123456789AB


@pytest.fixture(scope="module")
def pb():
    import particles_b200 as pb
    return pb


@pytest.fixture
def ctx(pb):
    from particles_b200.device import context
    c = context()
    c.seed(SEED)                                  # API call counter back to 0
    return c


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------ reductions
SAT = 256 * 4 * ar.MAX_GRID                       # n where grid_for(n, 1024) saturates
BATCH = 7 * ar.MAX_GRID * ar.BLOCK                # n above which thread 0 runs the 8-wide batch loop once
SIZES = [1, 2, 7, 255, 256, 257, SAT - 1, SAT, SAT + 1, BATCH, BATCH + 1, 8 * ar.MAX_GRID * ar.BLOCK + 1, 10_000_000]


def _lw(n, kind, seed):
    r = np.random.RandomState(seed)
    if kind == "gauss":
        lw = r.randn(n) * 4.0
        lw[n // 3: n // 3 + n // 10] = -np.inf               # a block of -inf
    elif kind == "single":
        lw = np.full(n, -np.inf)
        lw[r.randint(n)] = 3.5
    elif kind == "spread":
        lw = -1400.0 * r.rand(n)                               # W down to subnormal and flushed
        lw[0] = 0.0
    else:
        raise ValueError(kind)
    return lw


def _check_reductions(pb, lw):
    from particles_b200 import resampling as rs
    n = lw.size
    lwd = dev(lw)
    w = rs.Weights(lw=lwd)
    stats = host(w._stats)
    ar.check_weights(lw, host(lwd), stats, host(w.W))
    fin = ar.fix_nan(lw)
    for mode, f in (("sum", rs.log_sum_exp), ("mean", rs.log_mean_exp), ("essl", rs.essl)):
        val, b = ar.lse_ref(fin, mode)
        ar.within(f"{mode} n={n}", f(dev(fin)), np.atleast_1d(val), b)
    Wn = np.random.RandomState(n % 977).rand(n)
    Wn[::5] = 0.0
    val, b = ar.lse_ref(fin, "wmean", W=Wn)
    ar.within(f"weighted n={n}", rs.log_mean_exp(dev(fin), W=dev(Wn)), np.atleast_1d(val), b)
    W, bW = ar.exp_normalise_ref(fin)
    ar.within(f"exp_and_normalise n={n}", host(rs.exp_and_normalise(dev(fin))), W, bW)


@pytest.mark.parametrize("n", SIZES)
def test_reductions_at_grid_and_batch_edges(pb, n):
    grid = ar.grid_for(n, 1024)
    stride = grid * ar.BLOCK
    if n >= SAT:
        assert grid == ar.MAX_GRID
    assert (n > 7 * stride) == (n > BATCH)        # whether any thread runs the batch loop
    _check_reductions(pb, _lw(n, "gauss", n % 1000))


@pytest.mark.parametrize("kind", ["single", "spread"])
@pytest.mark.parametrize("n", [1, 257, BATCH + 1])
def test_reductions_single_entry_and_subnormal_weights(pb, kind, n):
    lw = _lw(n, kind, 3)
    if kind == "spread" and n > 1:
        W = host(pb.resampling.exp_and_normalise(dev(lw)))
        assert (W == 0).any() and np.isfinite(lw).all()          # the exponential's flushed tail is reached
    _check_reductions(pb, lw)


def test_reductions_nan_and_infinities_follow_the_reference(pb):
    """NaN anywhere, +inf anywhere, or every entry -inf: NaN from log_sum_exp, log_mean_exp (with and without W),
    essl and exp_and_normalise, whichever CTA or lane holds the odd value; Weights rewrites NaN to -inf in place."""
    from particles_b200 import resampling as rs
    cases = [np.array([np.nan, 0.0]), np.array([0.0, np.nan]), np.full(7, -np.inf), np.array([0.0, np.inf, 1.0]),
             np.concatenate([np.full(5000, -np.inf), [np.nan], np.zeros(3000)]),
             np.concatenate([np.zeros(300_000), [np.inf]])]
    for v in cases:
        for f in (rs.log_sum_exp, rs.log_mean_exp, rs.essl):
            assert np.isnan(f(dev(v))), (f.__name__, v.size)
        assert np.isnan(rs.log_mean_exp(dev(v), W=dev(np.full(v.size, 1.0 / v.size)))), v.size
        assert np.isnan(host(rs.exp_and_normalise(dev(v)))).all(), v.size
    lw = np.concatenate([np.full(5000, -np.inf), [np.nan], np.zeros(3000)])
    lwd = dev(lw)
    w = rs.Weights(lw=lwd)
    ar.check_weights(lw, host(lwd), host(w._stats), host(w.W))
    for bad in (np.full(5, -np.inf), np.array([0.0, np.inf, 1.0])):
        wb = rs.Weights(lw=dev(bad))
        assert np.isnan(wb.ESS) and np.isnan(wb.log_mean)


# ------------------------------------------------------------------------------------------- moments
WM_DIMS = [1, 2, 3, 4, 5, 8, 9, 15, 16, 17, 20, 32]
CAP = ar.WMOM_GRID * ar.BLOCK * 4                  # n from which k_wmoments runs its 592 CTAs


@pytest.mark.parametrize("d", WM_DIMS)
def test_wmoments_every_component_chunk(pb, d):
    from particles_b200 import resampling as rs
    r = np.random.RandomState(d)
    for n in (1, 2, 255, 511, 512, 513, CAP - 1, CAP + 1):
        grid, k = ar.wmoments_geometry(n)
        assert (grid == ar.WMOM_GRID) == (n > CAP - ar.BLOCK * 4)
        W = r.rand(n) ** 3
        W[r.rand(n) < 0.25] = 0.0                   # exact zeros
        W[0] = max(W[0], 1e-3)
        x = r.randn(n, d) * np.linspace(0.5, 3.0, d) + (1e6 if n % 2 else 0.0)  # offset data on odd n
        out = rs.wmean_and_var(dev(W), dev(x))
        got = np.concatenate([np.atleast_1d(out["mean"]), np.atleast_1d(out["var"])])
        ar.check_wmoments(W, x, got)


def test_wmoments_large_n_one_dimensional(pb):
    from particles_b200 import resampling as rs
    r = np.random.RandomState(0)
    n = 3_000_001
    W = r.rand(n)
    x = 1e6 + r.randn(n)
    out = rs.wmean_and_var(dev(W), dev(x))
    ar.check_wmoments(W, x, [out["mean"], out["var"]])
    with pytest.raises(Exception):
        rs.wmean_and_var(dev(W[:10]), dev(r.randn(10, 33)))


# ----------------------------------------------------------------------------------------- resampling
def _scratch_views(n, m, scratch):
    s = host(scratch)
    oz = (n + 1) & ~1
    ou = oz + ((m + 3) & ~1)
    return s[:n], s[oz:oz + m + 2], s[ou:ou + m + 2]


def _run_scheme(scheme, W, M, u=None):
    from particles_b200 import resampling as rs
    A, scratch = rs._resample(scheme, dev(W), M, u=u, return_scratch=True)
    return host(A), _scratch_views(W.size, M, scratch)


def _ns_weights(n, zero_frac, seed):
    """NS-SMC's weights: 0 (log-weight -inf) below the threshold, equal above it."""
    r = np.random.RandomState(seed)
    lw = np.where(r.rand(n) < zero_frac, -np.inf, 0.0)
    lw[r.randint(n)] = 0.0
    return ar.exp_normalise_ref(lw)[0].astype(np.float64)


@functools.lru_cache(maxsize=4)
def _spread_weights(n, seed):
    lw = np.random.RandomState(seed).randn(n) * 3.0
    w = np.exp(lw - lw.max())
    return w / w.sum()


@functools.lru_cache(maxsize=4)
def _cdf_ref(n, seed):
    return ar.cdf_ref(_spread_weights(n, seed))


NU = {"systematic": lambda M: 1, "stratified": lambda M: M, "multinomial": lambda M: M + 1}


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
@pytest.mark.parametrize("M", [1, 1023, 1024, 1025])
def test_inverse_cdf_few_outputs_on_ten_million(pb, ctx, scheme, M):
    """M << N = 10^7: the first tile spans the whole CDF and bisects in global memory (M = 1: one output, staged)."""
    n = 10_000_000
    W = _spread_weights(n, 1)
    u = np.random.RandomState(M).rand(NU[scheme](M))
    A, (cdf, z, _) = _run_scheme(scheme, W, M, u)
    su = z[:M] / z[M] if scheme == "multinomial" else ar.su_of(scheme, u, M)
    br = ar.search_branches(cdf, su)
    assert br.all() if M == 1 else not br[0]
    ar.check_inverse_cdf(scheme, W, M, u, A, cdf=cdf, z=z[:M + 1] if scheme == "multinomial" else None,
                         ref=_cdf_ref(n, 1))


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
@pytest.mark.parametrize("zero_frac", [0.9, 0.999])
@pytest.mark.parametrize("ratio", [1, 10])
def test_inverse_cdf_ns_weights(pb, ctx, scheme, zero_frac, ratio):
    """N = 10^6 NS-SMC weights with 90 % / 99.9 % zeros, interleaved as NS-SMC leaves them.  At M = N a tile's 1024
    outputs span about 1024 N / M entries, so 90 % zeros stay staged, while at 99.9 % the tiles that straddle a run of
    more than 4096 zeros bisect in global memory and the rest stage: both branches in one call.  M = N / 10, the
    waste-free resampling of N particles out of N x len_chain, takes every tile to the unstaged branch.  With 99.9 %
    zeros many scan chunks sum to 0, where the chunk bases once rounded below the previous chunk's values.  The
    device's own uniforms, restated bit for bit."""
    n = 1_000_000
    M = n // ratio
    W = _ns_weights(n, zero_frac, 2)
    A, (cdf, z, u) = _run_scheme(scheme, W, M)
    nu = NU[scheme](M)
    assert np.array_equal(u[:nu], ar.api_uniforms(nu, 0, SEED))
    su = z[:M] / z[M] if scheme == "multinomial" else ar.su_of(scheme, u, M)
    br = ar.search_branches(cdf, su)
    if ratio == 10:
        assert not br[:-1].any()
    else:
        assert br.all() if zero_frac == 0.9 else (br.any() and not br.all())
    decided = ar.check_inverse_cdf(scheme, W, M, u[:nu], A, cdf=cdf, z=z[:M + 1] if scheme == "multinomial" else None)
    assert decided > 0.99 * M


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_inverse_cdf_full_size_own_draws(pb, ctx, scheme):
    n = 10_000_000
    W = _spread_weights(n, 1)
    A, (cdf, z, u) = _run_scheme(scheme, W, n)
    nu = NU[scheme](n)
    assert np.array_equal(u[:nu], ar.api_uniforms(nu, 0, SEED))
    su = z[:n] / z[n] if scheme == "multinomial" else ar.su_of(scheme, u, n)
    assert ar.search_branches(cdf, su).all()
    ar.check_inverse_cdf(scheme, W, n, u[:nu], A, cdf=cdf, z=z[:n + 1] if scheme == "multinomial" else None,
                         ref=_cdf_ref(n, 1))


@pytest.mark.parametrize("case", ["spread", "ns", "integral", "single", "few"])
def test_residual(pb, ctx, case):
    if case == "spread":
        n, M, W = 1_000_003, 1_000_003, _spread_weights(1_000_003, 5)
    elif case == "ns":
        n, M, W = 1_000_000, 1_000_000, _ns_weights(1_000_000, 0.999, 6)
    elif case == "integral":                       # M W integral everywhere: sres = 0
        n, M = 4096, 8192
        W = np.random.RandomState(7).randint(0, 4, n).astype(np.float64)
        W[0] += 8192 - W.sum()
        W /= 8192
    elif case == "single":                         # sres = 1
        n, M = 3, 8
        W = np.array([1.5, 2.5, 4.0]) / 8
    else:                                          # M << N
        n, M, W = 2_000_000, 1025, _spread_weights(2_000_000, 8)
    ip, sip, sres, res = ar.residual_parts(W, M)
    assert {"integral": sres == 0, "single": sres == 1}.get(case, sres > 1)
    A, (cdf, z, u) = _run_scheme("residual", W, M)
    assert np.array_equal(u[:M + 1], ar.api_uniforms(M + 1, 0, SEED))
    ar.check_residual(W, M, u, A, cdf=cdf if sres else None, z=z if sres else None)


@pytest.mark.parametrize("kills", ["few", "many"])
@pytest.mark.parametrize("own", [False, True])
def test_killing(pb, ctx, kills, own):
    from particles_b200 import resampling as rs
    n = 1_000_000
    r = np.random.RandomState(9)
    if kills == "few":
        W = ar.exp_normalise_ref(r.rand(n) * 1e-3)[0].astype(np.float64)     # nearly flat: few kills
    else:
        W = _spread_weights(n, 10)
    if own:
        A = host(rs.killing(dev(W)))
        u = ar.api_uniforms(n, 0, SEED)
        nk = int((u * W.max() >= W).sum())
        um = ar.api_uniforms(nk + 1, 1, SEED)
    else:
        u = r.rand(n)
        nk = int((u * W.max() >= W).sum())
        um = r.rand(nk + 1)
        A = host(rs.killing(dev(W), u=dev(u), u_multinomial=dev(um)))
    assert (nk < 1500) if kills == "few" else (nk > 0.9 * n)
    C, _ = ar.cdf_ref(W)
    if kills == "few":                           # a multinomial draw of nk << N: the unstaged branch
        assert not ar.search_branches(C.astype(np.float64), np.sort(um[:nk]))[0]
    got_nk, decided = ar.check_killing(W, u, um, A)
    assert got_nk == nk and decided > 0.99 * nk


@pytest.mark.parametrize("own", [False, True])
def test_ssp_large(pb, ctx, own):
    from oracle import smc_numpy as orc
    from particles_b200 import resampling as rs
    n = 300_000
    W = _spread_weights(n, 11)
    if own:
        A = host(rs.ssp(dev(W)))
        u = ar.api_uniforms(n - 1, 0, SEED)
    else:
        u = np.random.RandomState(12).rand(n - 1)
        A = host(rs.ssp(dev(W), u=dev(u)))
    assert np.array_equal(A, orc.ssp(W, n, u=u))


# --------------------------------------------------------------------------------------- distributions
Z_LOGISTIC = np.array([-800.0, -709.8, -709.7, -40.0, 0.0, 40.0, 800.0])


def test_logistic_tails(pb):
    """z < -709.78: the overflowing form gave -inf where scipy's symmetric form gives about z."""
    from particles_b200 import distributions as dists
    v, b = ar.logistic_logpdf_ref(Z_LOGISTIC, 0.0, 1.0)
    ar.within("logistic", host(dists.Logistic().logpdf(dev(Z_LOGISTIC))), v, b)
    r = np.random.RandomState(0)
    x = np.concatenate([Z_LOGISTIC * 2.0, r.randn(5000) * 50])
    loc, sc = r.randn(x.size), np.exp(r.randn(x.size) * 0.5)
    v, b = ar.logistic_logpdf_ref(x, loc, sc)
    ar.within("logistic per-particle", host(dists.Logistic(loc=dev(loc), scale=dev(sc)).logpdf(dev(x))), v, b)
    v, b = ar.logistic_logpdf_ref(np.array([np.inf, -np.inf, np.nan]), 0.0, 1.0)
    ar.within("logistic inf", host(dists.Logistic().logpdf(dev(np.array([np.inf, -np.inf, np.nan])))), v, b)


def test_gamma_edges(pb):
    """x in {0, -0, 5e-324, +inf, NaN, < 0} with a in {0.5, 1, 2.5}: scipy's xlogy rules."""
    from scipy.special import gammaln
    from particles_b200 import distributions as dists
    x = np.array([0.0, -0.0, 5e-324, 1e-300, 0.7, 30.0, np.inf, -1.0, -np.inf, np.nan])
    for a in (0.5, 1.0, 2.5):
        for b in (1.0, 3.0):
            v, bd = ar.gamma_logpdf_ref(x, a, -gammaln(a), b)
            ar.within(f"gamma a={a} b={b}", host(dists.Gamma(a=a, b=b).logpdf(dev(x))), v, bd)
    r = np.random.RandomState(1)
    xs = np.abs(r.randn(4000)) * 3
    xs[::50] = 0.0
    bs = np.exp(r.randn(4000))
    v, bd = ar.gamma_logpdf_ref(xs, 1.0, 0.0, bs)
    ar.within("gamma per-particle rate", host(dists.Gamma(a=1.0, b=dev(bs)).logpdf(dev(xs))), v, bd)


def test_student_laplace_normal_tails_and_edges(pb):
    from scipy.special import gammaln
    from particles_b200 import distributions as dists
    x = np.array([1e154, -1e154, 1.34e154, 1.35e154, 1e300, 0.0, 3.0, np.inf, -np.inf, np.nan])
    for df in (1.0, 3.0, 4.5):
        c0 = gammaln(0.5 * (df + 1.0)) - gammaln(0.5 * df) - 0.5 * np.log(df * np.pi)
        v, b = ar.student_logpdf_ref(x, df, c0, 0.0, 1.0)
        ar.within(f"student {df}", host(dists.Student(df=df).logpdf(dev(x))), v, b)
    r = np.random.RandomState(2)
    y = np.concatenate([x, r.randn(3000) * 10, [800.0, -800.0]])
    loc, sc = r.randn(y.size), np.exp(r.randn(y.size) * 0.3)
    v, b = ar.laplace_logpdf_ref(y, loc, sc)
    ar.within("laplace", host(dists.Laplace(loc=dev(loc), scale=dev(sc)).logpdf(dev(y))), v, b)
    v, b = ar.normal_logpdf_ref(y, loc, sc)
    ar.within("normal", host(dists.Normal(loc=dev(loc), scale=dev(sc)).logpdf(dev(y))), v, b)
    v, b = ar.normal_logpdf_ref(y, 0.3, 1.7)
    ar.within("normal scalar", host(dists.Normal(loc=0.3, scale=1.7).logpdf(dev(y))), v, b)


def test_normal_rvs_own_draws(pb, ctx):
    from particles_b200 import distributions as dists
    n = 100_001
    r = np.random.RandomState(3)
    loc, sc = r.randn(n), np.exp(r.randn(n) * 0.3)
    got = host(dists.Normal(loc=dev(loc), scale=dev(sc)).rvs(size=n))
    z, bz = ar.api_normals(n, 0, SEED)
    want = ar._ld(loc) + ar._ld(sc) * z
    ar.within("normal rvs", got, want, ar._ld(sc) * bz + ar.SAFETY * ar.LD(ar.EPS) * (np.abs(want) + ar._ld(sc) * np.abs(z)))
    got = host(dists.Normal(loc=1.5, scale=0.5).rvs(size=77))
    z, bz = ar.api_normals(77, 1, SEED)
    ar.within("normal rvs scalar", got, 1.5 + 0.5 * z, 0.5 * bz + 4 * ar.LD(ar.EPS) * (1.5 + np.abs(z)))


def _ill_cov(d, cond, seed):
    r = np.random.RandomState(seed)
    Q, _ = np.linalg.qr(r.randn(d, d))
    return (Q * np.logspace(0, -np.log10(cond), d)) @ Q.T


@pytest.mark.parametrize("d", [1, 8, 9, 32])
@pytest.mark.parametrize("cond", [10.0, 1e8])
def test_mvnormal(pb, ctx, d, cond):
    """d = 8 is the last dimension of k_mvn_rvs / k_mvn_logpdf, d = 9 the first of k_mvn_big; per-particle loc and
    scale, an ill-conditioned covariance; injected normals, then the device's own in each kernel's counter layout."""
    from particles_b200 import distributions as dists
    cov = _ill_cov(d, cond, d)
    law = dists.MvNormal(loc=np.zeros(d), cov=cov)
    L = law.L
    r = np.random.RandomState(d)
    n = 20_001
    loc, sc = r.randn(n, d), np.exp(r.randn(n, d) * 0.3)
    x = loc + r.randn(n, d) * 2
    v, b = ar.mvn_logpdf_ref(L, x.T, loc.T, sc.T)
    ar.within("mvn logpdf", host(dists.MvNormal(loc=dev(loc), scale=dev(sc), cov=cov).logpdf(dev(x))), v, b)
    s0 = np.linspace(0.5, 2.0, d)
    v, b = ar.mvn_logpdf_ref(L, x.T, np.zeros(d), s0)
    ar.within("mvn logpdf scalar", host(dists.MvNormal(loc=np.zeros(d), scale=s0, cov=cov).logpdf(dev(x))), v, b)
    z = r.standard_normal((n, d))
    v, b = ar.mvn_rvs_ref(L, z.T, loc.T, sc.T)
    got = host(dists.MvNormal(loc=dev(loc), scale=dev(sc), cov=cov).rvs(size=n, z=z))
    ar.within("mvn rvs injected", got.T.reshape(-1), v.reshape(-1), b.reshape(-1))
    got = host(dists.MvNormal(loc=dev(loc), scale=dev(sc), cov=cov).rvs(size=n))       # API call 0
    zs, bz = (ar.mvn_big_normals if d > 8 else ar.mvn_small_normals)(n, d, 0, SEED)
    v, b = ar.mvn_rvs_ref(L, zs, loc.T, sc.T, dz=bz)
    ar.within("mvn rvs own draws", got.T.reshape(-1), v.reshape(-1), b.reshape(-1))


# ------------------------------------------------------------------------------------------ end to end
def _logistic_data(d, n_data, seed):
    r = np.random.RandomState(seed)
    X = r.randn(n_data, d)
    y = np.sign(X @ (r.randn(d) * 0.5) + r.randn(n_data))
    return X * y[:, None]


@pytest.mark.parametrize("sampler", ["tempering", "nested"])
def test_moments_collector_at_d20(pb, sampler):
    """collect=[Moments()] on a d = 20 sampler: wmean_and_var on (N, 20) particles every generation, the last one
    checked against the replay."""
    from particles_b200 import collectors as col
    from particles_b200 import nested
    from particles_b200 import smc_samplers as ssp
    data = _logistic_data(20, 60, 1)
    model = ssp.LogisticRegression(data=data)
    fk = (ssp.AdaptiveTempering(model=model, len_chain=5, ESSrmin=0.5) if sampler == "tempering"
          else nested.NestedSamplingSMC(model=model, len_chain=5, ESSrmin=0.5))
    pf = pb.SMC(fk=fk, N=1000, seed=3, collect=[col.Moments()])
    pf.run()
    mom = pf.summaries.moments
    assert len(mom) == pf.t and np.shape(mom[-1]["mean"]) == (20,)
    W = host(pf.W) if isinstance(pf.W, torch.Tensor) else np.asarray(pf.W)
    theta = pf.X.theta
    theta = host(theta) if isinstance(theta, torch.Tensor) else np.asarray(theta)
    ar.check_wmoments(W, theta, np.concatenate([mom[-1]["mean"], mom[-1]["var"]]))
