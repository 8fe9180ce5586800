"""The stand-alone kernels' replay (tests/api_replay.py) on the CPU: it predicts the oracle's weights, moments and
ancestors of every scheme on the golden cases and on seeded large inputs, its distribution bounds contain scipy's
values, its Philox layouts reproduce hand-built counters, and it rejects planted faults."""
import numpy as np
import pytest
from scipy import stats
from scipy.special import gammaln

import api_replay as ar
import philox_ref
from oracle import smc_numpy as orc

LW_CASES = ["gauss_1000", "equal_257", "dominant_513", "neginf_777", "nan_300", "single_1", "wide_4099", "tiny_2"]
RS_CASES = ["dirichlet_1000", "skewed_513", "M_lt_N", "M_gt_N", "zeros_300", "dominant_64", "equal_1025", "n7"]


def _seeded_lw(n, seed, spread=3.0):
    r = np.random.RandomState(seed)
    lw = r.randn(n) * spread
    lw[r.rand(n) < 0.1] = -np.inf
    return lw


# ------------------------------------------------------------------------------------------------- weights
@pytest.mark.parametrize("name", LW_CASES)
def test_weights_replay_predicts_golden(golden, name):
    lw_in = golden[f"w/{name}/lw_in"]
    s = golden[f"w/{name}/stats"]
    fin = ar.fix_nan(lw_in)
    m = fin.max()
    ssum = np.exp(fin - m).sum()
    ar.check_weights(lw_in, fin, [s[0], s[1], s[2], ssum], golden[f"w/{name}/W"])
    lse = golden[f"w/{name}/lse"]
    for mode, want in zip(("sum", "mean", "essl"), lse):
        val, b = ar.lse_ref(fin, mode)
        ar.within(mode, want, np.atleast_1d(val), b)
    val, b = ar.lse_ref(fin, "wmean", W=golden[f"w/{name}/Wn"])
    ar.within("weighted log_mean_exp", golden[f"w/{name}/log_mean_exp_W"][0], np.atleast_1d(val), b)
    W, bW = ar.exp_normalise_ref(fin)
    ar.within("exp_and_normalise", golden[f"w/{name}/exp_and_normalise"], W, bW)


@pytest.mark.parametrize("n,spread", [(1, 1.0), (257, 3.0), (100_003, 4.0), (20_000, 300.0)])
def test_weights_replay_predicts_oracle(n, spread):
    lw = _seeded_lw(n, n, spread)
    lw[0] = 0.0
    ref = orc.Weights(lw=lw.copy())
    ar.check_weights(lw, ref.lw, [ref.lw.max(), ref.log_mean, ref.ESS, np.exp(ref.lw - ref.lw.max()).sum()], ref.W)
    for mode, f in (("sum", orc.log_sum_exp), ("mean", orc.log_mean_exp), ("essl", orc.essl)):
        val, b = ar.lse_ref(ref.lw, mode)
        ar.within(mode, f(ref.lw), np.atleast_1d(val), b)
    Wn = np.random.RandomState(1).rand(n)
    val, b = ar.lse_ref(ref.lw, "wmean", W=Wn)
    ar.within("weighted", orc.log_mean_exp(ref.lw, W=Wn), np.atleast_1d(val), b)


def test_lse_edge_rules_are_the_references():
    """Any NaN, any +inf or all -inf: NaN from every reduction, as the reference's m + log(sum(exp(v - m))) gives."""
    cases = [np.full(5, -np.inf), np.array([0.0, np.inf, 1.0]), np.array([np.nan, 0.0]), np.array([-np.inf, np.nan])]
    with np.errstate(invalid="ignore"):
        for v in cases:
            for mode, f in (("sum", orc.log_sum_exp), ("mean", orc.log_mean_exp), ("essl", orc.essl)):
                val, _ = ar.lse_ref(v, mode)
                assert np.isnan(val) and np.isnan(f(v)), (v, mode)
            val, _ = ar.lse_ref(v, "wmean", W=np.full(v.size, 0.5))
            assert np.isnan(val) and np.isnan(orc.log_mean_exp(v, W=np.full(v.size, 0.5)))
            W, _ = ar.exp_normalise_ref(v)
            assert np.isnan(W.astype(float)).all() and np.isnan(orc.exp_and_normalise(v)).all()


def test_weights_subnormal_W():
    """A spread of 1400: W below 1e-308 is within the bound whether the kernel keeps it or flushes it to 0."""
    lw = np.linspace(0.0, -1400.0, 4001)
    r = ar.weights_ref(lw)
    W = orc.exp_and_normalise(lw)
    assert (W[(W > 0) & (W < 2.3e-308)]).size > 0
    ar.within("W", W, r["W"], r["b_W"])
    flushed = np.where(lw < -708, 0.0, W)
    ar.within("W flushed", flushed, r["W"], r["b_W"])


# ------------------------------------------------------------------------------------------------- moments
@pytest.mark.parametrize("d", [1, 2, 5, 17, 32])
@pytest.mark.parametrize("offset", [0.0, 1e6])
def test_wmoments_replay_predicts_oracle(d, offset):
    r = np.random.RandomState(d)
    n = 30_011
    W = r.rand(n) ** 4
    W[r.rand(n) < 0.2] = 0.0
    W /= W.sum()
    x = offset + r.randn(n, d)
    ref = orc.wmean_and_var(W, x)
    ar.check_wmoments(W, x, np.concatenate([ref["mean"], ref["var"]]))


def test_wmoments_rejects_a_slot_off_by_one_component():
    r = np.random.RandomState(0)
    n, d = 5000, 9
    W = r.rand(n)
    W /= W.sum()
    x = r.randn(n, d) * np.arange(1, d + 1) + np.arange(d)
    ref = orc.wmean_and_var(W, x)
    good = np.concatenate([ref["mean"], ref["var"]])
    ar.check_wmoments(W, x, good)
    bad = good.copy()
    bad[5:d] = bad[4:d - 1]                # components from 4 on written one slot late
    with pytest.raises(AssertionError):
        ar.check_wmoments(W, x, bad)


# ---------------------------------------------------------------------------------------------- resampling
@pytest.mark.parametrize("name", RS_CASES)
@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_search_replay_predicts_golden(golden, name, scheme):
    W, M = golden[f"rs/{name}/W"], int(golden[f"rs/{name}/M"][0])
    u = golden[f"rs/{name}/{scheme}/u"]
    A = golden[f"rs/{name}/{scheme}/A"]
    z = np.cumsum(-np.log(u[:M + 1])) if scheme == "multinomial" else None
    ar.check_inverse_cdf(scheme, W, M, u, A, z=z)


@pytest.mark.parametrize("name", RS_CASES)
def test_residual_killing_ssp_replay_predict_golden(golden, golden_rs_extra, name):
    W, M = golden[f"rs/{name}/W"], int(golden[f"rs/{name}/M"][0])
    u = golden[f"rs/{name}/residual/u"]
    ar.check_residual(W, M, u, golden[f"rs/{name}/residual/A"])
    x = golden_rs_extra
    assert np.array_equal(orc.ssp(W, M, u=x[f"rs/{name}/ssp/u"]), x[f"rs/{name}/ssp/A"])
    if M == W.size:
        ar.check_killing(W, x[f"rs/{name}/killing/u"], x[f"rs/{name}/killing/u_multinomial"],
                         x[f"rs/{name}/killing/A"])


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial", "residual", "killing"])
def test_resampling_replay_predicts_oracle_large(scheme):
    n = 50_000
    r = np.random.RandomState(7)
    W = orc.exp_and_normalise(_seeded_lw(n, 3))
    u = r.rand(n + 1)
    if scheme == "residual":
        ar.check_residual(W, n, u, orc.residual(W, n, u=u))
    elif scheme == "killing":
        nk = int((u[:n] * W.max() >= W).sum())
        um = r.rand(nk + 1)
        nk, decided = ar.check_killing(W, u[:n], um, orc.killing(W, n, u=u[:n], u_multinomial=um))
        assert nk > 0 and decided >= nk - 5
    else:
        u = u[:orc.n_uniforms(scheme, n)]
        A = orc.resampling(scheme, W, n, u=u)
        decided = ar.check_inverse_cdf(scheme, W, n, u, A)
        assert decided >= n - 5
    with pytest.raises(AssertionError):
        ar.check_inverse_cdf("systematic", W, n, u, orc.systematic(W, n, u=u[:1]) + 1)


def test_residual_integral_and_single_draw():
    """M W integral: sres = 0, no stochastic part; sres = 1: one draw on res itself."""
    W = np.array([1, 3, 0, 4], dtype=np.float64) / 8
    ip, sip, sres, _ = ar.residual_parts(W, 8)
    assert sres == 0 and np.array_equal(ip, [1, 3, 0, 4])
    ar.check_residual(W, 8, np.full(9, 0.5), orc.residual(W, 8, u=np.full(9, 0.5)))
    W = np.array([1.5, 2.5, 4.0]) / 8
    _, sip, sres, res = ar.residual_parts(W, 8)
    assert sres == 1 and sip == 7
    u = np.array([0.3, 0.6])
    ar.check_residual(W, 8, u, orc.residual(W, 8, u=u))


def test_search_rejects_a_one_ulp_cdf_entry():
    """A grid point on a knot: the kernel's CDF with that knot one ulp low would draw the next entry."""
    W = np.full(8, 0.125)
    cdf = np.cumsum(W)
    su = (0.5 + np.arange(8)) / 8
    su[3] = cdf[3]
    A = np.minimum(np.searchsorted(cdf, su, side="left"), 7)
    ar.check_search_exact("good", A, cdf, su)
    low = cdf.copy()
    low[3] = np.nextafter(low[3], 0)
    with pytest.raises(AssertionError):
        ar.check_search_exact("one ulp", A, low, su)
    with pytest.raises(AssertionError):
        ar.check_cdf("one ulp", np.concatenate([low[:3], [np.nextafter(low[3], 0) - 2 ** -40], low[4:]]), W)


def test_search_rejects_an_ancestor_moved_where_the_bound_decides():
    r = np.random.RandomState(2)
    W = r.rand(5000)
    W /= W.sum()
    u = r.rand(1)
    A = orc.systematic(W, 5000, u=u)
    C, bC = ar.cdf_ref(W)
    su = ar.su_of("systematic", u, 5000)
    lo, hi = ar.bracket(C, bC, su, np.zeros(5000, dtype=ar.LD))
    k = int(np.flatnonzero((lo == hi) & (A < 4999))[100])
    bad = A.copy()
    bad[k] += 1
    with pytest.raises(AssertionError):
        ar.check_ancestors("moved", bad, C, bC, su, 0, W)


def test_search_branches_helper():
    """Spread weights stage every tile; M << N, or 90 % zeros, leaves the tiles' slices longer than the stage."""
    n = 1_000_000
    cdf = np.cumsum(np.full(n, 1.0 / n))
    assert ar.search_branches(cdf, (0.5 + np.arange(n)) / n).all()
    assert not ar.search_branches(cdf, (0.5 + np.arange(4096)) / 4096).any()
    W = np.zeros(n)
    W[::10] = 1.0
    W /= W.sum()
    br = ar.search_branches(np.cumsum(W), (0.5 + np.arange(n // 100)) / (n // 100))
    assert not br.any()


def test_killing_rejects_a_moved_survivor():
    r = np.random.RandomState(4)
    W = orc.exp_and_normalise(r.randn(1000))
    u = r.rand(1000)
    um = r.rand(int((u * W.max() >= W).sum()) + 1)
    A = orc.killing(W, 1000, u=u, u_multinomial=um)
    ar.check_killing(W, u, um, A)
    keep = np.flatnonzero(u * W.max() < W)
    bad = A.copy()
    bad[keep[0]] = (keep[0] + 1) % 1000
    with pytest.raises(AssertionError):
        ar.check_killing(W, u, um, bad)


# ------------------------------------------------------------------------------------------- distributions
X_EDGE = np.array([-1e300, -800.0, -709.8, -709.7, -40.0, -1.0, -1e-300, 0.0, 1e-300, 0.5, 40.0, 800.0, 1e300])


def test_normal_student_laplace_bounds_contain_scipy():
    r = np.random.RandomState(0)
    x = np.concatenate([r.randn(2000) * 5, X_EDGE[(np.abs(X_EDGE) < 1e100)], [1e154, -1e154, 1.35e154, np.inf,
                                                                               -np.inf, np.nan]])
    loc, sc = 0.3, 1.7
    v, b = ar.normal_logpdf_ref(x, loc, sc)
    ar.within("normal", stats.norm.logpdf(x, loc=loc, scale=sc), v, b)
    for df in (1.0, 3.0, 4.5, 30.0):
        c0 = gammaln(0.5 * (df + 1.0)) - gammaln(0.5 * df) - 0.5 * np.log(df * np.pi)
        with np.errstate(over="ignore"):
            want = stats.t.logpdf(x, df, loc=loc, scale=sc)
        v, b = ar.student_logpdf_ref(x, df, c0, loc, sc)
        ar.within(f"student {df}", want, v, b)
    v, b = ar.laplace_logpdf_ref(x, loc, sc)
    small = np.abs((x - loc) / sc) < 700
    ar.within("laplace", stats.laplace.logpdf(x[small], loc=loc, scale=sc), v[small], b[small])
    assert np.isfinite(v[np.isfinite(x) & ~small].astype(float)).all()


def test_gamma_bounds_contain_scipy_with_xlogy_edges():
    x = np.array([0.0, -0.0, 5e-324, 1e-300, 0.3, 2.0, 700.0, np.inf, -1.0, -np.inf, np.nan])
    for a in (0.5, 1.0, 2.5):
        for b in (1.0, 3.0):
            with np.errstate(all="ignore"):
                want = stats.gamma.logpdf(x, a, scale=1.0 / b)
            v, bd = ar.gamma_logpdf_ref(x, a, -gammaln(a), b)
            ar.within(f"gamma a={a} b={b}", want, v, bd)
    v, _ = ar.gamma_logpdf_ref(np.array([0.0]), 1.0, 0.0, 3.0)
    assert v[0] == np.log(ar.LD(3))


def test_logistic_bounds_contain_scipy_and_reject_the_overflowing_form():
    x = np.concatenate([X_EDGE, np.random.RandomState(1).randn(1000) * 30])
    v, b = ar.logistic_logpdf_ref(x, 0.0, 1.0)
    ar.within("logistic", stats.logistic.logpdf(x), v, b)
    sc = np.exp(np.random.RandomState(2).randn(x.size))
    v2, b2 = ar.logistic_logpdf_ref(x, 0.25, sc)
    ar.within("logistic per-particle", stats.logistic.logpdf(x, loc=0.25, scale=sc), v2, b2)
    with pytest.raises(AssertionError):
        ar.within("overflowing", ar.logistic_logpdf_overflowing(x, 0.0, 1.0), v, b)


def _cov(d, cond, seed):
    r = np.random.RandomState(seed)
    Q, _ = np.linalg.qr(r.randn(d, d))
    ev = np.logspace(0, -np.log10(cond), d)
    return (Q * ev) @ Q.T + 1e-300 * np.eye(d)


@pytest.mark.parametrize("d", [1, 2, 8, 9, 20, 32])
@pytest.mark.parametrize("cond", [1e1, 1e8])
def test_mvn_bounds_contain_the_oracle(d, cond):
    cov = _cov(d, cond, d)
    r = np.random.RandomState(d + 1)
    n = 500
    loc, sc = r.randn(n, d), np.exp(r.randn(n, d) * 0.3)
    x = loc + r.randn(n, d)
    L = np.linalg.cholesky(cov)
    ref = orc.MvNormal(loc=loc, scale=sc, cov=cov)
    v, b = ar.mvn_logpdf_ref(L, x.T, loc.T, sc.T)
    ar.within("mvn logpdf", ref.logpdf(x), v, b)
    z = r.standard_normal((n, d))
    v, b = ar.mvn_rvs_ref(L, z.T, loc.T, sc.T)
    ar.within("mvn rvs", ref.rvs(size=n, z=z).T.reshape(-1), v.reshape(-1), b.reshape(-1))


# --------------------------------------------------------------------------------------------------- draws
SEED = 0x1234567890ABCDEF


def _bm64(r):
    u1, u2 = philox_ref.u53_open(r[0], r[1]), philox_ref.u53(r[2], r[3])
    rad = np.sqrt(-2.0 * np.log(u1))
    return rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)


@pytest.mark.parametrize("call", [0, 5, (3 << 32) + 7])
def test_philox_layouts_reproduce_hand_built_counters(call):
    k0, k1 = SEED & 0xFFFFFFFF, SEED >> 32
    lo, hi = call & 0xFFFFFFFF, call >> 32
    u = ar.api_uniforms(7, call, SEED)
    r = philox_ref.philox4x32_10(3, 0, lo, (hi << 8) | 3, k0, k1)
    assert u[6] == philox_ref.u53(r[0], r[1])
    z, b = ar.api_normals(7, call, SEED)
    assert abs(z[5] - _bm64(r if False else philox_ref.philox4x32_10(2, 0, lo, (hi << 8) | 3, k0, k1))[1]) <= 1e-13
    # k_mvn_rvs: component k in bits 8.. of word 3, call's high word from bit 16
    zs, _ = ar.mvn_small_normals(6, 3, call, SEED)
    r = philox_ref.philox4x32_10(2, 0, lo, (hi << 16) | (2 << 8) | 3, k0, k1)
    assert abs(zs[2, 5] - _bm64(r)[1]) <= 1e-13 and abs(zs[2, 4] - _bm64(r)[0]) <= 1e-13
    # k_mvn_big: one counter per particle, component pair j in word 3
    zb, _ = ar.mvn_big_normals(6, 11, call, SEED)
    r = philox_ref.philox4x32_10(4, 0, lo, (hi << 16) | (5 << 8) | 3, k0, k1)
    assert abs(zb[10, 4] - _bm64(r)[0]) <= 1e-13
    r = philox_ref.philox4x32_10(4, 0, lo, (hi << 16) | (3 << 8) | 3, k0, k1)
    assert abs(zb[6, 4] - _bm64(r)[0]) <= 1e-13 and abs(zb[7, 4] - _bm64(r)[1]) <= 1e-13


def test_mvn_layout_rejects_a_component_counter_swap():
    d, n, call = 5, 64, 9
    cov = _cov(d, 10.0, 3)
    L = np.linalg.cholesky(cov)
    zs, bz = ar.mvn_small_normals(n, d, call, SEED)
    v, b = ar.mvn_rvs_ref(L, zs, dz=bz)
    ar.within("mvn draws", (L @ zs.astype(np.float64)).reshape(-1), v.reshape(-1), b.reshape(-1))
    swapped = zs[[1, 0, 2, 3, 4]].astype(np.float64)
    with pytest.raises(AssertionError):
        ar.within("swapped", (L @ swapped).reshape(-1), v.reshape(-1), b.reshape(-1))
    big, _ = ar.mvn_big_normals(n, d, call, SEED)          # the other kernel's layout is another draw
    with pytest.raises(AssertionError):
        ar.within("layout", (L @ big.astype(np.float64)).reshape(-1), v.reshape(-1), b.reshape(-1))


def test_normal_bound_holds_for_numpy_box_muller():
    z, b = ar.api_normals(100_001, 3, SEED)
    ar.within("normals", philox_ref.normals(100_001, 3, SEED, w3=ar.API), z, b)


def test_lse_rejects_a_skipped_element():
    """A reduction that drops one value (a loop starting one stride late) is outside the bound."""
    lw = np.random.RandomState(5).randn(300_000)
    val, b = ar.lse_ref(lw, "sum")
    with pytest.raises(AssertionError):
        ar.within("skip", orc.log_sum_exp(np.delete(lw, 1234)), np.atleast_1d(val), b)
