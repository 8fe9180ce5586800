"""The binary-space replay (tests/binary_replay.py) checked without a GPU: a second fp64 implementation (the NumPy
oracle on scipy's LAPACK Cholesky) and the live reference's golden vectors lie inside its bounds on every design the
GPU tests use, ill-conditioned and badly scaled ones included; the bounds are tight where the design is well
conditioned; the nested-logistic and move replays predict the oracle's own draws and decisions; and the Philox layouts
and the warp tiers are what csrc/smcb_binary.cu uses."""
import os

import numpy as np
import pytest

import binary_oracle as bo
import binary_replay as br
import philox_ref

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "golden_binary.npz"))


def gammas(p, n, seed):
    """|gamma| = 0, 1, p - 1, p, the last coordinate only, coordinates >= 96 only, then random densities."""
    r = np.random.RandomState(seed)
    g = r.rand(n, p) < r.uniform(0.05, 0.95, (n, 1))
    g[0] = False
    g[1] = False
    g[1, r.randint(p)] = True
    g[2] = True
    g[2, r.randint(p)] = False
    g[3] = True
    g[4] = False
    g[4, p - 1] = True
    if p > 96:
        g[5] = False
        g[5, 96:] = True
    return g


def test_bin_warps_tiers():
    """8, 7, 6, 5, 4, 3 warps per CTA with the boundaries at k = 78, 84, 91, 100, 112; 198 KB at p = 128."""
    ks = np.arange(0, br.MAX_P + 1)
    w = np.array([br.bin_warps(int(k)) for k in ks])
    assert set(w) == {3, 4, 5, 6, 7, 8}
    assert list(ks[1:][np.diff(w) != 0]) == [78, 84, 91, 100, 112]
    assert br.bin_smem(128, br.bin_warps(128)) == 202776 and br.bin_smem(128, 3) // 1024 == 198
    assert all(br.bin_smem(int(k), br.bin_warps(int(k))) <= br.SMEM_BUDGET for k in ks)
    assert br.cta_warp(13, 3) == (4, 1) and br.words(32) == 1 and br.words(33) == 2 and br.words(128) == 4


@pytest.mark.parametrize("p", [1, 2, 33, 97, 128])
@pytest.mark.parametrize("dkind", ["gauss", "ar1", "scaled"])
@pytest.mark.parametrize("kind", ["bic", "bvs", "gprior"])
def test_oracle_inside_bounds(kind, dkind, p):
    """scipy's Cholesky (binary_oracle.chol_and_friends) and the oracle's llik lie inside the replay's bounds."""
    X, y = br.design(dkind, p, seed=p)
    desc = br.model_desc(kind, X, y)
    o = bo.VS(kind, X, y)
    g = gammas(p, 24, p + 1)
    want = br.vs_ld(desc, g)
    assert want["ok"].all()
    len_gam, ldet, wtw = o.chol(g)
    np.testing.assert_array_equal(len_gam, want["len_gam"])
    br.assert_close("ldet", ldet, want["ldet"], want["b_ldet"])
    br.assert_close("wtw", wtw, want["wtw"], want["b_wtw"])
    ll = o.loglik(g)
    fin = ~want["near0"]
    br.assert_close("llik", ll[fin], want["llik"][fin], want["b_llik"][fin])
    lp = bo.IIDBernoulli(0.5, p).logpdf(g)
    np.testing.assert_array_equal(want["lprior"], lp)       # the same terms added in the same order


@pytest.mark.parametrize("p", [33, 128])
@pytest.mark.parametrize("kind", ["bic", "bvs", "gprior"])
def test_bounds_are_tight(kind, p):
    """On a well-conditioned design the relative bounds are below 1e-10, and the oracle moved by 10x the bound falls
    outside them."""
    X, y = br.design("gauss", p, seed=3)
    desc = br.model_desc(kind, X, y)
    o = bo.VS(kind, X, y)
    g = gammas(p, 16, 4)
    want = br.vs_ld(desc, g)
    nz = want["len_gam"] > 0
    _, ldet, wtw = o.chol(g)
    ll = o.loglik(g)
    for name, got in (("ldet", ldet), ("wtw", wtw), ("llik", ll)):
        w = want[name].astype(np.float64)[nz]
        b = want["b_" + name][nz]
        assert np.all(b <= 1e-10 * np.abs(w)), (name, np.max(b / np.abs(w)))
        moved = got[nz] + 10 * b * np.where(got[nz] >= w, 1, -1)
        with pytest.raises(AssertionError):
            br.assert_close(name, moved[:1], want[name][nz][:1], b[:1])


@pytest.mark.parametrize("tag", ["p10", "p104"])
@pytest.mark.parametrize("kind", ["bic", "bvs", "gprior"])
def test_golden_inside_bounds(tag, kind):
    """The live reference's golden ldet / wtw / loglik lie inside the bounds."""
    X, y = (bo.small_design if tag == "p10" else bo.boston_like)()
    desc = br.model_desc(kind, X, y)
    g = G[tag + "/gamma"]
    want = br.vs_ld(desc, g)
    np.testing.assert_array_equal(want["len_gam"], G["%s/%s/len_gam" % (tag, kind)])
    br.assert_close("ldet", G["%s/%s/ldet" % (tag, kind)], want["ldet"], want["b_ldet"])
    br.assert_close("wtw", G["%s/%s/wtw" % (tag, kind)], want["wtw"], want["b_wtw"])
    br.assert_close("llik", G["%s/%s/loglik" % (tag, kind)], want["llik"], want["b_llik"])


def edgy_proposal(p, seed, kind="random"):
    """Nested-logistic coefficients: ``random``, ``saturated`` (|logit| 35-40, where 1 - pr is below 2^-53) or
    ``overflow`` (+-800), with every third coordinate edgy at probabilities 0, 1, 1e-300 and 0.5 in turn."""
    r = np.random.RandomState(seed)
    c = np.tril(r.standard_normal((p, p)) * 0.3, -1)
    d = r.standard_normal(p)
    if kind == "saturated":
        d = r.choice([-1.0, 1.0], p) * r.uniform(35, 40, p)
        c *= 0.0
    elif kind == "overflow":
        d = r.choice([-800.0, 800.0], p)
    c[np.diag_indices(p)] = d
    edgy = np.zeros(p, dtype=bool)
    edgy[::3] = True
    vals = np.array([0.0, 1.0, 1e-300, 0.5])
    for j, i in enumerate(np.flatnonzero(edgy)):
        c[i, :] = 0.0
        c[i, i] = vals[j % 4]
    return c, edgy


@pytest.mark.parametrize("kind", ["random", "saturated", "overflow"])
@pytest.mark.parametrize("p", [1, 33, 128])
def test_nested_logistic_replay_predicts_oracle(kind, p):
    """Every decided bit of the oracle's draw is predicted, the oracle's logpdf (rvs and arbitrary rows) lies inside
    the bound, and u == pr on an edgy coordinate gives 0 (the strict <)."""
    c, edgy = edgy_proposal(p, p, kind)
    nl = bo.NestedLogistic(c, edgy)
    r = np.random.RandomState(5)
    n = 300
    u = r.rand(p, n)
    u[:, 0], u[:, 1] = 0.0, 1.0 - 2.0 ** -53
    for i in np.flatnonzero(edgy):
        u[i, 2] = c[i, i]                                   # u == pr exactly
    x, _ = nl.rvs(n, u)
    _, dec, mism = br.nl_replay_draw(c, edgy, u, follow=x)
    assert not mism.any() and dec.mean() > 0.99
    assert not x[2, np.flatnonzero(edgy)].any()
    _, lo, hi = br.nl_ld(c, edgy, x)
    want, b = br.nl_logpdf(x, lo, hi)
    br.assert_close("logpdf of the draw", nl.logpdf(x), want, b)
    xa = r.rand(n, p) < 0.5                                 # arbitrary rows, bits of probability 0 included
    _, lo, hi = br.nl_ld(c, edgy, xa)
    want, b = br.nl_logpdf(xa, lo, hi)
    br.assert_close("logpdf of arbitrary rows", nl.logpdf(xa), want, b)
    if kind in ("saturated", "overflow") and p > 1:
        # saturated logits where the fp64 pr is exactly 1 (a 0 bit there costs log(1e-300), exactly) and exactly 0
        assert np.any((lo == 1.0) & ~edgy) and np.any((hi == 0.0) & ~edgy) if kind == "overflow" else \
            np.any((lo == 1.0) & ~edgy)


@pytest.mark.parametrize("p,kind,epn", [(10, "bvs", 0.4), (10, "bic", 1.0), (33, "gprior", 0.0), (65, "bvs", 0.4)])
def test_move_replay_predicts_oracle(p, kind, epn):
    """check_generation, fed the oracle's own waste-free move (binary_oracle.wf_move with injected draws), sees every
    decision and row, decides at least 99 % of the chain-steps, and rejects a flipped decision and a one-ulp change
    in a rejected chain's llik."""
    M, P = 120, 5
    if p == 10:
        X, y = bo.small_design()
        c, edgy = G["p10/fit/coeffs"], G["p10/fit/edgy"]
    else:
        X, y = br.design("gauss", p, seed=p)
        c, edgy = edgy_proposal(p, p + 1)
    desc = br.model_desc(kind, X, y)
    o = bo.VS(kind, X, y, prior=bo.IIDBernoulli(0.5, p))
    prop = bo.NestedLogistic(c, edgy)
    np.random.seed(p)
    x0 = bo.ThetaParticles(theta=prop.rvs(M)[0])
    bo.target(o, epn)(x0)
    xo, pbo, (up, ua) = bo.wf_move(x0, bo.target(o, epn), prop, P)
    rows = [{k: getattr(xo, k)[s * M:(s + 1) * M] for k in ("theta", "lprior", "llik", "lpost")} for s in range(P)]
    n_acc = n_und = 0
    for s in range(1, P):
        res = br.check_generation(s, desc, c, edgy, epn, rows[s - 1], rows[s], pbo[s - 1], up[s - 1], ua[s - 1], 8)
        n_acc += int(res["accepted"].sum())
        n_und += res["undecided"]
    assert 0 < n_acc < (P - 1) * M and n_und <= 0.01 * (P - 1) * M
    s = 1
    acc = br.check_generation(s, desc, c, edgy, epn, rows[0], rows[1], pbo[0], up[0], ua[0], 8)["accepted"]
    j = int(np.flatnonzero(~acc)[0])
    bent = dict(rows[1], llik=rows[1]["llik"].copy())
    bent["llik"][j] = np.nextafter(bent["llik"][j], np.inf)
    with pytest.raises(AssertionError):
        br.check_generation(s, desc, c, edgy, epn, rows[0], bent, pbo[0], up[0], ua[0], 8)
    j = int(np.flatnonzero(acc)[0])
    bent = dict(rows[1], theta=rows[1]["theta"].copy(), lprior=rows[1]["lprior"].copy(),
                llik=rows[1]["llik"].copy(), lpost=rows[1]["lpost"].copy())
    for k in ("theta", "lprior", "llik", "lpost"):
        bent[k][j] = rows[0][k][j]                          # the accepted chain rejected
    ub = ua[0].copy()
    with pytest.raises(AssertionError):
        br.check_generation(s, desc, c, edgy, epn, rows[0], bent, pbo[0], up[0], ub, 8)


def test_philox_layouts():
    """The three counter layouts draw different uniforms wherever their counter words differ: coordinate 0 vs 32 vs
    64 vs 96, step 1 vs 257 (the step field is 16 bits wide), call 0 vs 1, proposal vs acceptance vs rvs."""
    seed = 0xABCDEF12345
    M = 64
    pr = br.prop_uniforms(M, 128, 1, 0, seed)
    assert len({pr[i, 0] for i in (0, 32, 64, 96)}) == 4
    assert not np.array_equal(pr[0], br.prop_uniforms(M, 1, 257, 0, seed)[0])
    assert not np.array_equal(br.acc_uniforms(M, 1, 0, seed), br.acc_uniforms(M, 257, 0, seed))
    assert not np.array_equal(br.acc_uniforms(M, 1, 0, seed), br.acc_uniforms(M, 1, 1, seed))
    rv = br.rvs_uniforms(M, 128, 0, seed)
    assert len({rv[i, 3] for i in (0, 32, 64, 96, 127)}) == 5
    assert not np.array_equal(rv[0], br.rvs_uniforms(M, 1, 1, seed)[0])
    assert not np.array_equal(rv[0], pr[0])
    # the layouts are philox_ref's counter words: chain in words 0-1, call in word 2, the field in word 3
    r = philox_ref._ctr(np.arange(M, dtype=np.uint64), 0, (1 << 16) | (5 << 8) | br.PURPOSE_PROP, seed)
    np.testing.assert_array_equal(pr[5], philox_ref.u53(r[0], r[1]))
    assert np.all((pr >= 0) & (pr < 1))
