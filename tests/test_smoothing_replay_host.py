"""The smoothing replay (tests/smoothing_replay.py) on the CPU: its transition densities and bounds against the host
build of the device density (tests/trans_host.cpp) and the NumPy oracle, its draw checks against the reference's
own indices, counts and estimates (golden_smoothing.npz, golden_twofilter.npz), its Philox layouts against
hand-built counters, and the rule for a row with no positive weight as the reference gives it."""
import ctypes as C
import os

import numpy as np
import pytest

import smoothing_replay as sr
from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm
from philox_ref import philox4x32_10, u53_open
from test_smoothing_host import build_trans_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = C.c_void_p
SEEDS = {"lg": 11, "sv": 12, "cox": 13, "mvlg2": 14}


def _cases():
    from particles_b200 import kalman, state_space_models as ssm
    return [("StochVol", ssm.StochVol()), ("StochVolLeverage", ssm.StochVolLeverage(phi=-0.6)),
            ("LinearGauss", kalman.LinearGauss(rho=0.9)), ("DiscreteCox", ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9)),
            ("ThetaLogistic", ssm.ThetaLogistic()), ("Gordon_etal", ssm.Gordon_etal()),
            ("MVLinearGauss2", kalman.MVLinearGauss_Guarniero_etal(0.4, 2)),
            ("MVLinearGauss3", kalman.MVLinearGauss_Guarniero_etal(0.4, 3)),
            ("MVLinearGauss4", kalman.MVLinearGauss_Guarniero_etal(0.4, 4)), ("BearingsOnly", ssm.BearingsOnly())]


def spec_of(model, T=12):
    from particles_b200 import state_space_models as ssm
    dy = getattr(model, "dy", 1)
    return ssm.transition_spec(ssm.Bootstrap(ssm=model, data=[np.ones(dy)] * T))


def host_trans(spec, t, xp, x):
    lib = build_trans_host()
    n, dim = xp.shape[0], spec["dim"]
    params = np.ascontiguousarray(spec["params"], dtype=np.float64)
    sc = spec["step_consts"]
    sc = None if sc is None else np.ascontiguousarray(sc, dtype=np.float64)
    soa = lambda a: np.ascontiguousarray(a.reshape(n, -1).T)      # noqa: E731
    xp_s, x_s, out = soa(xp), soa(x), np.empty(n)
    rc = lib.mh_trans_logpdf(spec["model"], dim, params.ctypes.data_as(P), None if sc is None else sc.ctypes.data_as(P),
                             C.c_long(t), xp_s.ctypes.data_as(P), x_s.ctypes.data_as(P), C.c_long(n),
                             out.ctypes.data_as(P))
    assert rc == 0
    return out


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_trans_bounds_hold_and_are_tight(case):
    """The host build of the device density (the kernel's arithmetic without fma contraction) lies within the
    replay's bound of the long-double value at every pair; the bound is below 1e-12 of max(1, |value|) on these
    well-conditioned models, and above the rounding level (it is not vacuous)."""
    name, model = case
    spec = spec_of(model)
    tr = sr.Trans(spec)
    r = np.random.RandomState(7)
    n, D = 2000, spec["dim"]
    xp = r.standard_normal((n, D)) * (3.0 if name == "Gordon_etal" else 1.0)
    if name == "BearingsOnly":
        xp = xp * 0.01 + np.array([0.0, 0.0, 1.0, 1.0])
        x = np.column_stack([xp[:, :2] + 0.3 * r.standard_normal((n, 2)), xp[:, 0] + xp[:, 2], xp[:, 1] + xp[:, 3]])
        x[::3, 2] = np.nextafter(x[::3, 2], 9.0)                 # one Dirac in three broken by one ulp
    else:
        x = 0.9 * xp + r.standard_normal(xp.shape)
    for t in (1, 5, 11):
        v, b = tr.lpdf(t, xp, x)
        got = host_trans(spec, t, xp, x)
        fin = np.isfinite(np.float64(v))
        assert np.array_equal(fin, np.isfinite(got)), name
        if name == "BearingsOnly":
            assert fin.any() and (~fin).any()
        err = np.abs(np.float64(sr.LD(1) * got[fin] - v[fin]))
        assert np.all(err <= b[fin]), (name, t, float((err / b[fin]).max()))
        scale = np.maximum(1.0, np.abs(np.float64(v[fin])))
        assert np.max(b[fin] / scale) < 1e-12, (name, float(np.max(b[fin] / scale)))
        assert np.max(b[fin] / scale) > 1e-17


def test_philox_layouts_are_the_documented_counters():
    seed, call = 0x0123456789ABCDEF, 7
    u0, u1 = sr.smooth_uniforms(seed, call, np.array([0, 5, 70000]), 3, np.array([0, 2, 41]), sr.PURPOSE_SMOOTH)
    for k, (m, trial) in enumerate(((0, 0), (5, 2), (70000, 41))):
        r = philox4x32_10(np.uint32(m), np.uint32(3), np.uint32(call), np.uint32((trial << 8) | 4),
                          0x89ABCDEF, 0x01234567)
        assert u0[k] == u53_open(r[0], r[1]) and u1[k] == u53_open(r[2], r[3])
    # the t and call words are distinct fields: swapping them changes every draw
    a, _ = sr.smooth_uniforms(seed, 2, np.arange(64), 9, 0, sr.PURPOSE_EXACT)
    b, _ = sr.smooth_uniforms(seed, 9, np.arange(64), 2, 0, sr.PURPOSE_EXACT)
    assert not np.any(a == b)
    assert np.all((a > 0) & (a < 1))
    # PaRIS: the run's seed mixed with kOnlineSeedMix; m = n * Np + i, t-field 0, call = t
    assert sr.paris_seed(0) == 0x9E3779B97F4A7C15 and sr.paris_seed(0x9E3779B97F4A7C15) == 0
    # draw_cdf: the first j with cdf[j] >= u * cdf[-1]; a weight-zero particle is never the answer
    cdf = np.array([0.0, 0.25, 0.25, 0.75, 1.0])
    assert list(sr.draw_cdf(cdf, np.array([1e-300, 0.25, 0.2500001, 0.75, 0.9999]))) == [1, 1, 3, 3, 4]
    assert sr.draw_cdf(np.zeros(4), np.array([0.5]))[0] == 0


def test_all_zero_row_rule_is_the_reference_rule():
    """The reference's exact draw on a row with no positive weight: exp_and_normalise gives NaN everywhere and
    searchsorted on the NaN cumsum gives 0 for every u -- the rule the kernels follow."""
    for N in (1, 7, 300):
        lwm = np.full(N, -np.inf)
        with np.errstate(invalid="ignore"):
            W = orc.exp_and_normalise(lwm)
            assert np.all(np.isnan(W))
            for u in (1e-12, 0.3, 0.999999):
                assert orc.multinomial_once(W, u) == 0
    # the replay states the same rule, and refuses N - 1 or a NaN-weighted particle
    v = np.array([[-np.inf] * 5, [0.0, np.nan, -1.0, -np.inf, 0.5]], dtype=sr.LD)
    b = np.full(v.shape, 1e-15)
    assert sr.exact_draw_check(v, b, np.array([0.5, 0.5]), np.array([0, 4])) == (0, 1)
    with pytest.raises(AssertionError, match="all-zero"):
        sr.exact_draw_check(v, b, np.array([0.5, 0.5]), np.array([4, 4]))
    with pytest.raises(AssertionError, match="zero-weight"):
        sr.exact_draw_check(v, b, np.array([0.5, 0.5]), np.array([0, 1]))
    with pytest.raises(AssertionError, match="bracket"):
        sr.exact_draw_check(v, b, np.array([0.5, 0.01]), np.array([0, 4]))


@pytest.fixture(scope="module")
def gs():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_smoothing.npz"))


def golden_trans(name):
    from particles_b200 import kalman, state_space_models as ssm
    m = {"lg": lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "sv": lambda: ssm.StochVol(),
         "cox": lambda: ssm.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9),
         "mvlg2": lambda: kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=2)}[name]()
    return sr.Trans(spec_of(m, 50))


def oracle_model(name):
    return {"lg": lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "sv": lambda: orc.StochVol(),
            "cox": lambda: orc.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9),
            "mvlg2": lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[name]()


def _oracle(gs, name, fn, seed, *a, **kw):
    state = np.random.get_state()
    try:
        np.random.seed(seed)
        h = {"X": list(gs[f"{name}/X"]), "lw": list(gs[f"{name}/lw"]), "A": list(gs[f"{name}/A"])}
        return fn(h, osm.px_logpt(oracle_model(name)), *a, **kw)
    finally:
        np.random.set_state(state)


@pytest.mark.parametrize("name", list(SEEDS))
def test_replay_predicts_the_reference_on2_draws(gs, name):
    tr = golden_trans(name)
    X, lw = gs[f"{name}/X"], gs[f"{name}/lw"]
    M = int(gs["meta/T_N_M"][2])
    idx, noise = _oracle(gs, name, osm.backward_ON2, SEEDS[name] + 200, M)
    assert np.array_equal(idx, gs[f"{name}/idx_on2"])
    near = 0
    for t in range(X.shape[0] - 1):
        v, b = sr.row_values(tr, t + 1, X[t], lw[t], X[t + 1][idx[t + 1]])
        near += sr.exact_draw_check(v, b, noise["u"][:, t], idx[t])[0]
    assert near <= 1


@pytest.mark.parametrize("name", list(SEEDS))
def test_replay_predicts_the_reference_mcmc_and_reject(gs, name):
    tr = golden_trans(name)
    X, A, lw, bound = gs[f"{name}/X"], gs[f"{name}/A"], gs[f"{name}/lw"], gs[f"{name}/bound"]
    T, M = X.shape[0], int(gs["meta/T_N_M"][2])
    idx, noise = _oracle(gs, name, osm.backward_mcmc, SEEDS[name] + 300, M, nsteps=2)
    undecided = 0
    for t in range(T - 1):
        xn = sr.as_rows(X[t + 1])[idx[t + 1]]
        got, sure = sr.mcmc_step(tr, t, X[t], xn, A[t + 1][idx[t + 1]], noise["prop"][t], noise["lu"][t])
        assert np.array_equal(got[sure], idx[t][sure]), (name, t)
        undecided += int((~sure).sum())
    assert undecided <= 2
    for mt, key in ((None, ""), (2, "2")):
        seed = SEEDS[name] + (400 if mt is None else 500)
        idx, acc_rate, noise = _oracle(gs, name, osm.backward_reject, seed, M, lambda t: bound[t], max_trials=mt)
        assert np.array_equal(idx, gs[f"{name}/idx_reject" + key])
        for t in range(T - 1):
            xn = sr.as_rows(X[t + 1])[idx[t + 1]]
            first, choice, sure = sr.reject_trials(tr, t + 1, X[t], xn, noise["prop"][t], noise["lu"][t], bound[t + 1])
            assert sure.all()
            ok = first >= 0
            assert np.array_equal(choice[ok], idx[t][ok])
            nprop = np.where(ok, first + 1, noise["prop"].shape[2])
            assert ok.sum() / nprop.sum() == gs[f"{name}/acc_rate" + key][t]
            if (~ok).any():
                v, b = sr.row_values(tr, t + 1, X[t], lw[t], xn[~ok])
                sr.exact_draw_check(v, b, noise["u_exact"][t][~ok], idx[t][~ok])


@pytest.fixture(scope="module")
def gt():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_twofilter.npz"))


def test_twofilter_replay_predicts_the_oracle(gt):
    """ON2_ROWS and ON_LOGW checks hold on the float64 row restatement and the reference's log-weights."""
    import twofilter_oracle as tfo
    from particles_b200 import kalman, state_space_models as ssm
    models = {"cox": (ssm.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9), orc.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9)),
              "lg": (kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), orc.LinearGauss(sigmaX=1.0, sigmaY=0.2,
                                                                                          rho=0.9))}
    for name, (dm, om) in models.items():
        if f"{name}/X" not in gt.files:
            continue
        X, lw, Xi, lwi = gt[f"{name}/X"], gt[f"{name}/lw"], gt[f"{name}/Xinfo"], gt[f"{name}/lwinfo"]
        T = X.shape[0]
        tr = sr.Trans(spec_of(dm, T))
        logpt = osm.px_logpt(om)
        for t in (0, T // 2, T - 2):
            ti = T - 2 - t
            v = lw[t][None, :] + logpt(t + 1, X[t][None, :], Xi[ti][:, None])
            L = np.logaddexp.reduce(v, axis=1)
            psi = np.outer(Xi[ti], np.ones(X.shape[1])) * X[t][None, :]
            S = np.sum(np.exp(v - L[:, None]) * psi, axis=1)
            sr.on2_rows_check(tr, t, X[t], lw[t], Xi[ti], psi, L, S)
            r = np.random.RandomState(t)
            I, J = r.randint(0, Xi.shape[1], 300), r.randint(0, X.shape[1], 300)
            mf, mi = tfo.prop_modifiers(X, Xi, t)
            lo = logpt(t + 1, X[t][J], Xi[ti][I]) - mf[J] - mi[I]
            sr.on_logw_check(tr, t, X[t], Xi[ti], I, J, mf, mi, lo)


def test_online_replay_predicts_fp64_weights_and_phi():
    """The ON2 backward weights and both Phi updates computed in plain fp64 lie inside the replay's bounds."""
    from particles_b200 import state_space_models as ssm
    tr = sr.Trans(spec_of(ssm.Gordon_etal(), 12))
    r = np.random.RandomState(3)
    N = 300
    Xp, X, lwp = 3 * r.standard_normal(N), 3 * r.standard_normal(N), r.standard_normal(N)
    v = np.float64(sr.row_values(tr, 5, Xp, lwp, X[:40])[0])
    om = np.exp(v - v.max(1)[:, None])
    om /= om.sum(1)[:, None]
    sr.on2_weights_check(tr, 5, Xp, lwp, X[:40], om)
    K = 3
    phi_prev, psi = r.standard_normal((N, K)), r.standard_normal((40, N, K))
    phi = np.einsum("rn,rnk->rk", om, phi_prev[None] + psi) / om.sum(1)[:, None]
    sr.phi_on2_check(om, phi_prev, psi, phi)
    Np = 3
    B = r.randint(0, N, N * Np)
    psi2 = r.standard_normal((N * Np, K))
    phi2 = (phi_prev[B] + psi2).reshape(N, Np, K).sum(1) / Np
    sr.phi_paris_check(B, Np, phi_prev, psi2, phi2)
