"""Single-run variance estimators and fixed-lag smoothing on the H100 (csrc/smcb_variance.cu behind
``particles_b200.variance_estimators`` and ``collectors.Fixed_lag_smooth``): replays of the live reference's runs
(tests/golden/golden_variance.npz), the fused ``run()`` against the NumPy oracle (tests/variance_oracle.py) with
injected noise, full size without host syncs, determinism, statistical parity with the reference, the reference's
own objects under ``install()``, and the errors of the public surface."""
import gc
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

import variance_oracle as vo
from oracle import smc_numpy as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
CASES = {"sv_sys": "systematic", "lg_multi": "multinomial", "sv_strat": "stratified", "mvlg2": "systematic",
         "sv_ssp": "ssp", "sv_resid": "residual", "sv_kill": "killing", "collapse": "multinomial"}
HAND = ["all_equal", "unsorted_ends", "unsorted", "n1", "singletons", "vector"]


@pytest.fixture(scope="module")
def gv():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_variance.npz"))


def host(t):
    return t.detach().cpu().numpy()


def rel(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))


def phi_of(name):
    return None if name == "mvlg2" else (lambda x: x ** 2)


def phi_fl(xs):
    return sum(x if x.ndim == 1 else x[:, 0] for x in xs)


def replay(gv, name, cols_):
    """Drive public collectors over a golden history through a stub of the running SMC (plugin path)."""
    from particles_b200 import resampling as rs, smoothing
    X, lw, A, rsf = gv[f"{name}/X"], gv[f"{name}/lw"], gv[f"{name}/A"].astype(np.int64), gv[f"{name}/rs"]
    hist = smoothing.RollingParticleHistory(int(gv["meta/T_N_LAG"][2]))
    for t in range(X.shape[0]):
        wg = rs.Weights(lw=torch.from_numpy(lw[t].copy()).cuda())
        smc = types.SimpleNamespace(fused=False, t=t, resampling=CASES[name], X=torch.from_numpy(X[t].copy()).cuda(),
                                    wgts=wg, W=wg.W, rs_flag=bool(rsf[t]), N=X.shape[1],
                                    A=None if t == 0 else torch.from_numpy(A[t].copy()).cuda(), hist=hist)
        hist.save(smc)
        for c in cols_:
            c.collect(smc)


def check_close(got, ref, tol=1e-12, scale=None):
    """Within ``tol`` relative, and exact zeros where the reference gives zeros.  ``scale``: the errors are relative
    to it instead (the rows of Lag_based_var share one centring, and the long lags of a collapsed genealogy cancel
    to a small fraction of the lag-0 estimate)."""
    got, ref = np.array(got, dtype=float), np.asarray(ref, dtype=float)
    assert got.shape == ref.shape
    assert np.array_equal(got == 0.0, ref == 0.0)
    if scale is None:
        assert rel(got, ref) < tol
    else:
        assert np.max(np.abs(got - ref)) < tol * scale


@pytest.mark.parametrize("name", list(CASES))
def test_replay_against_reference(gv, name):
    from particles_b200 import collectors as cols, variance_estimators as ve
    phi = phi_of(name)
    c = [ve.Var(phi=phi), ve.Var_logLt(), ve.Lag_based_var(phi=phi), cols.Fixed_lag_smooth(phi=phi_fl)]
    replay(gv, name, c)
    check_close(c[0].summary, gv[f"{name}/var"])
    check_close(c[1].summary, gv[f"{name}/var_logLt"])
    check_close(c[3].summary, gv[f"{name}/fixed_lag_smooth"])
    assert isinstance(c[0].summary[-1], float) == (name != "mvlg2")
    lagv = gv[f"{name}/lag_based_var"]
    X, lw, A = gv[f"{name}/X"], gv[f"{name}/lw"], gv[f"{name}/A"].astype(np.int64)
    f = (lambda x: 1.0 * x) if phi is None else phi
    for t, row in enumerate(c[2].summary):
        assert len(row) == min(t + 1, lagv.shape[1])
        # the scale of the centred sums: (sum W |phi|)^2, which a degenerate genealogy cancels down from
        scale = max(np.max(np.abs(lagv[t, 0])), np.max(np.sum(vo.normalise(lw[t]) * np.abs(f(X[t])).T, -1)) ** 2)
        check_close(row, lagv[t, :len(row)], scale=scale)
    # var_estimate on the same inputs: the oracle's Eve rows and normalised weights
    got = [ve.var_estimate(vo.normalise(lw[t]), f(X[t]), B) for t, B in enumerate(vo.eve_rows(A))]
    check_close(got, gv[f"{name}/var"])


@pytest.mark.parametrize("case", HAND)
def test_var_estimate_hand_made(gv, case):
    from particles_b200 import variance_estimators as ve
    W, phi, B = (gv[f"hand/{case}/{k}"] for k in ("W", "phi", "B"))
    got = ve.var_estimate(torch.from_numpy(W).cuda(), phi, B)
    check_close(np.atleast_1d(got), np.atleast_1d(gv[f"hand/{case}/out"]))


def make_noise(N, T, seed):
    r = np.random.RandomState(seed)
    return r.standard_normal((T, N)), r.rand(T, N + 1)


def sv_data(T, seed=5):
    np.random.seed(seed)
    _, y = orc.StochVol().simulate(T)
    return [np.atleast_1d(v) for v in y]


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_fused_run_against_oracle(scheme):
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm, variance_estimators as ve
    N, T, lag = 2000, 100, 8
    y = sv_data(T)
    z, u = make_noise(N, T, 17)
    nu = {"systematic": 1, "stratified": N, "multinomial": N + 1}[scheme]
    ref = orc.SMC(orc.Bootstrap(orc.StochVol(), y), N=N, resampling=scheme,
                  noise=orc.InjectedNoise(z, [row[:nu] for row in u]), keep=True).run()
    X = [tr["X"] for tr in ref.trace]
    lw = [tr["lw"] for tr in ref.trace]
    A = [np.arange(N)] + [tr["A"] for tr in ref.trace[1:]]
    exp = vo.replay(X, lw, A, lambda x: x, lag)
    mk = lambda **kw: pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=N, resampling=scheme,  # noqa: E731
                             noise=(z, u), **kw)
    pf = mk(collect=[ve.Var(), ve.Var_logLt()])
    assert pf.fused
    pf.run()
    ph = mk(collect=[ve.Lag_based_var()], store_history=lag)
    anc = []
    for _ in ph:
        if ph.t > 1 and ph.rs_flag:
            anc.append((ph.t - 1, host(ph.A)))
    assert anc and all(np.array_equal(a, A[t]) for t, a in anc)    # the ancestors match the oracle
    check_close(pf.summaries.var, exp["var"])
    check_close(pf.summaries.var_logLt, exp["var_logLt"])
    for t in range(T):
        check_close(ph.summaries.lag_based_var[t], exp["lag_based_var"][t],
                    scale=np.max(np.abs(exp["lag_based_var"][t][0])))


def test_full_size_against_oracle():
    """N = 1e6: the estimates at several t against the oracle on the history pulled back to the host."""
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm, variance_estimators as ve
    N, T, at = 10 ** 6, 100, (0, 10, 57, 99)
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=sv_data(T)), N=N, seed=3,
                collect=[ve.Var(), ve.Var_logLt()])
    B = np.arange(N)
    for _ in pf:
        t = pf.t - 1
        if t > 0 and pf.rs_flag:
            B = B[host(pf.A)]
        if t in at:
            W = vo.normalise(host(pf.wgts.lw))
            check_close([pf.summaries.var[t]], [vo.var_estimate(W, host(pf.X), B)])
            check_close([pf.summaries.var_logLt[t]], [vo.var_logLt(W, B)])
    assert sum(pf.summaries.rs_flags) > 0


def test_fused_run_has_no_host_sync(monkeypatch):
    import particles_b200 as pb
    from particles_b200 import core, state_space_models as ssm, variance_estimators as ve

    def no_state(self):
        raise AssertionError("_FusedEngine.state called")
    monkeypatch.setattr(core._FusedEngine, "state", no_state)
    counts, where = [], []
    for T in (20, 20, 200):       # the first window holds torch's one-time set-up: not counted
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=sv_data(T)), N=10 ** 6, seed=1,
                    collect=[ve.Var(phi=lambda x: x ** 2), ve.Var_logLt()])
        assert pf.fused
        torch.cuda.synchronize()
        gc.collect()
        gc.disable()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                pf.run()
            finally:
                torch.cuda.set_sync_debug_mode(0)
                gc.enable()
        syncs = [x for x in w if "synchroniz" in str(x.message)]
        counts.append(len(syncs))
        where.append([f"{x.filename}:{x.lineno}" for x in syncs])
        assert len(pf.summaries.var) == T and len(pf.summaries.var_logLt) == T
    assert counts[1] == counts[2], (counts, where)


def _sv_run(collect, T=60, **kw):
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=sv_data(T)), N=5000, collect=collect, seed=7, **kw)
    pf.run()
    return pf


def test_determinism_paths_and_fusion_modes(monkeypatch):
    import particles_b200 as pb
    from particles_b200 import collectors as cols, state_space_models as ssm, variance_estimators as ve
    mk = lambda: [ve.Var(phi=lambda x: x ** 2), ve.Var_logLt()]  # noqa: E731
    outs = []
    for mode in ("0", "1", "2", "1"):
        monkeypatch.setenv("SMCB_FUSE", mode)
        pf = _sv_run(mk())
        outs.append((pf.summaries.var, pf.summaries.var_logLt))
    for o in outs[1:]:
        assert o == outs[0]                                        # same seed -> the same bits
    ps = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=sv_data(60)), N=5000, collect=mk(), seed=7)
    for _ in ps:                                                    # per-step loop
        pass
    assert (ps.summaries.var, ps.summaries.var_logLt) == outs[0]
    # Moments() and Paris() next to these collectors keep their own results, and these keep theirs
    SV = type("SVA", (ssm.StochVol,), {"add_func": lambda self, t, xp, x: 0.0 * x if t == 0 else (x - xp) ** 2,
                                       "upper_bound_log_pt": lambda self, t: -0.5 * np.log(2 * np.pi * self.sigma ** 2)})
    run = lambda collect: pb.SMC(fk=ssm.Bootstrap(ssm=SV(), data=sv_data(60)), N=5000, collect=collect,  # noqa: E731
                                 seed=7)
    alone = run([cols.Moments(), cols.Paris()])
    alone.run()
    both = run([cols.Moments(), cols.Paris()] + mk())
    both.run()
    assert both.fused and both._dev_moments
    assert both.summaries.paris == alone.summaries.paris and both.summaries.moments == alone.summaries.moments
    assert (both.summaries.var, both.summaries.var_logLt) == outs[0]


def test_statistical_parity_with_reference(gv):
    """300 device runs of the notebook's model: the mean of var_logLt[t] and var[t] against the reference's within
    4 combined standard errors."""
    import particles_b200 as pb
    from particles_b200 import kalman, state_space_models as ssm, variance_estimators as ve
    runs, T, N = (int(v) for v in gv["stat/runs"])
    fk = ssm.Bootstrap(ssm=kalman.LinearGauss(rho=0.9, sigmaX=1.0, sigmaY=0.2), data=list(gv["stat/data"]))
    v, vl = [], []
    for r in range(runs):
        pf = pb.SMC(fk=fk, N=N, resampling="multinomial", collect=[ve.Var(), ve.Var_logLt()], seed=1000 + r)
        pf.run()
        v.append(pf.summaries.var)
        vl.append(pf.summaries.var_logLt)
    for key, a in (("var", np.array(v)), ("var_logLt", np.array(vl))):
        for t in (9, 29, 49):
            se = np.sqrt(a[:, t].var(ddof=1) / runs + gv[f"stat/{key}_sd"][t] ** 2 / runs)
            assert abs(a[:, t].mean() - gv[f"stat/{key}_mean"][t]) < 4 * se, (key, t)


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "particles")), reason="the reference is not staged")
def test_reference_collectors_under_install():
    pytest.importorskip("numba")             # the reference's variance_estimators imports it
    sys.path.insert(0, REF)
    try:
        import particles
        from particles import collectors as rcols, state_space_models as rssm, variance_estimators as rve
        import particles_b200 as pb
        from particles_b200 import variance_estimators as ve
        uninstall = pb.install()
        try:
            y = sv_data(30)
            fk = rssm.Bootstrap(ssm=rssm.StochVol(), data=y)
            pf = particles.SMC(fk=fk, N=1000, seed=2, collect=[rve.Var(phi=lambda x: x ** 2), rve.Var_logLt()])
            assert isinstance(pf, pb.SMC) and pf.fused
            assert [type(c) for c in pf.summaries._collectors[3:]] == [ve.Var, ve.Var_logLt]
            pf.run()
            assert len(pf.summaries.var) == 30 and isinstance(pf.summaries.var_logLt[-1], float)
            ph = particles.SMC(fk=fk, N=1000, seed=2, store_history=4,
                               collect=[rve.Lag_based_var(), rcols.Fixed_lag_smooth(phi=phi_fl)])
            ph.run()
            assert len(ph.summaries.lag_based_var[-1]) == 4 and len(ph.summaries.fixed_lag_smooth) == 30
        finally:
            uninstall()
    finally:
        sys.path.remove(REF)


def test_errors(gv):
    import particles_b200 as pb
    from particles_b200 import collectors as cols, state_space_models as ssm, variance_estimators as ve
    fk = ssm.Bootstrap(ssm=ssm.StochVol(), data=sv_data(10))
    with pytest.raises(ValueError):
        pb.SMC(fk=fk, N=100, collect=[ve.Var(phi=lambda x: x[:10])]).run()
    with pytest.raises(ValueError):
        ve.var_estimate(np.ones(5) / 5, np.ones((5, 2, 2)), np.arange(5))
    with pytest.raises(AttributeError):
        pb.SMC(fk=fk, N=100, collect=[ve.Lag_based_var()]).run()
    with pytest.raises(TypeError):
        pb.SMC(fk=fk, N=100, store_history=3, collect=[cols.Fixed_lag_smooth()]).run()
    # a scheme said to give sorted ancestors that does not: the kernel's flag is raised at the flush
    gv_resid = {k.replace("sv_resid/", "x/"): gv[k] for k in gv.files if k.startswith("sv_resid/")}
    gv_resid["meta/T_N_LAG"] = gv["meta/T_N_LAG"]
    CASES["x"] = "systematic"
    try:
        with pytest.raises(RuntimeError):
            replay(gv_resid, "x", [ve.Var_logLt()])
    finally:
        del CASES["x"]
