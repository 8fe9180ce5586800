"""On-line smoothing on the H100: the naive, O(N^2) and PaRIS collectors (csrc/smcb_online.cu behind
``particles_b200.collectors``) against the live reference on its own histories (tests/golden/golden_online.npz, with
the reference's PaRIS randomness injected), against the Kalman smoother, inside a fused ``run()`` without host
syncs, and on the edge cases of the public surface."""
import gc
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

import online_oracle as oo
from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
PARIS = [("paris", 2, None), ("paris2", 3, 2)]


@pytest.fixture(scope="module")
def go():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_online.npz"))


def oracle_model(name):
    return {"lg": lambda: orc.LinearGauss(**oo.PARAMS["lg"]), "sv": lambda: orc.StochVol(),
            "cox": lambda: orc.DiscreteCox(**oo.PARAMS["cox"]),
            "mvlg2": lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[name]()


def with_hooks(cls, name):
    """A user subclass of a stock model adding only add_func and the bound (what the book scripts write)."""
    def add_func(self, t, xp, x):
        return oo.add_func(name, self)(t, xp, x)

    def upper_bound_log_pt(self, t):
        return oo.log_bound(name, self)(t)
    return type(cls.__name__ + "A", (cls,), {"add_func": add_func, "upper_bound_log_pt": upper_bound_log_pt})


def device_model(name, plugin=False):
    from particles_b200 import distributions as dists, kalman, state_space_models as ssm
    if plugin:        # user models written with particles_b200.distributions: fk.logpt on CUDA tensors
        class LG(ssm.StateSpaceModel):
            default_params = dict(sigmaX=1.0, sigmaY=0.2, rho=0.9)

            def PX(self, t, xp):
                return dists.Normal(loc=self.rho * xp, scale=self.sigmaX)

        class SV(ssm.StateSpaceModel):
            default_params = dict(mu=-1.02, rho=0.9702, sigma=0.178)

            def PX(self, t, xp):
                return dists.Normal(loc=self.mu + self.rho * (xp - self.mu), scale=self.sigma)
        return with_hooks({"lg": LG, "sv": SV}[name], name)()
    cls = {"lg": kalman.LinearGauss, "sv": ssm.StochVol, "cox": ssm.DiscreteCox,
           "mvlg2": kalman.MVLinearGauss_Guarniero_etal}[name]
    return with_hooks(cls, name)(**oo.PARAMS[name])


def replay(go, name, fk, col):
    """Drive a public collector over the golden history through a stub of the running SMC; returns per-step B."""
    X, lw, A = go[f"{name}/X"], go[f"{name}/lw"], go[f"{name}/A"]
    Bs = []
    for t in range(X.shape[0]):
        smc = types.SimpleNamespace(fused=False, fk=fk, _seed=3, t=t, X=torch.from_numpy(X[t].copy()).cuda(),
                                    wgts=types.SimpleNamespace(lw=torch.from_numpy(lw[t].copy()).cuda()),
                                    A=None if t == 0 else torch.from_numpy(A[t].copy()).cuda())
        col.collect(smc)
        if t > 0 and hasattr(col, "_B"):
            Bs.append(col._B.cpu().numpy())
    return Bs


def rel(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))


@pytest.mark.parametrize("name,plugin", [("lg", False), ("cox", False), ("sv", False), ("mvlg2", False),
                                         ("lg", True), ("sv", True)])
def test_collectors_against_reference(go, name, plugin):
    from particles_b200 import collectors as cols, state_space_models as ssm
    fk = ssm.Bootstrap(ssm=device_model(name, plugin), data=list(go[f"{name}/data"]))
    assert (ssm.transition_spec(fk) is None) == plugin
    col = cols.Online_smooth_naive()
    replay(go, name, fk, col)
    assert rel(col.summary, go[f"{name}/naive"]) < 1e-13
    col = cols.Online_smooth_ON2()
    replay(go, name, fk, col)
    assert rel(col.summary, go[f"{name}/on2"]) < 1e-10
    assert isinstance(col.summary[-1], float) == (name != "mvlg2")
    m = oracle_model(name)
    h = oo.history(go, name)
    for i, (key, Np, mt) in enumerate(PARIS):
        np.random.seed(oo.SEEDS[name] + 202 + i)
        _, nprop, Bs_ref, noises = oo.paris(h, oo.add_func(name, m), osm.px_logpt(m), oo.log_bound(name, m),
                                            Nparis=Np, max_trials=mt)
        col = cols.Paris(Nparis=Np, max_trials=mt, noise=lambda t: noises[t - 1])
        Bs = replay(go, name, fk, col)
        same = np.mean([np.mean(a == b) for a, b in zip(Bs, Bs_ref)])
        assert same == 1.0 if name != "mvlg2" else same >= 0.999, (key, same)
        assert col.nprop == nprop
        np.testing.assert_array_equal(np.array(col.nprop, dtype=float), go[f"{name}/{key}_nprop"])
        if same == 1.0:
            assert rel(col.summary, go[f"{name}/{key}"]) < 1e-12, key


def _lg_problem(T=100):
    om = orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9)
    om.F, om.G, om.covX, om.covY = np.array([[0.9]]), np.eye(1), np.eye(1), np.array([[0.25]])
    om.mu0, om.cov0 = np.zeros(1), np.array([[om.sigma0 ** 2]])
    np.random.seed(31)
    _, y = orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9).simulate(T)
    y = [np.atleast_1d(np.asarray(v, dtype=float)) for v in y]
    return om, y


@pytest.mark.parametrize("fused", [True, False])
def test_against_kalman(fused):
    """Phi_t estimates sum_{s <= t} E[X_s | y_{0:t}] for psi = x: the exact value from the Kalman smoother on the
    prefix; the mean of 8 seeds within 4 empirical standard errors, per method and t."""
    import particles_b200 as pb
    from particles_b200 import collectors as cols, kalman, state_space_models as ssm
    om, y = _lg_problem()
    exact = {t: osm.kalman_smoother(om, y[:t + 1])[0].sum() for t in (10, 50, 99)}
    LG = type("LG", (kalman.LinearGauss,), {"add_func": lambda self, t, xp, x: 1.0 * x,
                                            "upper_bound_log_pt": lambda self, t: -0.5 * np.log(2.0 * np.pi)})
    runs = [(lambda: cols.Paris(), 10 ** 5, "paris"), (lambda: cols.Online_smooth_ON2(), 4096, "on2"),
            (lambda: cols.Online_smooth_naive(), 10 ** 6, "naive")]
    for mk, N, key in runs:
        est = []
        for seed in range(8):
            pf = pb.SMC(fk=ssm.Bootstrap(ssm=LG(sigmaX=1.0, sigmaY=0.5, rho=0.9), data=y), N=N, collect=[mk()],
                        seed=100 + seed, fused=fused)
            assert pf.fused == fused
            pf.run()
            est.append(getattr(pf.summaries, {"paris": "paris", "on2": "online_smooth_ON2",
                                             "naive": "online_smooth_naive"}[key]))
        est = np.array(est)
        for t, ex in exact.items():
            se = est[:, t].std(ddof=1) / np.sqrt(8)
            assert abs(est[:, t].mean() - ex) < 4 * se + 1e-9 * abs(ex), (key, t, est[:, t].mean(), ex, se)


def _sv_fk(T):
    from particles_b200 import state_space_models as ssm
    np.random.seed(5)
    _, y = orc.StochVol().simulate(T)
    return ssm.Bootstrap(ssm=device_model("sv"), data=[np.atleast_1d(v) for v in y])


def test_fused_run_has_no_host_sync(monkeypatch):
    import particles_b200 as pb
    from particles_b200 import collectors as cols, core

    def no_state(self):
        raise AssertionError("_FusedEngine.state called")
    monkeypatch.setattr(core._FusedEngine, "state", no_state)
    counts, where = [], []
    for T in (20, 20, 200):       # the first window holds torch's one-time set-up: not counted
        pf = pb.SMC(fk=_sv_fk(T), N=10 ** 4, collect=[cols.Paris()], seed=1)
        assert pf.fused
        torch.cuda.synchronize()
        gc.collect()              # an object freed by the collector inside the window would add its own sync
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
        assert len(pf.summaries.paris) == T and len(pf.summaries._collectors[3].nprop) == T
    assert counts[1] == counts[2], (counts, where)


def _sv_run(collect, **kw):
    import particles_b200 as pb
    pf = pb.SMC(fk=_sv_fk(60), N=5000, collect=collect, seed=7, **kw)
    pf.run()
    return pf


def test_determinism_and_fusion_modes(monkeypatch):
    from particles_b200 import collectors as cols
    outs = []
    for mode in ("0", "1", "2", "1"):
        monkeypatch.setenv("SMCB_FUSE", mode)
        pf = _sv_run([cols.Paris(), cols.Online_smooth_naive(), cols.Online_smooth_ON2()])
        outs.append((pf.summaries.paris, pf.summaries.online_smooth_naive, pf.summaries.online_smooth_ON2,
                     pf.summaries._collectors[3].nprop))
    for o in outs[1:]:
        assert o == outs[0]


def test_moments_next_to_smoother_and_per_step_path():
    from particles_b200 import collectors as cols
    pf = _sv_run([cols.Moments(), cols.Paris(Nparis=3)])
    assert pf._dev_moments
    import particles_b200 as pb
    ps = pb.SMC(fk=_sv_fk(60), N=5000, collect=[cols.Moments(), cols.Paris(Nparis=3)], seed=7)
    for _ in ps:                       # per-step path: the collectors see each generation
        pass
    assert pf.summaries.paris == ps.summaries.paris
    assert pf.summaries._collectors[4].nprop == ps.summaries._collectors[4].nprop
    np.testing.assert_allclose([m["mean"] for m in pf.summaries.moments], [m["mean"] for m in ps.summaries.moments],
                               rtol=1e-12)
    pl = _sv_run([cols.Paris(Nparis=3)], fused=False)    # the plugin filter, same device draws
    assert not pl.fused and len(pl.summaries.paris) == 60


def test_routing_and_errors():
    import particles_b200 as pb
    from particles_b200 import collectors as cols, state_space_models as ssm
    np.random.seed(5)
    _, y = orc.StochVol().simulate(20)
    y = [np.atleast_1d(v) for v in y]
    hooks = ssm.Bootstrap(ssm=device_model("sv"), data=y)
    # a model with hooks runs fused only when it is smoothed on-line; a stock model routes as before
    assert ssm.fused_spec(hooks) is None and ssm.fused_spec(hooks, smoothing_hooks=True) is not None
    assert pb.SMC(fk=hooks, N=100).fused is False
    assert pb.SMC(fk=hooks, N=100, collect=[cols.Paris()]).fused is True
    stock = ssm.Bootstrap(ssm=ssm.StochVol(), data=y)
    assert pb.SMC(fk=stock, N=100).fused is True

    class Other(ssm.StochVol):          # overrides a closure: never fused
        def PX(self, t, xp):
            return ssm.StochVol.PX(self, t, xp)

        def add_func(self, t, xp, x):
            return x
    assert pb.SMC(fk=ssm.Bootstrap(ssm=Other(), data=y), N=100, collect=[cols.Paris()]).fused is False
    # a missing bound raises as in the reference; a missing add_func too
    nob = ssm.Bootstrap(ssm=type("SVf", (ssm.StochVol,), {"add_func": lambda self, t, xp, x: x})(), data=y)
    with pytest.raises(NotImplementedError):
        pb.SMC(fk=nob, N=100, collect=[cols.Paris()]).run()
    with pytest.raises(NotImplementedError):
        pb.SMC(fk=stock, N=100, collect=[cols.Online_smooth_naive()]).run()


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "particles")), reason="the reference is not staged")
def test_reference_collectors_under_install():
    sys.path.insert(0, REF)
    try:
        import particles
        from particles import collectors as rcols, state_space_models as rssm
        import particles_b200 as pb
        uninstall = pb.install()
        try:
            class SV(rssm.StochVol):
                def upper_bound_log_pt(self, t):
                    return -0.5 * np.log(2.0 * np.pi * self.sigma ** 2)

                def add_func(self, t, xp, x):
                    return 0.0 * x if t == 0 else (x - xp) ** 2
            np.random.seed(5)
            _, y = orc.StochVol().simulate(30)
            pf = particles.SMC(fk=rssm.Bootstrap(ssm=SV(), data=[np.atleast_1d(v) for v in y]), N=1000, seed=2,
                               collect=[rcols.Paris(Nparis=3), rcols.Online_smooth_ON2(), rcols.Online_smooth_naive()])
            assert isinstance(pf, pb.SMC) and pf.fused
            pf.run()
            assert len(pf.summaries.paris) == 30 and len(pf.summaries.online_smooth_ON2) == 30
            assert len(pf.summaries._collectors[3].nprop) == 30
        finally:
            uninstall()
    finally:
        sys.path.remove(REF)
