"""Off-line smoothing on the H100: the device FFBS samplers (csrc/smcb_smooth.cu) behind
``ParticleHistory.backward_sampling_ON2 / _mcmc / _reject``, against the live reference's indices on its own
histories (tests/golden/golden_smoothing.npz, with the reference's randomness injected), against the plugin path
(``fk.logpt`` on CUDA tensors), against the Kalman smoother, and on the edge cases of the public surface."""
import os

import numpy as np
import pytest
import torch

from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = {"lg": 11, "sv": 12, "cox": 13, "mvlg2": 14}


@pytest.fixture(scope="module")
def gs():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_smoothing.npz"))


def _bounded(cls, bound):
    return type(cls.__name__ + "_bounded", (cls,), {"upper_bound_log_pt": lambda self, t: float(bound[t])})


def models(name, bound=None):
    from particles_b200 import kalman, state_space_models as ssm
    dev = {"lg": (kalman.LinearGauss, dict(sigmaX=1.0, sigmaY=0.2, rho=0.9)), "sv": (ssm.StochVol, {}),
           "cox": (ssm.DiscreteCox, dict(mu=0.0, sigma=0.5, phi=0.9)),
           "mvlg2": (kalman.MVLinearGauss_Guarniero_etal, dict(alpha=0.4, dx=2))}[name]
    cls, kw = dev
    dm = (_bounded(cls, bound) if bound is not None else cls)(**kw)
    om = {"lg": lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "sv": lambda: orc.StochVol(),
          "cox": lambda: orc.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9),
          "mvlg2": lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[name]()
    return dm, om


def golden_history(gs, name, fk):
    """A ParticleHistory holding the reference's own history (row-major (N, d) particles)."""
    from particles_b200 import resampling as rs
    from particles_b200.smoothing import ParticleHistory
    h = ParticleHistory(fk, False)
    X, lw, A = gs[f"{name}/X"], gs[f"{name}/lw"], gs[f"{name}/A"]
    for t in range(X.shape[0]):
        h.X.append(torch.from_numpy(np.ascontiguousarray(X[t])).cuda())
        h.A.append(None if t == 0 else torch.from_numpy(A[t]).cuda())
        h.wgts.append(rs.Weights(lw=torch.from_numpy(lw[t].copy()).cuda()))
    return h


def fk_of(gs, name):
    from particles_b200 import state_space_models as ssm
    dm, om = models(name, gs[f"{name}/bound"])
    return ssm.Bootstrap(ssm=dm, data=list(gs[f"{name}/data"])), om


def oracle_noise(gs, name, method, **kw):
    h = {"X": list(gs[f"{name}/X"]), "lw": list(gs[f"{name}/lw"]), "A": list(gs[f"{name}/A"])}
    _, om = models(name)
    bound = gs[f"{name}/bound"]
    state = np.random.get_state()
    try:
        if method == "on2":
            np.random.seed(SEEDS[name] + 200)
            return osm.backward_ON2(h, osm.px_logpt(om), kw["M"])
        if method == "mcmc":
            np.random.seed(SEEDS[name] + 300)
            return osm.backward_mcmc(h, osm.px_logpt(om), kw["M"], nsteps=2)
        np.random.seed(SEEDS[name] + (400 if kw.get("max_trials") is None else 500))
        return osm.backward_reject(h, osm.px_logpt(om), kw["M"], lambda t: bound[t], max_trials=kw.get("max_trials"))
    finally:
        np.random.set_state(state)


@pytest.mark.parametrize("name", list(SEEDS))
def test_on2_against_reference_indices(gs, name):
    """Every device draw brackets the reference's uniform on the NumPy CDF built from the device's own x_{t+1};
    at least 99.9 % of the indices equal the reference's."""
    fk, om = fk_of(gs, name)
    h = golden_history(gs, name, fk)
    M = int(gs["meta/T_N_M"][2])
    _, noise = oracle_noise(gs, name, "on2", M=M)
    paths = h.backward_sampling_ON2(M, noise=noise)
    idx = h._bs_idx.cpu().numpy()
    X, lw, T = gs[f"{name}/X"], gs[f"{name}/lw"], len(paths)
    assert np.array_equal(idx[-1], noise["idx_T"])
    ties = 0
    for t in range(T - 1):
        for m in range(M):
            xn = X[t + 1][idx[t + 1, m]]
            C = np.cumsum(orc.exp_and_normalise(lw[t] + om.PX(t + 1, X[t]).logpdf(xn)))
            n, u = idx[t, m], noise["u"][m, t]
            lo = C[n - 1] if n > 0 else 0.0
            if not (lo < u <= C[n]):
                assert min(abs(u - lo), abs(u - C[n])) < 1e-12, (name, t, m)
                ties += 1
    assert ties <= 1e-3 * M * (T - 1)
    assert np.mean(idx == gs[f"{name}/idx_on2"]) >= 0.999
    P = torch.stack(paths).cpu().numpy()
    ref = np.array([X[t][idx[t]] for t in range(T)])
    assert np.array_equal(P, ref)


@pytest.mark.parametrize("name", list(SEEDS))
def test_mcmc_and_reject_against_reference(gs, name):
    fk, _ = fk_of(gs, name)
    h = golden_history(gs, name, fk)
    M = int(gs["meta/T_N_M"][2])
    need = 1.0 if name != "mvlg2" else 0.999        # MVLinearGauss: BLAS vs fma algebra, 1e-11 apart
    _, noise = oracle_noise(gs, name, "mcmc", M=M)
    h.backward_sampling_mcmc(M, nsteps=2, noise=noise)
    assert np.mean(h._bs_idx.cpu().numpy() == gs[f"{name}/idx_mcmc"]) >= need
    for mt, key in ((None, ""), (2, "2")):
        _, acc, noise = oracle_noise(gs, name, "reject", M=M, max_trials=mt)
        h.backward_sampling_reject(M, max_trials=mt, noise=noise)
        assert np.mean(h._bs_idx.cpu().numpy() == gs[f"{name}/idx_reject" + key]) >= need
        if need == 1.0:
            assert np.array_equal(h.acc_rate, gs[f"{name}/acc_rate" + key])
        else:
            np.testing.assert_allclose(h.acc_rate, gs[f"{name}/acc_rate" + key], atol=0.02)


def _fused_history(model, y, N, seed=3, smoothing_model=None):
    """Forward pass of a stock model on the fused kernels; ``smoothing_model`` (a subclass adding
    upper_bound_log_pt, which the filter's stricter recogniser would send down the plugin path) for the backward
    pass."""
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, store_history=True, seed=seed)
    assert pf.fused
    pf.run()
    if smoothing_model is not None:
        pf.hist.fk = ssm.Bootstrap(ssm=smoothing_model, data=y)
    return pf


def test_device_density_matches_plugin_logpt():
    """The device transition density of every fused model against ``fk.logpt`` on CUDA tensors: the same ON2
    draws (same injected uniforms) through the kernel and through the plugin path."""
    from particles_b200 import kalman, state_space_models as ssm
    cases = [ssm.StochVol(), ssm.StochVolLeverage(phi=-0.5), kalman.LinearGauss(rho=0.8), ssm.Gordon_etal(),
             ssm.ThetaLogistic(), ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), ssm.BearingsOnly(),
             kalman.MVLinearGauss_Guarniero_etal(0.4, 2)]
    T, N, M = 8, 64, 16
    r = np.random.RandomState(0)
    for model in cases:
        y = [np.atleast_1d(v.cpu().numpy() if hasattr(v, "cpu") else v) for v in model.simulate(T)[1]] \
            if not isinstance(model, ssm.BearingsOnly) else [np.array([0.5 + 0.01 * t]) for t in range(T)]
        pf = _fused_history(model, y, N)
        assert ssm.transition_spec(pf.fk) is not None
        noise = {"idx_T": r.randint(0, N, M), "u": r.rand(M, T - 1)}
        dev = pf.hist.backward_sampling_ON2(M, noise=noise)
        idx_dev = pf.hist._bs_idx.cpu().numpy()

        class Plugin(ssm.Bootstrap):
            def logpt(self, t, xp, x):
                return ssm.Bootstrap.logpt(self, t, xp, x)
        pf.hist.fk = Plugin(ssm=model, data=y)
        assert ssm.transition_spec(pf.hist.fk) is None
        plug = pf.hist.backward_sampling_ON2(M, noise=noise)
        idx_plug = pf.hist._bs_idx.cpu().numpy()
        assert np.mean(idx_dev == idx_plug) >= 0.99, type(model).__name__
        same = idx_dev[0] == idx_plug[0]
        np.testing.assert_array_equal(dev[0].cpu().numpy()[same], plug[0].cpu().numpy()[same])


def _kalman_check(om, y, pf, M, methods, nsig=6.0):
    mean, cov = osm.kalman_smoother(om, y)
    sd = np.sqrt(np.array([np.diag(np.atleast_2d(c)) for c in cov]))
    out = {}
    for meth in methods:
        if meth == "on2":
            paths = pf.hist.backward_sampling_ON2(M, seed=7)
        elif meth == "mcmc":
            paths = pf.hist.backward_sampling_mcmc(M, seed=7)
        else:
            paths = pf.hist.backward_sampling_reject(M, seed=7)
            assert np.all((pf.hist.acc_rate > 0) & (pf.hist.acc_rate <= 1))
        P = torch.stack(paths).cpu().numpy().reshape(len(y), M, -1)
        est = P.mean(axis=1)
        z = (est - mean.reshape(len(y), -1)) / (sd / np.sqrt(M))
        # smoothed means within nsig standard errors of the exact ones; the draws are correlated through the
        # N filter particles, so the envelope is wide but still far below the spread of the data
        assert np.max(np.abs(z)) < nsig * 3, (meth, np.max(np.abs(z)))
        assert np.mean(np.abs(z)) < nsig, (meth, np.mean(np.abs(z)))
        out[meth] = est
    return out


def test_smoothed_means_match_kalman_lineargauss():
    from particles_b200 import kalman
    om = orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9)
    om.F, om.G, om.covX, om.covY = np.array([[0.9]]), np.eye(1), np.eye(1), np.array([[0.25]])
    om.mu0, om.cov0 = np.zeros(1), np.array([[om.sigma0 ** 2]])
    np.random.seed(21)
    _, y = orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9).simulate(40)

    class LG(kalman.LinearGauss):
        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi)
    N = M = 20000
    kw = dict(sigmaX=1.0, sigmaY=0.5, rho=0.9)
    pf = _fused_history(kalman.LinearGauss(**kw), y, N, smoothing_model=LG(**kw))
    _kalman_check(om, y, pf, M, ("mcmc", "reject"))
    pf = _fused_history(kalman.LinearGauss(**kw), y, 4096, smoothing_model=LG(**kw))
    _kalman_check(om, y, pf, 4096, ("on2",))


@pytest.mark.parametrize("dx", [2, 4])
def test_smoothed_means_match_kalman_mvlineargauss(dx):
    from particles_b200 import kalman

    class MV(kalman.MVLinearGauss_Guarniero_etal):
        def upper_bound_log_pt(self, t):
            return -0.5 * self.dx * np.log(2 * np.pi)
    om = orc.MVLinearGauss_Guarniero_etal(0.4, dx)
    np.random.seed(30 + dx)
    _, y = om.simulate(30)
    y = [np.asarray(v).reshape(-1) for v in y]
    stock = kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=dx)
    pf = _fused_history(stock, y, 20000, smoothing_model=MV(alpha=0.4, dx=dx))
    assert pf.hist.X[0].stride() == (1, 20000)           # fused layout: strided (N, d) views of SoA buffers
    _kalman_check(om, y, pf, 20000, ("mcmc", "reject"))
    pf = _fused_history(stock, y, 2048, smoothing_model=MV(alpha=0.4, dx=dx))
    _kalman_check(om, y, pf, 2048, ("on2",))


def test_stochvol_methods_agree():
    from particles_b200 import state_space_models as ssm

    class SV(ssm.StochVol):
        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi * self.sigma ** 2)
    y = list(orc.config2_data(40, 3))
    y = [np.atleast_1d(v) for v in y]
    pf = _fused_history(ssm.StochVol(), y, 4096, smoothing_model=SV())
    P = {}
    for meth in ("on2", "mcmc", "reject"):
        fn = {"on2": pf.hist.backward_sampling_ON2, "mcmc": pf.hist.backward_sampling_mcmc,
              "reject": pf.hist.backward_sampling_reject}[meth]
        P[meth] = torch.stack(fn(4096, seed=5)).cpu().numpy()
    sd = P["on2"].std(axis=1) / np.sqrt(4096)
    for a, b in (("on2", "mcmc"), ("on2", "reject"), ("mcmc", "reject")):
        z = (P[a].mean(axis=1) - P[b].mean(axis=1)) / (np.sqrt(2) * sd)
        assert np.max(np.abs(z)) < 18 and np.mean(np.abs(z)) < 6, (a, b)


def test_edge_cases_and_surface():
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    y = [np.array([0.1 * t]) for t in range(6)]
    # T = 1: only the final-time draw
    pf = _fused_history(ssm.StochVol(), y[:1], 100)
    for fn in (pf.hist.backward_sampling_ON2, pf.hist.backward_sampling_mcmc):
        p = fn(5)
        assert len(p) == 1 and tuple(p[0].shape) == (5,)
    # M = 1: squeezed output (a list of states)
    pf = _fused_history(ssm.StochVol(), y, 50)
    p = pf.hist.backward_sampling_mcmc(1)
    assert len(p) == 6 and p[0].dim() == 0
    # N = 1: every path is the single particle
    from particles_b200 import resampling as rs
    from particles_b200.smoothing import ParticleHistory
    h1 = ParticleHistory(ssm.Bootstrap(ssm=ssm.StochVol(), data=y), False)
    for t in range(6):
        h1.X.append(torch.full((1,), 0.1 * t, dtype=torch.float64, device="cuda"))
        h1.A.append(None if t == 0 else torch.zeros(1, dtype=torch.int64, device="cuda"))
        h1.wgts.append(rs.Weights(lw=torch.zeros(1, dtype=torch.float64, device="cuda")))
    for fn in (h1.backward_sampling_ON2, h1.backward_sampling_mcmc):
        p = fn(3)
        assert all(torch.equal(p[t], torch.full((3,), 0.1 * t, dtype=torch.float64, device="cuda")) for t in range(6))
    # fused d = 4 (strided) history
    from particles_b200 import kalman
    pf = _fused_history(kalman.MVLinearGauss_Guarniero_etal(0.4, 4), [np.ones(4) * 0.1 * t for t in range(6)], 300)
    p = pf.hist.backward_sampling_mcmc(20, seed=1)
    idx = pf.hist._bs_idx
    assert tuple(p[0].shape) == (20, 4)
    for t in range(6):
        assert torch.equal(p[t], pf.hist.X[t][idx[t]])
    # views into ONE tensor
    assert p[0].untyped_storage().data_ptr() == p[5].untyped_storage().data_ptr()
    # same seed -> identical paths, other seed -> different
    a = torch.stack(pf.hist.backward_sampling_mcmc(20, seed=1))
    b = torch.stack(pf.hist.backward_sampling_mcmc(20, seed=2))
    assert torch.equal(a, torch.stack(p)) and not torch.equal(a, b)
    # rejection without a bound: the reference's NotImplementedError
    with pytest.raises(NotImplementedError, match="upper_bound_log_pt"):
        pf.hist.backward_sampling_reject(10)
    with pytest.raises(NotImplementedError):
        pf.hist.backward_sampling_qmc(10)
    with pytest.raises(NotImplementedError, match="not built"):
        pf.hist.two_filter_smoothing(0, None, None, None)

    # plugin path: the README's ToySSM, a user model
    class ToySSM(ssm.StateSpaceModel):
        def PX0(self):
            from particles_b200 import distributions as dists
            return dists.Normal()

        def PX(self, t, xp):
            from particles_b200 import distributions as dists
            return dists.Normal(loc=xp)

        def PY(self, t, xp, x):
            from particles_b200 import distributions as dists
            return dists.Normal(loc=x, scale=0.2)

        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi)
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=ToySSM(), data=y), N=200, store_history=True, seed=4)
    pf.run()
    assert not pf.fused and ssm.transition_spec(pf.fk) is None
    for fn in (pf.hist.backward_sampling_ON2, pf.hist.backward_sampling_mcmc, pf.hist.backward_sampling_reject):
        p = fn(8, seed=3)
        idx = pf.hist._bs_idx
        assert len(p) == 6 and all(torch.equal(p[t], pf.hist.X[t][idx[t]]) for t in range(6))
    assert pf.hist.acc_rate.shape == (5,)
