"""Two-filter smoothing on the H100: ``ParticleHistory.two_filter_smoothing`` (csrc/smcb_twofilter.cu on a stock
model's transition, ``fk.logpt`` on CUDA tensors otherwise) against the live reference's estimates on its own
histories (tests/golden/golden_twofilter.npz, with the reference's draws injected), against the Kalman smoother,
against FFBS through ``smoothing_worker``, against a float64 host replay at N = 8192, and on the edge cases of
the public surface."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import twofilter_oracle as otf  # noqa: E402

MU, PHI, SIGMA = 0.0, 0.9, 0.5
CASES = ("cox", "lg", "sv")


@pytest.fixture(scope="module")
def gt():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_twofilter.npz"))


def psit(t, x, xf, mu=MU, phi=PHI, sigma=SIGMA):
    """The book's additive function (book/smoothing/offline_smoothing.py), on tensors or arrays."""
    if t == 0:
        return (-0.5 / sigma ** 2 + (0.5 * (1.0 - phi ** 2) / sigma ** 4) * (x - mu) ** 2
                + psit(1, x, xf, mu, phi, sigma))
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((xf - mu) - phi * (x - mu)) ** 2


def add_func(name):
    return psit if name == "cox" else (lambda t, x, xf: x * xf)


def log_gamma_cox(x):
    scale = SIGMA / np.sqrt(1.0 - PHI ** 2)
    z = (x - MU) / scale
    return -z * z / 2.0 - 0.5 * np.log(2.0 * np.pi) - np.log(scale)


def stock_model(name, plugin=False):
    from particles_b200 import kalman, state_space_models as ssm
    cls, kw = {"cox": (ssm.DiscreteCox, dict(mu=MU, sigma=SIGMA, phi=PHI)),
               "lg": (kalman.LinearGauss, dict(sigmaX=1.0, sigmaY=0.5, rho=0.9)),
               "sv": (ssm.StochVol, {})}[name]
    if plugin:                                   # a user subclass overriding PX: fk.logpt on CUDA tensors
        cls = type("User" + cls.__name__, (cls,), {"PX": lambda self, t, xp, _c=cls: _c.PX(self, t, xp)})
    return cls(**kw)


def oracle_model(name):
    return {"cox": lambda: orc.DiscreteCox(mu=MU, sigma=SIGMA, phi=PHI),
            "lg": lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9),
            "sv": lambda: orc.StochVol()}[name]()


def _hist(fk, X, lw):
    from particles_b200 import resampling as rs
    from particles_b200.smoothing import ParticleHistory
    h = ParticleHistory(fk, False)
    for t in range(X.shape[0]):
        h.X.append(torch.from_numpy(np.ascontiguousarray(X[t])).cuda())
        h.A.append(None)
        h.wgts.append(rs.Weights(lw=torch.from_numpy(np.array(lw[t])).cuda()))
    return h


def golden_pair(gt, name, plugin=False):
    """The reference's forward history, and an information 'filter' holding its information history."""
    from particles_b200 import state_space_models as ssm
    y = list(gt[f"{name}/data"])
    fk = ssm.Bootstrap(ssm=stock_model(name, plugin), data=y)
    assert (ssm.transition_spec(fk) is None) == plugin
    h = _hist(fk, gt[f"{name}/X"], gt[f"{name}/lw"])
    info = types.SimpleNamespace(hist=_hist(fk, gt[f"{name}/Xinfo"], gt[f"{name}/lwinfo"]))
    return h, info


def golden_gamma(gt, name, ti):
    """The reference's loggamma(Xinfo_ti), computed on the host as the fixture fed it."""
    v = torch.from_numpy(otf.log_gamma(name, gt[f"{name}/Xinfo"][ti])).cuda()
    return lambda x: v


@pytest.mark.parametrize("plugin", [False, True], ids=["kernel", "plugin"])
@pytest.mark.parametrize("name", CASES)
def test_on2_matches_reference(gt, name, plugin):
    h, info = golden_pair(gt, name, plugin)
    T, f = h.T, add_func(name)
    est = torch.stack([h.two_filter_smoothing(t, info, lambda x, xf, t=t: f(t, x, xf), golden_gamma(gt, name, T - 2 - t))
                       for t in range(T - 1)]).cpu().numpy()
    np.testing.assert_allclose(est, gt[f"{name}/on2"], rtol=1e-10, atol=0)


@pytest.mark.parametrize("plugin", [False, True], ids=["kernel", "plugin"])
@pytest.mark.parametrize("tag", ["on", "prop"])
@pytest.mark.parametrize("name", CASES)
def test_on_with_reference_draws(gt, name, tag, plugin):
    h, info = golden_pair(gt, name, plugin)
    T, f = h.T, add_func(name)
    out = []
    for t in range(T - 1):
        kw = {}
        if tag == "prop":
            mf, mi = otf.prop_modifiers(gt[f"{name}/X"], gt[f"{name}/Xinfo"], t)
            kw = {"modif_forward": mf, "modif_info": mi}
        noise = {"I": gt[f"{name}/{tag}_I"][t].astype(np.int64), "J": gt[f"{name}/{tag}_J"][t].astype(np.int64)}
        e, s = h.two_filter_smoothing(t, info, lambda x, xf, t=t: f(t, x, xf), golden_gamma(gt, name, T - 2 - t),
                                      linear_cost=True, return_ess=True, noise=noise, **kw)
        assert e.dim() == 0 and s.dim() == 0 and e.is_cuda
        out.append(torch.stack([e, s]))
    out = torch.stack(out).cpu().numpy()
    np.testing.assert_allclose(out[:, 0], gt[f"{name}/{tag}_est"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(out[:, 1], gt[f"{name}/{tag}_ess"], rtol=1e-12, atol=0)


def _lg_runs(y, N, R, seed):
    import particles_b200 as pb
    from particles_b200 import kalman, state_space_models as ssm
    model = kalman.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9)
    for r in range(R):
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, store_history=True, seed=seed + r)
        pf.run()
        info = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y[::-1]), N=N, store_history=True, seed=seed + 1000 + r)
        info.run()
        yield pf, info


def test_lineargauss_against_kalman_smoother(gt):
    """Independent device runs: the two-filter estimates of E[X_t | Y] (phi = x) and E[X_{t+1} | Y] (phi = xf)
    within 6 standard errors of the run-to-run spread of the Kalman smoother's means, for ON2 and ON."""
    y = list(gt["lg/data"])
    T, kal = len(y), gt["lg/kalman_mean"]
    scale = 1.0 / np.sqrt(1.0 - 0.9 ** 2)

    def lgam(x):
        z = x / scale
        return -z * z / 2.0 - 0.5 * np.log(2.0 * np.pi) - np.log(scale)
    R = 12
    for method, N in (("on2", 2048), ("on", 100000)):
        rows = []
        for pf, info in _lg_runs(y, N, R, seed=100 if method == "on2" else 200):
            h = pf.hist
            if method == "on2":
                e = [torch.stack([h.two_filter_smoothing(t, info, lambda x, xf: x, lgam),
                                  h.two_filter_smoothing(t, info, lambda x, xf: xf, lgam)]) for t in range(T - 1)]
            else:
                e = [h.two_filter_smoothing(t, info, lambda x, xf: torch.stack([x, xf], 1), lgam, linear_cost=True)
                     for t in range(T - 1)]
            rows.append(torch.stack(e))
        est = torch.stack(rows).cpu().numpy()              # (R, T-1, 2)
        truth = np.stack([kal[:-1], kal[1:]], 1)
        se = est.std(axis=0, ddof=1) / np.sqrt(R)
        z = (est.mean(axis=0) - truth) / se
        assert np.max(np.abs(z)) < 6.0, (method, np.max(np.abs(z)))


def test_worker_methods_agree_on_the_book_model():
    """The book's DiscreteCox: smoothing_worker's two-filter estimates of the score agree with FFBS_ON2 within
    their MC spread, under utils.multiplexer as the book script calls it."""
    from particles_b200 import state_space_models as ssm, utils
    from particles_b200.smoothing import smoothing_worker

    class DiscreteCox_with_add_f(ssm.DiscreteCox):
        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi * self.sigma ** 2)
    model = DiscreteCox_with_add_f(mu=MU, phi=PHI, sigma=SIGMA)
    np.random.seed(5)
    _, y = orc.DiscreteCox(mu=MU, sigma=SIGMA, phi=PHI).simulate(50)
    y = [np.atleast_1d(v) for v in y]
    fk = ssm.Bootstrap(ssm=model, data=y)
    fk_info = ssm.Bootstrap(ssm=model, data=y[::-1])
    methods = ["FFBS_ON2", "two-filter_ON2", "two-filter_ON", "two-filter_ON_prop"]
    np.random.seed(7)
    res = utils.multiplexer(f=smoothing_worker, method=methods, N=[1000], fk=fk, fk_info=fk_info,
                            add_func=psit, log_gamma=log_gamma_cox, nprocs=0, nruns=8)
    tot = {m: np.array([r["est"].sum() for r in res if r["method"] == m]) for m in methods}
    for r in res:
        assert r["est"].shape == (49,) and np.all(np.isfinite(r["est"])) and r["cpu"] > 0
    ref = tot["FFBS_ON2"]
    for m in methods[1:]:
        se = np.sqrt(tot[m].var(ddof=1) / len(tot[m]) + ref.var(ddof=1) / len(ref))
        assert abs(tot[m].mean() - ref.mean()) < 6.0 * se, (m, tot[m].mean(), ref.mean(), se)
    with pytest.raises(NotImplementedError, match="SQMC"):
        smoothing_worker(method="FFBS_QMC", N=100, fk=fk, add_func=psit, log_gamma=log_gamma_cox)


def _device_pair(N, T=12, seed=3):
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    np.random.seed(seed)
    _, y = orc.DiscreteCox(mu=MU, sigma=SIGMA, phi=PHI).simulate(T)
    y = [np.atleast_1d(v) for v in y]
    model = ssm.DiscreteCox(mu=MU, phi=PHI, sigma=SIGMA)
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, store_history=True, seed=seed)
    pf.run()
    info = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y[::-1]), N=N, store_history=True, seed=seed + 1)
    info.run()
    return pf.hist, info


def test_on2_at_8192_against_host_replay():
    """One t at N = 8192 (6.7e7 pairs) against a float64 NumPy replay of the row decomposition on the device's own
    histories."""
    h, info = _device_pair(8192)
    t = 5
    ti = h.T - 2 - t
    dev = float(h.two_filter_smoothing(t, info, lambda x, xf: psit(t, x, xf), log_gamma_cox).item())
    X, lw = h.X[t].cpu().numpy(), h.wgts[t].lw.cpu().numpy()
    Xi, lwi = info.hist.X[ti].cpu().numpy(), info.hist.wgts[ti].lw.cpu().numpy()
    host = otf.on2_rows(t, X, lw, Xi, lwi - log_gamma_cox(Xi), osm.px_logpt(oracle_model("cox")),
                        lambda x, xf: psit(t, x, xf), chunk=512)
    assert abs(dev - host) <= 1e-10 * max(1.0, abs(host)), (dev, host)


def test_edge_cases():
    from particles_b200 import collectors
    h, info = _device_pair(300, T=8, seed=11)
    phi = lambda x, xf: x * xf           # noqa: E731
    for t in (-1, h.T - 1):
        with pytest.raises(ValueError, match="range"):
            h.two_filter_smoothing(t, info, phi, log_gamma_cox)
    short, _ = _device_pair(300, T=6, seed=12)
    with pytest.raises(ValueError, match="same"):
        h.two_filter_smoothing(0, types.SimpleNamespace(hist=short), phi, log_gamma_cox)
    with pytest.raises(ValueError, match="store_history"):
        h.two_filter_smoothing(0, types.SimpleNamespace(hist=None), phi, log_gamma_cox)
    other, oinfo = _device_pair(257, T=8, seed=13)
    with pytest.raises(ValueError, match="same N"):
        h.two_filter_smoothing(2, oinfo, phi, log_gamma_cox, linear_cost=True)
    with pytest.raises(ValueError, match="one value per pair"):
        h.two_filter_smoothing(2, info, lambda x, xf: torch.stack([x, xf], 1), log_gamma_cox)
    # ON2 with Ninfo != N: against the host replay
    t, ti = 3, h.T - 2 - 3
    e = float(h.two_filter_smoothing(t, oinfo, phi, log_gamma_cox).item())
    Xi = oinfo.hist.X[ti].cpu().numpy()
    ref = otf.on2_rows(t, h.X[t].cpu().numpy(), h.wgts[t].lw.cpu().numpy(), Xi,
                       oinfo.hist.wgts[ti].lw.cpu().numpy() - log_gamma_cox(Xi), osm.px_logpt(oracle_model("cox")),
                       lambda x, xf: x * xf)
    assert abs(e - ref) <= 1e-11 * max(1.0, abs(ref))
    # one row block and many row blocks give the same estimate
    one = h.two_filter_smoothing(t, info, phi, log_gamma_cox)
    saved = collectors._ON2_PAIRS
    try:
        collectors._ON2_PAIRS = 300 * 7
        many = h.two_filter_smoothing(t, info, phi, log_gamma_cox)
    finally:
        collectors._ON2_PAIRS = saved
    assert abs(float(one) - float(many)) <= 1e-13 * max(1.0, abs(float(one)))
    # same seed -> identical bits; another seed -> other draws
    a = h.two_filter_smoothing(t, info, phi, log_gamma_cox, linear_cost=True, return_ess=True, seed=4)
    b = h.two_filter_smoothing(t, info, phi, log_gamma_cox, linear_cost=True, return_ess=True, seed=4)
    c = h.two_filter_smoothing(t, info, phi, log_gamma_cox, linear_cost=True, return_ess=True, seed=5)
    assert torch.equal(torch.stack(a), torch.stack(b)) and not torch.equal(torch.stack(a), torch.stack(c))
    # no positive pair weight anywhere: NaN, as the reference's 0 / 0; on both paths
    from particles_b200 import resampling as rs, state_space_models as ssm
    from particles_b200.smoothing import ParticleHistory
    for plugin in (False, True):
        fk = ssm.Bootstrap(ssm=stock_model("cox", plugin), data=h.fk.data)
        z = ParticleHistory(fk, False)
        z.X, z.A = list(h.X), list(h.A)
        z.wgts = [rs.Weights._from_device_stats(torch.full_like(w.lw, -np.inf), w._stats) for w in h.wgts]
        assert torch.isnan(z.two_filter_smoothing(t, info, phi, log_gamma_cox))
        # one information particle with no positive pair weight contributes exactly 0
        zi = ParticleHistory(fk, False)
        zi.X, zi.A, zi.wgts = list(info.hist.X), list(info.hist.A), list(info.hist.wgts)
        zi.X[ti] = info.hist.X[ti].clone()
        zi.X[ti][7] = np.inf
        flat = lambda x: torch.zeros_like(x)      # noqa: E731
        with_dead = float(_with_fk(h, fk).two_filter_smoothing(t, types.SimpleNamespace(hist=zi), phi, flat))
        Xi = info.hist.X[ti].cpu().numpy()
        keep = np.arange(Xi.shape[0]) != 7
        ref = otf.on2_rows(t, h.X[t].cpu().numpy(), h.wgts[t].lw.cpu().numpy(), Xi[keep],
                           info.hist.wgts[ti].lw.cpu().numpy()[keep], osm.px_logpt(oracle_model("cox")),
                           lambda x, xf: x * xf)
        assert abs(with_dead - ref) <= 1e-11 * max(1.0, abs(ref)), (plugin, with_dead, ref)
    # vector phi in ON: a (k,) estimate
    v = h.two_filter_smoothing(t, info, lambda x, xf: torch.stack([x, xf, x * xf], 1), log_gamma_cox,
                               linear_cost=True, seed=9)
    s = h.two_filter_smoothing(t, info, phi, log_gamma_cox, linear_cost=True, seed=9)
    assert tuple(v.shape) == (3,) and abs(float(v[2]) - float(s)) <= 1e-12 * max(1.0, abs(float(s)))


def _with_fk(h, fk):
    from particles_b200.smoothing import ParticleHistory
    g = ParticleHistory(fk, False)
    g.X, g.A, g.wgts = h.X, h.A, h.wgts
    return g
