"""SQMC on the device (csrc/smcb_sqmc.cu): Sobol' points and Hilbert keys against the host build, per-step replay of
the resampling of ``SMC(qmc=True)``, and the variance reduction SQMC is for."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch
from scipy.special import ndtri
from scipy.stats import qmc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_sqmc_host as hh  # noqa: E402

import particles_b200 as pb  # noqa: E402
from particles_b200 import hilbert, kalman, rqmc  # noqa: E402
from particles_b200 import state_space_models as ssm  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d,n", [(1, 1), (3, 1000), (5, 4099), (32, 70000)])
def test_device_sobol_equals_host(d, n):
    for scramble in (True, False):
        u, raw = rqmc.sobol_points(n, d, seed=2026, call=7, scramble=scramble, raw=True)
        hu, hraw = hh.host_sobol(d, n, scramble=scramble, seed=2026, call=7)
        assert np.array_equal(raw.cpu().numpy(), hraw)
        assert np.array_equal(u.cpu().numpy(), hu)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = qmc.Sobol(d, scramble=False).random(n)
    assert np.array_equal(raw.cpu().numpy().T * 2.0 ** -30, ref)
    s = rqmc.sobol(64, 3)
    assert s.shape == (64, 3) and s.is_cuda and float(s.min()) > 0 and float(s.max()) < 1
    with pytest.raises(NotImplementedError):
        rqmc.halton(8, 2)


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("n", [100, 4096, 2 ** 20 + 3])
def test_device_hilbert_equals_host(d, n):
    rng = np.random.default_rng(d * 7 + n)
    x = rng.standard_normal((n, d)) * rng.uniform(0.5, 3.0, size=d)
    xt = torch.from_numpy(np.ascontiguousarray(x.T)).cuda()
    if d == 1:
        order = hilbert.hilbert_order(xt[0]).cpu().numpy()
        assert np.array_equal(x[order, 0], np.sort(x[:, 0]))
        return
    order, keys = hilbert.hilbert_order(xt, keys=True)
    order, keys = order.cpu().numpy(), keys.cpu().numpy()
    xs = 1.0 / (1.0 + np.exp(-((x - x.mean(0)) / x.std(0)))) * np.floor(2 ** (62 / d))
    # device mean, std and exp may differ from NumPy's in the last bit, which moves xs * maxint by up to a few
    # ulp(xs) * maxint (2.4e-7 at d = 2): compare the points that no such change can move across an integer
    safe = np.all(np.abs(xs - np.round(xs)) > 1e-5, axis=1)
    hk = hh.host_hilbert_keys(np.floor(xs).astype(np.int64))
    assert safe.mean() > 0.99
    assert np.array_equal(keys[safe], hk[safe])
    assert np.array_equal(np.sort(order), np.arange(n))
    assert np.all(np.diff(keys[order]) >= 0)                   # sorted as signed int64
    assert np.array_equal(hilbert.hilbert_sort(torch.from_numpy(x).cuda()).cpu().numpy(), order)


def _models():
    lg = kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9)
    return {"lg": lg, "sv": ssm.StochVol(), "gordon": ssm.Gordon_etal(),
            "bearings": ssm.BearingsOnly(), "mv2": kalman.MVLinearGauss_Guarniero_etal(dx=2),
            "mv3": kalman.MVLinearGauss_Guarniero_etal(dx=3)}


KINDS = {"boot": ssm.Bootstrap, "guided": ssm.GuidedPF, "apf": ssm.AuxiliaryPF, "auxboot": ssm.AuxiliaryBootstrap}
CASES = [(m, k) for m in ("lg", "sv", "mv2", "mv3") for k in KINDS] + [("gordon", "boot"), ("bearings", "boot")]


def _data(model, T, seed):
    torch.manual_seed(seed)
    np.random.seed(seed)
    _, y = model.simulate(T)
    return [v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v) for v in y]


@pytest.mark.parametrize("name,kind", CASES)
@pytest.mark.parametrize("N", [100, 4096, 2 ** 16 + 1, 2 ** 20])
def test_per_step_replay(name, kind, N):
    """From the filter's own X_{t-1}, W_{t-1} (bootstrap and guided kinds) and the step's regenerated points, the
    ancestors are A = h[searchsorted(cumsum(W[h]), sort(u[:, 0]))]; every row says rs_flag = 1 and its logLt is the
    running sum of the log-mean weights."""
    model = _models()[name]
    T = 20
    y = _data(model, T, 11)
    fk = KINDS[kind](ssm=model, data=y)
    pf = pb.SMC(fk=fk, N=N, qmc=True, seed=4242, collect="off")
    assert pf.fused
    e = pf._engine
    dim = e.dim
    lm = []
    prev = None
    for t in range(T):
        next(pf)
        lw = e.lw[t & 1].cpu().numpy().astype(np.longdouble)
        m = lw.max()
        lm.append(float(m + np.log(np.mean(np.exp(lw - m)))))
        if prev is not None and kind in ("boot", "guided"):
            Xp, lwp = prev
            u, raw = rqmc.sobol_points(N, dim + 1, seed=4242, call=t, raw=True)
            raw0 = raw[0].cpu().numpy()
            su = hh.squeeze(np.sort(raw0).astype(np.float64) * 2.0 ** -30)
            h = hilbert.hilbert_order(torch.from_numpy(Xp).cuda()).cpu().numpy()
            W = np.exp(lwp - lwp.max())
            W = W / W.sum()
            cdf = np.cumsum(W[h])
            idx = np.minimum(np.searchsorted(cdf, su, side="left"), N - 1)
            A = e.A.cpu().numpy()
            near = np.abs(su[:, None] - cdf[np.clip(idx[:, None] + np.array([-1, 0]), 0, N - 1)]).min(1) < 1e-12
            assert np.array_equal(A[~near], h[idx][~near]), (name, kind, N, t)
            if name == "lg" and kind == "boot":
                tau = np.argsort(raw0, kind="stable")
                v = u[1].cpu().numpy()[tau]
                X = e.X[t & 1].cpu().numpy()
                ref = model.rho * Xp[A] + model.sigmaX * ndtri(v)
                np.testing.assert_allclose(X, ref, rtol=0, atol=1e-13 * (1 + np.abs(ref)).max())
        prev = (e.X[t & 1].cpu().numpy().copy(), e.lw[t & 1].cpu().numpy().copy())
    table = e.summ.cpu().numpy()
    assert np.all(table[1:, 2] == 1) and table[0, 2] == 0
    np.testing.assert_allclose(table[:, 3], lm, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(table[:, 1], np.cumsum(lm), rtol=1e-11, atol=1e-10)
    assert pf.h_order.shape == (N,)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_sqmc.npz")
REF_MODELS = {0: lambda: ssm.StochVol(), 1: lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
              2: lambda: ssm.Gordon_etal(), 3: lambda: ssm.BearingsOnly(),
              4: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=2), 5: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=3)}
REF_KINDS = {0: ssm.Bootstrap, 1: ssm.GuidedPF, 2: ssm.AuxiliaryPF, 3: ssm.AuxiliaryBootstrap}


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", range(16))
def test_reference_runs(case, fused):
    """The reference's SQMC (particles.SMC(qmc=True)) recorded on fixed point sets: fed the same points, the device
    filter -- fused engine and plugin path alike -- reproduces its ancestors and Hilbert orders exactly and its
    particles, weights and logLt to 1e-12 at every step."""
    g = np.load(GOLDEN)
    mc, kc, N, T = (int(v) for v in g[f"run_{case}_meta"])
    y = [row for row in g[f"run_{case}_y"]]
    fk = REF_KINDS[kc](ssm=REF_MODELS[mc](), data=y)
    pts = [g[f"run_{case}_u{t}"] for t in range(T)]
    pf = pb.SMC(fk=fk, N=N, qmc=True, noise=pts, fused=None if fused else False, collect="off")
    assert pf.fused == fused
    for t in range(T):
        next(pf)
        X = pf.X.cpu().numpy().reshape(g[f"run_{case}_X{t}"].shape)
        np.testing.assert_allclose(X, g[f"run_{case}_X{t}"], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(pf.W.cpu().numpy(), g[f"run_{case}_W{t}"], rtol=1e-11, atol=1e-14)
        assert abs(pf.logLt - g[f"run_{case}_logLt"][t]) <= 1e-12 * max(1.0, abs(pf.logLt))
        if t > 0:
            assert np.array_equal(pf.A.cpu().numpy(), g[f"run_{case}_A{t}"]), t
            assert np.array_equal(pf.h_order.cpu().numpy(), g[f"run_{case}_h{t}"]), t


def _lg_exact(model, y):
    """Exact log-likelihood of a scalar LinearGauss model (Kalman filter in NumPy)."""
    m, P, ll = 0.0, model.sigma0 ** 2, 0.0
    for t, yt in enumerate(y):
        if t > 0:
            m, P = model.rho * m, model.rho ** 2 * P + model.sigmaX ** 2
        yt = float(np.asarray(yt.cpu() if torch.is_tensor(yt) else yt).reshape(-1)[0])
        S = P + model.sigmaY ** 2
        ll += -0.5 * np.log(2 * np.pi * S) - 0.5 * (yt - m) ** 2 / S
        K = P / S
        m, P = m + K * (yt - m), (1 - K) * P
    return ll


def _logLts(fk, N, R, qmc_):
    out = []
    for r in range(R):
        pf = pb.SMC(fk=fk, N=N, qmc=qmc_, seed=1000 + r, collect="off")
        pf.run()
        out.append(pf.logLt)
    return np.array(out)


@pytest.mark.parametrize("name,kind", [("lg", "boot"), ("lg", "guided"), ("sv", "boot"), ("sv", "guided")])
def test_variance_reduction(name, kind):
    model = _models()[name]
    y = _data(model, 100, 5)
    fk = KINDS[kind](ssm=model, data=y)
    q = _logLts(fk, 1024, 64, True)
    s = _logLts(fk, 1024, 64, False)
    assert np.all(np.isfinite(q))
    assert q.var() / s.var() < 0.25, (q.var(), s.var())
    if name == "lg":
        exact = _lg_exact(model, y)
        assert abs(q.mean() + q.var() / 2 - exact) < 3 * q.std() / np.sqrt(len(q)), (q.mean(), exact, q.std())


@pytest.mark.parametrize("dx,fused,T", [(2, True, 100), (5, False, 30)])
def test_mv_kalman(dx, fused, T):
    """MVLinearGauss_Guarniero_etal: dx = 2 on the fused engine, dx = 5 on the plugin path (the book's
    sqmc_as_dim_grows workload); the mean logLt of R = 64 SQMC runs lies within 3 sigma of the Kalman log-likelihood."""
    model = kalman.MVLinearGauss_Guarniero_etal(dx=dx)
    y = _data(model, T, 8)
    kf = kalman.Kalman(ssm=model, data=y)
    kf.filter()
    exact = float(torch.as_tensor(kf.logpyt).sum())
    fk = ssm.Bootstrap(ssm=model, data=y)
    q = []
    for r in range(64):
        pf = pb.SMC(fk=fk, N=1024, qmc=True, seed=500 + r, fused=None if fused else False, collect="off")
        pf.run()
        assert pf.fused == fused
        q.append(pf.logLt)
    q = np.array(q)
    # the filter estimates the likelihood without bias, so its log sits var / 2 below on average (Jensen; logLt is
    # close to Gaussian): compare mean + var / 2 with the Kalman value, within 3 sigma of the mean of R runs
    assert abs(q.mean() + q.var() / 2 - exact) < 3 * q.std() / np.sqrt(len(q)), (q.mean(), exact, q.std())


@pytest.mark.parametrize("case", [0, 1, 4, 11, 12])
def test_fused_and_plugin_ancestors_agree(case):
    """fused=False on a stock model gives the fused SQMC's ancestors for the same (Sobol' key) points."""
    g = np.load(GOLDEN)
    mc, kc, N, T = (int(v) for v in g[f"run_{case}_meta"])
    y = [row for row in g[f"run_{case}_y"]]
    fk = REF_KINDS[kc](ssm=REF_MODELS[mc](), data=y)
    a = pb.SMC(fk=fk, N=4096, qmc=True, seed=77, collect="off")
    b = pb.SMC(fk=fk, N=4096, qmc=True, seed=77, fused=False, collect="off")
    assert a.fused and not b.fused
    for t in range(T):
        next(a)
        next(b)
        if t > 0:
            assert np.array_equal(a.A.cpu().numpy(), b.A.cpu().numpy()), t
        np.testing.assert_allclose(a.X.cpu().numpy(), b.X.cpu().numpy(), rtol=1e-12, atol=1e-12)
    assert abs(a.logLt - b.logLt) < 1e-10 * abs(a.logLt)


def test_ppf_matches_scipy():
    from scipy import stats
    from particles_b200 import distributions as dists
    rng = np.random.default_rng(4)
    u = hh.squeeze(rng.random((1000, 3)))
    loc, scale = rng.standard_normal(1000), rng.uniform(0.5, 2.0, 1000)
    got = dists.Normal(loc=torch.from_numpy(loc).cuda(), scale=torch.from_numpy(scale).cuda()).ppf(u[:, 0])
    ref = stats.norm.ppf(u[:, 0], loc=loc, scale=scale)
    np.testing.assert_allclose(got.cpu().numpy(), ref, rtol=1e-14, atol=1e-14)
    cov = np.array([[2.0, 0.3, 0.1], [0.3, 1.0, 0.2], [0.1, 0.2, 0.5]])
    mv = dists.MvNormal(loc=np.array([1.0, -1.0, 0.5]), cov=cov)
    L = np.linalg.cholesky(cov)
    mv_ref = np.array([1.0, -1.0, 0.5]) + stats.norm.ppf(u) @ L.T
    np.testing.assert_allclose(mv.ppf(u).cpu().numpy(), mv_ref, rtol=1e-13, atol=1e-13)
    z2 = np.zeros((1000, 3))
    z2[:, :2] = stats.norm.ppf(u[:, :2])                  # fewer columns than dim: zero-filled (Rosenblatt)
    np.testing.assert_allclose(mv.ppf(u[:, :2]).cpu().numpy(), np.array([1.0, -1.0, 0.5]) + z2 @ L.T,
                               rtol=1e-13, atol=1e-13)
    ip = dists.IndepProd(dists.Normal(loc=2.0, scale=3.0), dists.Dirac(loc=5.0))
    out = ip.ppf(u[:, :2]).cpu().numpy()
    np.testing.assert_allclose(out[:, 0], stats.norm.ppf(u[:, 0], loc=2.0, scale=3.0), rtol=1e-14, atol=1e-14)
    assert np.all(out[:, 1] == 5.0)
    with pytest.raises(NotImplementedError):
        dists.Gamma(a=2.0, b=1.0).ppf(u[:, 0])
    assert mv_ref.shape == (1000, 3)


def test_surface():
    model = _models()["sv"]
    y = _data(model, 30, 3)
    fk = ssm.Bootstrap(ssm=model, data=y)
    pf = pb.SMC(fk=fk, N=500, qmc=True, store_history=True, collect=[pb.collectors.Moments()], seed=9)
    pf.run()
    assert len(pf.summaries.moments) == 30 and len(pf.summaries.logLts) == 30
    assert all(pf.summaries.rs_flags[1:])
    traj = pf.hist.extract_one_trajectory()
    assert len(traj) == 30
    a = pb.SMC(fk=fk, N=500, qmc=True, seed=9)
    a.run()
    assert a.logLt == pf.logLt                      # the points of a run are a function of its seed
    out = pb.multiSMC(fk=fk, N=256, qmc={"smc": False, "sqmc": True}, nruns=2)
    assert len(out) == 4 and {o["qmc"] for o in out} == {"smc", "sqmc"}
    assert all(np.isfinite(o["output"].logLt) for o in out)

    b = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=500, qmc=True, fused=False, seed=9)
    b.run()                                               # the plugin path: same points, same filter
    assert not b.fused and abs(b.logLt - a.logLt) < 1e-10 * abs(a.logLt)
    with pytest.raises(NotImplementedError):
        a._engine.step_timed(1)
