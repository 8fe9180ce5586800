"""The Kalman filter and smoother on the H100: ``kalman.Kalman`` (csrc/smcb_kalman.cu) against the live reference's
fixture (tests/golden/golden_kalman.npz), against the replay (tests/kalman_replay.py) at both tiers and their edges
with batches wider than one wave, batch rows against the same model alone, stepping against one launch, the PMMH
grid and chain of the host tests run as one batched call, the torch step functions, and the edges of the surface.

Tolerances, as max |device - reference| over max |reference| per field and model: 1e-12 against the fixture and
against the long-double replay.  On the host the replay's own fp64 run (the device's roundings) is within 1.5e-14
of long double on the fixture's cases (tests/test_kalman_host.py) and within 5e-15 on the random models below."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kalman_replay as rp  # noqa: E402

CASES = "abcdefgh"
PARAMS = ("F", "G", "covX", "covY", "mu0", "cov0")
FIELDS = ("pred_mean", "pred_cov", "filt_mean", "filt_cov", "logpyt", "smth_mean", "smth_cov")
TOL = 1e-12


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_kalman.npz"))


def host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def rel(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(a - ref)) / max(np.max(np.abs(ref)), np.finfo(float).tiny))


def fields(kf):
    out = {"logpyt": kf.logpyt}
    for k in ("pred", "filt", "smth"):
        s = getattr(kf, k)
        out[k + "_mean"], out[k + "_cov"] = s.mean, s.cov
    return out


class _Model:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def fixture_model(g, c):
    return _Model(**{k: g[c + "_" + k] for k in PARAMS})


def random_batch(rng, B, dx, dy):
    """B stable, well-conditioned models (non-symmetric F, cov0 != covX, non-zero mu0)."""
    A = rng.normal(size=(B, dx, dx))
    F = 0.9 * A / np.max(np.abs(np.linalg.eigvals(A)), axis=1)[:, None, None]

    def spd(d, s):
        M = rng.normal(size=(B, d, d))
        return s * (M @ np.swapaxes(M, 1, 2) / d + np.eye(d))

    return dict(F=F, G=rng.normal(size=(B, dy, dx)) / np.sqrt(dx), covX=spd(dx, 0.5), covY=spd(dy, 0.3),
                mu0=rng.normal(size=(B, dx)), cov0=spd(dx, 2.0))


# ------------------------------------------------------------------------------------------------------------------
# 1. against the reference's fixture
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES)
def test_against_fixture(g, c):
    from particles_b200 import kalman
    y = g[c + "_y"]
    T, dx = y.shape[0], g[c + "_F"].shape[0]
    kf = kalman.Kalman(ssm=fixture_model(g, c), data=list(y))
    kf.smoother()
    assert kf.t == T and len(kf.filt) == T and kf.smth.mean.shape == (T, dx) and kf.pred.cov.shape == (T, dx, dx)
    assert kf.logpyt.is_cuda and kf.logpyt.shape == (T,)
    for k, v in fields(kf).items():
        assert rel(host(v), g[c + "_" + k]) <= TOL, k
    assert torch.equal(kf.filt[-1].mean, kf.filt.mean[T - 1]) and torch.equal(kf.pred[0].cov, kf.pred.cov[0])


def test_stock_models_against_fixture(g):
    from particles_b200 import kalman
    for c, m in (("a", kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9)),
                 ("d", kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=4))):
        kf = kalman.Kalman(ssm=m, data=g[c + "_y"])
        kf.smoother()
        for k, v in fields(kf).items():
            assert rel(host(v), g[c + "_" + k]) <= TOL, (c, k)


def test_incremental_smoothing_of_fixture(g):
    from particles_b200 import kalman
    kf = kalman.Kalman(ssm=fixture_model(g, "a"), data=list(g["a_y"]))
    means, covs = [], []
    for _ in range(10):
        kf.next()
        kf.smoother()
        means.append(host(kf.smth.mean))
        covs.append(host(kf.smth.cov))
    assert rel(np.concatenate(means), g["a_smth_steps_mean"]) <= TOL
    assert rel(np.concatenate(covs), g["a_smth_steps_cov"]) <= TOL


# ------------------------------------------------------------------------------------------------------------------
# 2. both tiers against the replay, 1000 models per batch (more than one wave)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dx,dy", [(1, 1), (2, 2), (31, 31), (32, 32), (32, 1), (1, 32)])
def test_against_replay(dx, dy):
    from particles_b200 import kalman
    B = 1000
    T = 24 if max(dx, dy) <= 2 else 6
    rng = np.random.RandomState(100 * dx + dy)
    p = random_batch(rng, B, dx, dy)
    y = rng.normal(size=(B, T, dy))
    kf = kalman.Kalman(ssm=kalman.MVLinearGauss(**p), data=y)
    kf.smoother()
    dev = {k: host(v) for k, v in fields(kf).items()}
    sel = np.r_[0:B:10, B - 1]                        # the replay is slow in long double: 101 rows of the batch
    sub = {k: v[sel] for k, v in p.items()}
    ld = rp.run(*(sub[k] for k in PARAMS), y[sel])
    f64 = rp.run(*(sub[k] for k in PARAMS), y[sel], dtype=np.float64)
    for k in FIELDS:
        for i, b in enumerate(sel):
            assert rel(dev[k][b], ld[k][i].astype(np.float64)) <= TOL, (k, b)
        if k != "logpyt":                            # the device's roundings: bit for bit but for log()
            assert np.array_equal(dev[k][sel], f64[k]), k
    np.testing.assert_allclose(dev["logpyt"][sel], f64["logpyt"], rtol=1e-14, atol=1e-13)


# ------------------------------------------------------------------------------------------------------------------
# 3. batch rows, shared inputs, stepping
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dx,dy", [(1, 1), (3, 2)])
def test_batch_row_is_the_model_alone(dx, dy):
    from particles_b200 import kalman
    B, T = 37, 20
    rng = np.random.RandomState(7)
    p = random_batch(rng, B, dx, dy)
    y = rng.normal(size=(B, T, dy))
    kf = kalman.Kalman(ssm=kalman.MVLinearGauss(**p), data=y)
    kf.smoother()
    full = fields(kf)
    for b in (0, 5, B - 1):
        one = kalman.Kalman(ssm=_Model(**{k: v[b] for k, v in p.items()}), data=y[b])
        one.smoother()
        for k, v in fields(one).items():
            assert torch.equal(v, full[k][b]), (b, k)
    # shared parameters and data give the bits of the same values repeated per row
    shared = {k: v[0] for k, v in p.items()}
    kf_s = kalman.Kalman(ssm=_Model(**{**shared, "F": p["F"]}), data=y[0])
    kf_r = kalman.Kalman(ssm=kalman.MVLinearGauss(**{k: np.repeat(v[:1], B, 0) if k != "F" else v
                                                     for k, v in p.items()}), data=np.repeat(y[:1], B, 0))
    kf_s.smoother()
    kf_r.smoother()
    for k, v in fields(kf_s).items():
        assert torch.equal(v, fields(kf_r)[k]), k


def test_next_equals_filter_and_appending_continues(g):
    from particles_b200 import kalman
    m = fixture_model(g, "e")
    y = g["e_y"]
    full = kalman.Kalman(ssm=m, data=y)
    full.filter()
    step = kalman.Kalman(ssm=m, data=y)
    for _ in step:
        pass
    with pytest.raises(StopIteration):
        step.next()
    for k in ("pred", "filt"):
        assert torch.equal(getattr(step, k).mean, getattr(full, k).mean) and torch.equal(
            getattr(step, k).cov, getattr(full, k).cov), k
    assert torch.equal(step.logpyt, full.logpyt)
    data = [torch.tensor(r, device="cuda") for r in y[:17]]
    grow = kalman.Kalman(ssm=m, data=data)
    grow.filter()
    data.extend(torch.tensor(r, device="cuda") for r in y[17:40])
    grow.next()
    grow.filter()
    data.extend(list(y[40:]))
    grow.filter()
    assert grow.t == y.shape[0]
    assert torch.equal(grow.filt.cov, full.filt.cov) and torch.equal(grow.logpyt, full.logpyt)
    grow.smoother()
    full.smoother()
    assert torch.equal(grow.smth.mean, full.smth.mean) and torch.equal(grow.smth.cov, full.smth.cov)


# ------------------------------------------------------------------------------------------------------------------
# 4. the exact-likelihood use cases: the PMMH grid and an exact PMMH chain
# ------------------------------------------------------------------------------------------------------------------
def test_pmmh_grid_in_one_call():
    """test_gpu_pmcmc.test_pmmh_posterior's 4000-point rho grid: one batched call against the host loop."""
    from oracle.smc_numpy import LinearGauss as OLG
    from particles_b200 import kalman
    T = 50
    r = np.random.RandomState(2)
    x = np.empty(T)
    x[0] = OLG(rho=0.7, sigmaX=1.0, sigmaY=0.2).sigma0 * r.standard_normal()
    for t in range(1, T):
        x[t] = 0.7 * x[t - 1] + r.standard_normal()
    y = x + 0.2 * r.standard_normal(T)
    grid = np.linspace(-1, 1, 4002)[1:-1]
    ll_host = np.array([OLG(rho=v, sigmaX=1.0, sigmaY=0.2).kalman_loglik(y).sum() for v in grid])
    kf = kalman.Kalman(ssm=kalman.LinearGauss(rho=grid, sigmaX=1.0, sigmaY=0.2), data=y)
    kf.filter()
    assert kf.logpyt.shape == (grid.size, T)
    np.testing.assert_allclose(host(kf.logpyt.sum(1)), ll_host, rtol=1e-12, atol=0)


def test_exact_pmmh_reproduces_the_reference_chain():
    """A PMMH whose loglik is one batched Kalman call: the reference's chain of golden_pmcmc.npz (exact-Kalman
    stub, np.random.seed(4)) with its draws injected -- theta and nacc exactly, lpost to 1e-12."""
    from particles_b200 import distributions as dists, kalman, mcmc
    G = np.load(os.path.join(ROOT, "tests", "golden", "golden_pmcmc.npz"))
    YP = G["pmmh_y"]

    class DeviceKalmanPMMH(mcmc.PMMH):
        def loglik(self, theta):
            if theta.shape[0] == 0:
                return np.empty(0)
            kf = kalman.Kalman(ssm=kalman.LinearGauss(rho=np.asarray(theta["rho"], float)), data=YP)
            kf.filter()
            return host(kf.logpyt.sum(-1)).reshape(-1)

    prior = dists.StructDist({"rho": dists.Uniform(a=-1.0, b=1.0)})
    for tag, adaptive in (("ad", True), ("na", False)):
        z, u = G["pmmh_%s_z" % tag], G["pmmh_%s_u" % tag]
        th0 = np.array([(0.2,)], dtype=[("rho", float)])
        p = DeviceKalmanPMMH(niter=z.shape[0], ssm_cls=kalman.LinearGauss, prior=prior, data=YP, theta0=th0,
                             adaptive=adaptive, rw_cov=np.array([[0.3 ** 2]]),
                             noise={"z": z[:, None, :], "u": u[:, None]})
        p.run()
        assert np.array_equal(p.chain.theta["rho"], G["pmmh_%s_theta" % tag]), tag
        assert p.nacc == int(G["pmmh_%s_nacc" % tag]), tag
        np.testing.assert_allclose(p.chain.lpost, G["pmmh_%s_lpost" % tag], rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------------------------
# 5. step functions
# ------------------------------------------------------------------------------------------------------------------
def test_step_functions_match_the_oracle(g):
    import kalman_oracle as ko
    from particles_b200 import kalman
    for c in ("c", "e", "f"):
        m = fixture_model(g, c)
        y = g[c + "_y"]
        pred, filt, lp = ko.kalman_filter(m, list(y))
        sm, sc = ko.kalman_smoother(m, list(y))
        f = None
        for t in range(y.shape[0]):
            p = kalman.MeanAndCov(mean=m.mu0, cov=m.cov0) if t == 0 else kalman.predict_step(m.F, m.covX, f)
            f, lpt = kalman.filter_step(m.G, m.covY, p, y[t])
            assert rel(host(p.cov), pred[t][1]) <= TOL and rel(host(f.mean), filt[t][0]) <= TOL, (c, t)
            assert abs(float(host(lpt).reshape(-1)[0]) - lp[t]) <= TOL * abs(lp[t]), (c, t)
        T = y.shape[0]
        s = kalman.MeanAndCov(mean=filt[-1][0], cov=filt[-1][1])
        for t in range(T - 2, -1, -1):
            s = kalman.smoother_step(m.F, kalman.MeanAndCov(*filt[t]), kalman.MeanAndCov(*pred[t + 1]), s)
            assert rel(host(s.mean), sm[t]) <= TOL and rel(host(s.cov), sc[t]) <= TOL, (c, t)
    # N predictive means at once (the particle-filter use of the reference)
    m = fixture_model(g, "e")
    xs = np.random.RandomState(1).normal(size=(6, 5))
    f, lpt = kalman.filter_step_asarray(m.G, m.covY, kalman.MeanAndCov(mean=xs, cov=m.covX), g["e_y"][0])
    assert f.mean.shape == (6, 5) and lpt.shape == (6,)
    for n in range(6):
        _, fl, ll = ko.kalman_filter(_Model(**{**{k: getattr(m, k) for k in PARAMS}, "mu0": xs[n], "cov0": m.covX}),
                                     [g["e_y"][0]])
        assert rel(host(f.mean[n]), fl[0][0]) <= TOL and abs(float(lpt[n]) - ll[0]) <= TOL * abs(ll[0])


# ------------------------------------------------------------------------------------------------------------------
# 6. edges
# ------------------------------------------------------------------------------------------------------------------
def test_empty_data_and_one_row(g):
    from particles_b200 import kalman
    kf = kalman.Kalman(ssm=fixture_model(g, "e"), data=[])
    kf.filter()
    assert kf.t == 0 and kf.logpyt.shape == (0,) and kf.filt.mean.shape == (0, 5)
    with pytest.raises(StopIteration):
        next(kf)
    with pytest.raises(IndexError):
        kf.smoother()
    kf = kalman.Kalman(ssm=fixture_model(g, "h"), data=g["h_y"])
    kf.smoother()
    assert kf.t == 1 and torch.equal(kf.smth.cov, kf.filt.cov)
    for k, v in fields(kf).items():
        assert rel(host(v), g["h_" + k]) <= TOL, k


def test_non_positive_definite_covY_is_nan_from_that_step():
    from particles_b200 import kalman
    covY = np.array([1.0, -10.0, 1.0])[:, None, None]       # model 1: S = P + covY < 0 at every step
    m = kalman.MVLinearGauss(F=np.ones((1, 1)) * 0.5, G=np.ones((1, 1)), covX=np.ones((1, 1)), covY=covY)
    y = np.linspace(-1.0, 1.0, 8)
    kf = kalman.Kalman(ssm=m, data=y)
    kf.smoother()
    out = fields(kf)
    assert torch.isnan(out["logpyt"][1]).all() and torch.isnan(out["filt_mean"][1]).all()
    assert torch.isnan(out["smth_cov"][1]).all() and torch.isfinite(out["pred_cov"][1, 0]).all()
    for b in (0, 2):
        assert all(torch.isfinite(v[b]).all() for v in out.values()), b
    # warp tier, dy = 2: covY indefinite only for model 1; that model's rows become NaN, its neighbours do not
    covY = np.stack([np.eye(2), np.array([[1.0, 3.0], [3.0, 1.0]]), np.eye(2)])
    m = kalman.MVLinearGauss(covX=np.eye(2), covY=covY)
    kf = kalman.Kalman(ssm=m, data=np.zeros((5, 2)))
    kf.filter()
    assert torch.isnan(kf.filt.mean[1]).all() and torch.isnan(kf.logpyt[1]).all()
    assert torch.isfinite(kf.filt.cov[0]).all() and torch.isfinite(kf.filt.cov[2]).all()


def test_reference_model_object_and_wrong_data(g):
    from particles_b200 import kalman
    m = fixture_model(g, "f")
    with pytest.raises(ValueError):
        kalman.Kalman(ssm=m, data=np.zeros((4, 3))).filter()            # rows of 3 values where dy = 7
