"""Particle MCMC pieces that need no device: the combinations the samplers refuse, PMMH's host logic against the live
reference's chain (tests/golden/golden_pmcmc.npz), the oracle CSMC against the reference's history and trajectories,
the host build of the pinned weight against the oracle's logG, and the Gibbs update order."""
import ctypes as C
import os

import numpy as np
import pytest
from oracle import pmcmc_numpy as pmo
from oracle.smc_numpy import LinearGauss as OLG
from particles_b200 import _lib, bank, distributions as dists, kalman, mcmc, state_space_models as ssm

HERE = os.path.dirname(os.path.abspath(__file__))


PRIOR = dists.StructDist({"rho": dists.Uniform(a=-1.0, b=1.0)})
Y = np.random.RandomState(0).standard_normal(20)


def _pmmh(**kw):
    args = dict(niter=5, ssm_cls=kalman.LinearGauss, prior=PRIOR, data=Y, Nx=50,
                noise={"z": np.zeros((5, 1, 1)), "u": np.ones((5, 1))})
    args.update(kw)
    return mcmc.PMMH(**args)


def test_unsupported_combinations_raise():
    class Mine(ssm.StochVol):
        pass

    class SMC:                    # not this package's or the reference's SMC
        pass

    with pytest.raises(NotImplementedError):
        _pmmh(ssm_cls=Mine)
    with pytest.raises(NotImplementedError):
        _pmmh(ssm_cls=ssm.BearingsOnly)
    with pytest.raises(NotImplementedError):
        _pmmh(fk_cls=ssm.AuxiliaryPF)
    with pytest.raises(NotImplementedError):
        _pmmh(ssm_cls=ssm.Gordon_etal, prior=dists.StructDist({"a": dists.Uniform(a=0.0, b=1.0)}),
              fk_cls=ssm.GuidedPF)
    with pytest.raises(NotImplementedError):
        _pmmh(smc_options={"resampling": "residual"})
    with pytest.raises(NotImplementedError):
        _pmmh(smc_options={"qmc": True})
    with pytest.raises(NotImplementedError):
        _pmmh(smc_cls=SMC)
    for cls in (ssm.BearingsOnly, Mine):
        with pytest.raises(NotImplementedError):
            mcmc.ParticleGibbs(ssm_cls=cls, prior=PRIOR, data=Y)
    with pytest.raises(NotImplementedError):
        mcmc.ParticleGibbs(ssm_cls=kalman.LinearGauss, prior=PRIOR, data=Y, fk_cls=ssm.AuxiliaryBootstrap)
    with pytest.raises(NotImplementedError, match="regenerate_data"):
        mcmc.ParticleGibbs(ssm_cls=ssm.DiscreteCox, prior=dists.StructDist({"mu": dists.Normal()}),
                           data=np.ones(5), regenerate_data=True)
    _pmmh()                       # the supported case constructs without a device


G = np.load(os.path.join(HERE, "golden", "golden_pmcmc.npz"))
YP = G["pmmh_y"]


class _KalmanPMMH(mcmc.PMMH):
    def loglik(self, theta):
        return np.array([OLG(rho=float(r)).kalman_loglik(YP).sum() for r in theta["rho"]])


def _logpost(r):
    lp = PRIOR.logpdf(np.array([(r[0],)], dtype=[("rho", float)]))[0]
    return lp + OLG(rho=r[0]).kalman_loglik(YP).sum() if np.isfinite(lp) else lp


@pytest.mark.parametrize("tag,adaptive", [("ad", True), ("na", False)])
def test_pmmh_reproduces_the_reference_chain(tag, adaptive):
    """The reference's PMMH (smc_cls = exact Kalman stub) after np.random.seed(4): the product with the same draws
    injected, and the oracle's replay, give its chain bit for bit."""
    z, u = G["pmmh_%s_z" % tag], G["pmmh_%s_u" % tag]
    niter = z.shape[0]
    rw_cov = np.array([[0.3 ** 2]])
    th0 = np.array([(0.2,)], dtype=[("rho", float)])
    p = _KalmanPMMH(niter=niter, ssm_cls=kalman.LinearGauss, prior=PRIOR, data=YP, theta0=th0, adaptive=adaptive,
                    rw_cov=rw_cov, noise={"z": z[:, None, :], "u": u[:, None]})
    p.run()
    assert np.array_equal(p.chain.theta["rho"], G["pmmh_%s_theta" % tag])
    assert np.array_equal(p.chain.lpost, G["pmmh_%s_lpost" % tag])
    assert p.nacc == int(G["pmmh_%s_nacc" % tag])
    arr, lp, nacc = pmo.rwhm(_logpost, np.array([0.2]), z, u, adaptive=adaptive, rw_cov=rw_cov)
    assert np.array_equal(arr[:, 0], G["pmmh_%s_theta" % tag]) and np.array_equal(lp, G["pmmh_%s_lpost" % tag])
    assert nacc == int(G["pmmh_%s_nacc" % tag])


@pytest.mark.parametrize("adaptive", [False, True])
def test_pmmh_chains_are_independent_replays(adaptive):
    """K chains: each is the one-chain algorithm on its own draws; layout (niter, K)."""
    niter, K = 60, 3
    r = np.random.RandomState(5)
    z, u = r.standard_normal((niter, K, 1)), r.rand(niter, K)
    rw_cov = np.array([[0.3 ** 2]])
    th0 = np.array([(0.2,)], dtype=[("rho", float)])
    p = _KalmanPMMH(niter=niter, ssm_cls=kalman.LinearGauss, prior=PRIOR, data=YP, theta0=th0, adaptive=adaptive,
                    rw_cov=rw_cov, nchains=K, noise={"z": z, "u": u})
    p.run()
    assert p.chain.theta.shape == (niter, K)
    for k in range(K):
        arr, lp, nacc = pmo.rwhm(_logpost, np.array([0.2]), z[:, k], u[:, k], adaptive=adaptive, rw_cov=rw_cov)
        assert np.array_equal(p.chain.theta["rho"][:, k], arr[:, 0])
        assert np.array_equal(p.chain.lpost[:, k], lp)
        assert p.nacc[k] == nacc


@pytest.mark.parametrize("name", ["sv", "lg"])
def test_oracle_csmc_reproduces_the_reference(name):
    """The oracle CSMC replaying the global stream: the reference's history, logLt and both trajectories."""
    from oracle import smc_numpy as orc
    from oracle.smoothing_numpy import px_logpt
    model = orc.StochVol() if name == "sv" else orc.LinearGauss()
    y = G[name + "_y"]
    np.random.seed(3)
    c = pmo.CSMC(orc.Bootstrap(model, y), N=50, xstar=G[name + "_xstar"]).run()
    h = c.hist
    assert np.array_equal(np.array(h["X"]), G[name + "_X"])
    assert np.array_equal(np.array(h["A"][1:]), G[name + "_A"])
    assert np.array_equal(np.array(h["lw"]), G[name + "_lw"])
    assert c.logLt == float(G[name + "_logLt"])
    assert np.array_equal(np.array(pmo.extract_one_trajectory(h)), G[name + "_traj"])
    idx, _ = pmo.backward_ON2(h, px_logpt(model), 1)
    assert np.array_equal(np.array([h["X"][t][idx[t, 0]] for t in range(len(y))]), G[name + "_bwd"])


_fk_lib = None


def _fk_host():
    global _fk_lib
    if _fk_lib is None:
        import subprocess
        root = os.path.join(HERE, "..")
        out = os.path.join(root, "oracle", "_build")
        os.makedirs(out, exist_ok=True)
        so = os.path.join(out, "libpmcmc_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(root, "particles_b200", "csrc"), "-I", os.path.join(root, "include"),
                               os.path.join(HERE, "pmcmc_host.cpp"), "-o", so])
        _fk_lib = C.CDLL(so)
        _fk_lib.mh_init()
    return _fk_lib


_MODELS = {"StochVol": ssm.StochVol, "StochVolLeverage": ssm.StochVolLeverage, "LinearGauss": kalman.LinearGauss,
           "Gordon_etal": ssm.Gordon_etal, "ThetaLogistic": ssm.ThetaLogistic, "DiscreteCox": ssm.DiscreteCox}
BUILT = [(n, k) for n, (_, _, prop, _) in bank._MAPS.items()
         for k in ([_lib.FK_BOOTSTRAP, _lib.FK_GUIDED] if prop else [_lib.FK_BOOTSTRAP])]


@pytest.mark.parametrize("name,kind", BUILT)
def test_pinned_weight_matches_oracle_logG(name, kind):
    """fk_logG0 / fk_logG (the pinned particle's weight) at given states against the oracle's Bootstrap / GuidedPF
    logG, every (model, kind) the conditional filter builds; t = 0 and t > 0."""
    from oracle import smc_numpy as orc
    T, n = 12, 64
    r = np.random.RandomState(17)
    data = r.poisson(2.0, T).astype(float) if name == "DiscreteCox" else r.standard_normal(T)
    m = bank.ThetaMap(_MODELS[name], [], data)
    params = np.ascontiguousarray(m.params(np.empty((1, 0)))[0])
    sc = m.step_consts(np.empty((1, 0)))
    sc = m.shared_sc if sc is None else np.ascontiguousarray(sc[0])
    cols = {k: float(v[0]) for k, v in m.columns(np.empty((1, 0))).items()}
    model = getattr(orc, name)(**cols)
    fk = (orc.GuidedPF if kind == _lib.FK_GUIDED else orc.Bootstrap)(model, data)
    lib = _fk_host()
    P = C.c_void_p
    for t in (0, 1, 5, T - 1):
        xp, x = r.standard_normal(n), r.standard_normal(n)
        out = np.empty(n)
        rc = lib.mh_fk_logG(m.model, kind, params.ctypes.data_as(P), data.ctypes.data_as(P), C.c_long(T),
                            None if sc is None else sc.ctypes.data_as(P), C.c_long(t), xp.ctypes.data_as(P),
                            x.ctypes.data_as(P), C.c_long(n), out.ctypes.data_as(P))
        assert rc == 0
        ref = fk.logG(t, None if t == 0 else xp, x)
        np.testing.assert_allclose(out, ref, rtol=1e-13, atol=1e-13)


def test_gibbs_draws_states_given_the_new_theta():
    """GenericGibbs calls update_states with theta_n (the oracle's corrected loop), not theta_{n-1}."""
    seen = []

    class Stub(mcmc.GenericGibbs):
        def update_theta(self, theta, x):
            new = theta.copy()
            new["rho"] = theta["rho"] + 1.0
            return new

        def update_states(self, n):
            th = float(self.chain.theta["rho"][n])
            seen.append(th)
            return np.full((1, 3), th)

    g = Stub(niter=5, prior=PRIOR, data=np.zeros(3), theta0=np.array([(0.0,)], dtype=[("rho", float)]))
    g.run()
    theta, x = pmo.gibbs(0.0, 5, lambda th, x: th + 1.0, lambda th, x: np.full(3, th))
    assert seen == theta
    assert np.array_equal(g.chain.theta["rho"], np.array(theta))


def test_vanish_cov_tracker():
    r = np.random.RandomState(1)
    tr = mcmc.VanishCovTracker(dim=2, Sigma0=np.eye(2) * 0.5)
    mu, S = np.zeros(2), np.eye(2) * 0.5
    for t in range(1, 50):
        v = r.standard_normal(2)
        tr.update(v)
        g = (t + 1) ** (-0.6)
        mu = (1 - g) * mu + g * v
        S = (1 - g) * S + g * np.outer(v - mu, v - mu)
        assert np.array_equal(tr.mu, mu) and np.allclose(tr.Sigma, S, rtol=1e-15, atol=0)
    np.testing.assert_allclose(tr.L @ tr.L.T, tr.Sigma, rtol=1e-12)


def test_msjd():
    th = np.zeros(4, dtype=[("a", float), ("b", float)])
    th["a"], th["b"] = [0, 1, 3, 3], [0, 0, 1, 1]
    assert mcmc.msjd(th) == 1 + 4 + 0 + 1
