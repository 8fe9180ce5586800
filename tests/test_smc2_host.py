"""SMC^2 pieces that need no device: the theta -> model-constant map against the scalar specs, the static-parameter
laws against scipy, and the sampler's host logic (exchange trigger, Nx bookkeeping, waste-free reshape) over a stub
bank."""
import numpy as np
import pytest
from scipy import stats

from particles_b200 import bank, kalman, state_space_models as ssm

MODELS = {
    "StochVol": (ssm.StochVol, ssm.spec_stochvol, {"mu": (-2, 0), "rho": (0.5, 0.99), "sigma": (0.05, 1)}),
    "StochVolLeverage": (ssm.StochVolLeverage, ssm.spec_stochvollev,
                         {"mu": (-2, 0), "rho": (0.5, 0.99), "sigma": (0.05, 1), "phi": (-0.9, 0.9)}),
    "LinearGauss": (kalman.LinearGauss, ssm.spec_lingauss, {"rho": (-0.9, 0.9), "sigmaX": (0.1, 2), "sigmaY": (0.1, 2)}),
    "Gordon_etal": (ssm.Gordon_etal, ssm.spec_gordon, {"a": (0.01, 0.1), "b": (0.2, 0.8), "d": (1, 10), "e": (0.5, 2)}),
    "ThetaLogistic": (ssm.ThetaLogistic, ssm.spec_thetalogistic,
                      {"tau0": (0, 0.3), "tau1": (0, 0.3), "tau2": (0.05, 0.2), "sigmaX": (0.1, 1), "sigmaY": (0.1, 1)}),
    "DiscreteCox": (ssm.DiscreteCox, ssm.spec_discretecox, {"mu": (-1, 1), "sigma": (0.1, 1), "phi": (0.5, 0.99)}),
}


def _ulps(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("partial", [False, True])
def test_theta_map_matches_scalar_specs(name, partial):
    """Row i of the vectorised map equals spec_*(ssm_cls(**theta_i)) to 1 ulp: NumPy's array loops for log / cos may
    round differently from its scalar path by one ulp, nothing else differs (the same expressions).  With
    ``partial`` the rows name only the first parameter and the others take the class's defaults."""
    cls, spec, ranges = MODELS[name]
    names = list(ranges)[:1] if partial else list(ranges)
    rng = np.random.RandomState(7)
    n, T = 64, 30
    theta = np.stack([rng.uniform(*ranges[k], size=n) for k in names], axis=1)
    data = rng.poisson(2.0, size=T).astype(float)
    m = bank.ThetaMap(cls, names, data)
    P = m.params(theta)
    SC = m.step_consts(theta)
    assert P.shape == (n, m.n_params)
    worst = 0.0
    for i in range(n):
        obj = cls(**{k: theta[i, j] for j, k in enumerate(names)})
        ref = spec(obj, T, list(data)) if spec is ssm.spec_discretecox else spec(obj, T)
        worst = max(worst, _ulps(P[i], np.asarray(ref["params"], dtype=np.float64)).max())
        if SC is not None:
            worst = max(worst, _ulps(SC[i], ref["step_consts"]).max())
        elif spec is ssm.spec_discretecox:
            assert np.array_equal(m.shared_sc, ref["step_consts"])
    assert worst <= 1.0, worst


def test_theta_map_rejects_other_models():
    class Mine(ssm.StochVol):
        pass

    for cls in (Mine, ssm.BearingsOnly, kalman.MVLinearGauss):
        with pytest.raises(NotImplementedError, match="StochVol, StochVolLeverage"):
            bank.ThetaMap(cls, ["sigma"], np.zeros(5))


def test_static_laws_vs_scipy():
    from particles_b200 import distributions as dists
    x = np.linspace(-1.5, 1.5, 301)
    u = dists.Uniform(a=-1.0, b=1.0)
    ref = stats.uniform.logpdf(x, loc=-1.0, scale=2.0)
    assert np.array_equal(np.isfinite(u.logpdf(x)), np.isfinite(ref))
    np.testing.assert_allclose(u.logpdf(x)[np.isfinite(ref)], ref[np.isfinite(ref)], rtol=1e-12)
    xb = np.linspace(1e-6, 1 - 1e-6, 501)
    for a, b in ((9.0, 1.0), (2.0, 3.5), (0.5, 0.5)):
        np.testing.assert_allclose(dists.Beta(a=a, b=b).logpdf(xb), stats.beta.logpdf(xb, a, b), rtol=1e-12)
    assert np.all(dists.Beta(a=2.0, b=2.0).logpdf(np.array([-0.1, 1.1])) == -np.inf)

    class ScipyGamma:                       # a host law with the two methods (the reference's duck type)
        def logpdf(self, v):
            return stats.gamma.logpdf(v, 2.0, scale=0.5)

    prior = dists.StructDist({"rho": dists.Beta(a=9.0, b=1.0), "phi": dists.Uniform(a=-1.0, b=1.0),
                              "sigma": ScipyGamma()})
    assert [k for k, _ in prior.dtype] == ["phi", "rho", "sigma"]
    th = np.zeros(50, dtype=prior.dtype)
    rng = np.random.RandomState(3)
    th["phi"], th["rho"], th["sigma"] = rng.uniform(-1, 1, 50), rng.uniform(0.5, 1, 50), rng.gamma(2.0, 0.5, 50)
    ref = (stats.uniform.logpdf(th["phi"], loc=-1, scale=2) + stats.beta.logpdf(th["rho"], 9.0, 1.0)
           + stats.gamma.logpdf(th["sigma"], 2.0, scale=0.5))
    np.testing.assert_allclose(prior.logpdf(th), ref, rtol=1e-12)


# ---------------------------------------------------------------------------------------------- host logic, stub bank
class StubBank:
    """What SMC2 asks of a FilterBank, on the host: every filter's loglt is -1 per step."""

    def __init__(self, N, R):
        import torch
        self.N, self.R = N, R
        self.state = torch.zeros((R, 8), dtype=torch.float64)
        self.advanced = []

    def advance(self, t1, idx=None, restart=False):
        import torch
        rows = torch.arange(self.R) if idx is None else idx.cpu()
        t0 = torch.zeros(len(rows)) if restart else self.state[rows, 0]
        self.state[rows, 1] = (0.0 if restart else self.state[rows, 1]) - (t1 - t0).double()
        self.state[rows, 7] = -1.0
        self.state[rows, 0] = float(t1)
        self.advanced.append((t1, None if idx is None else len(rows), restart))

    @property
    def logLt(self):
        return self.state[:, 1]

    @property
    def loglt(self):
        return self.state[:, 7]


def _stub_smc2(monkeypatch, **kw):
    import torch
    from particles_b200 import distributions as dists, smc_samplers as ss
    monkeypatch.setattr(ss, "as_device", lambda a, dtype=torch.float64, device=None: torch.as_tensor(
        np.array(a), dtype=dtype))
    fk = ss.SMC2(ssm_cls=ssm.StochVol, prior=dists.StructDist({"rho": dists.Beta(a=9.0, b=1.0)}),
                 data=np.zeros(10), **kw)
    made = []

    def stub(theta_dev, Nx, keys):
        b = StubBank(Nx, theta_dev.shape[0])
        made.append(b)
        return b

    monkeypatch.setattr(fk, "_bank", stub)
    return fk, made


def _particles(fk, n, Nx):
    import torch
    from particles_b200 import smc_samplers as ss
    x = ss.SMC2Particles(shared={"Nxs": [Nx]}, names=["rho"], keys=ss._KeyCounter(0),
                         theta_dev=torch.full((n, 1), 0.9, dtype=torch.float64))
    fk.current_target(-1, Nx)(x)
    return x


def test_exchange_trigger_and_nx_bookkeeping(monkeypatch):
    """The exchange step runs at 2 Nx exactly when the step follows a move whose mean acceptance rate is below
    ar_to_increase_Nx (smc_samplers.py:1101-1108); shared['Nxs'] records Nx at every t > 0; the log-weight
    increment is loglt plus the change of lpost."""
    torch = pytest.importorskip("torch")
    fk, made = _stub_smc2(monkeypatch, ar_to_increase_Nx=0.3, wastefree=False)
    x = _particles(fk, 4, 10)
    assert np.all(x.lpost.numpy() == x.lprior.numpy())
    lw0 = fk.logG(0, None, x)
    assert np.all(lw0.numpy() == -1.0) and x.shared["Nxs"] == [10]
    x.shared["rs_flag"], x.shared["acc_rates"] = True, [[torch.tensor([0.5]), torch.tensor([0.4])]]
    fk.logG(1, None, x)                                     # acceptance 0.45 >= 0.3: no exchange
    assert x.bank.N == 10 and x.shared["Nxs"] == [10, 10]
    x.shared["acc_rates"].append([torch.tensor([0.2]), torch.tensor([0.1])])
    before = x.lpost.clone()
    lw = fk.logG(2, None, x)                                # 0.15 < 0.3: exchange at 20 particles
    assert x.bank.N == 20 and x.shared["Nxs"] == [10, 10, 20]
    assert made[-1].advanced == [(2, 4, True), (3, None, False)]
    # the stub's logLt after re-running steps 0, 1 is -2 (same as before): the increment is loglt = -1
    np.testing.assert_allclose(lw.numpy(), -1.0)
    np.testing.assert_allclose(x.lpost.numpy(), before.numpy() - 1.0)
    x.shared["rs_flag"] = False                             # no move at this step: no exchange whatever the rate
    fk.logG(3, None, x)
    assert x.bank.N == 20


def test_infinite_prior_rows_are_not_run(monkeypatch):
    torch = pytest.importorskip("torch")
    fk, made = _stub_smc2(monkeypatch)
    from particles_b200 import smc_samplers as ss
    x = ss.SMC2Particles(shared={}, names=["rho"], keys=ss._KeyCounter(0),
                         theta_dev=torch.tensor([[0.9], [1.5], [0.8], [-0.2]], dtype=torch.float64))
    fk.current_target(4, 10)(x)
    assert made[-1].advanced == [(5, 2, True)]
    lp = x.lpost.numpy()
    assert np.isfinite(lp[[0, 2]]).all() and np.all(lp[[1, 3]] == -np.inf)


def test_wastefree_sizes():
    from particles_b200 import distributions as dists, smc_samplers as ss
    prior = dists.StructDist({"rho": dists.Beta(a=9.0, b=1.0)})
    wf = ss.SMC2(ssm_cls=ssm.StochVol, prior=prior, data=np.zeros(5), len_chain=6)
    assert isinstance(wf.move, ss.MCMCSequenceWF) and wf.move.nsteps == 5
    assert isinstance(wf.move.mcmc, ss.BankRandomWalk)
    st = ss.SMC2(ssm_cls=ssm.StochVol, prior=prior, data=np.zeros(5), wastefree=False, len_chain=6)
    assert isinstance(st.move, ss.AdaptiveMCMCSequence) and st.move.nsteps == 5
    seen = []
    wf._M0 = lambda n: seen.append(n)
    st._M0 = lambda n: seen.append(n)
    wf.M0(100)
    st.M0(100)
    assert seen == [600, 100]


def test_constructor_checks():
    from particles_b200 import distributions as dists, smc_samplers as ss
    prior = dists.StructDist({"rho": dists.Beta(a=9.0, b=1.0)})
    with pytest.raises(ValueError):
        ss.SMC2(ssm_cls=ssm.StochVol, prior=prior, data=np.zeros(5), smc_options={"data": 1})
    with pytest.raises(NotImplementedError):
        ss.SMC2(ssm_cls=ssm.StochVol, prior=prior, data=np.zeros(5), smc_options={"qmc": True})
    with pytest.raises(NotImplementedError):
        ss.SMC2(ssm_cls=ssm.BearingsOnly, prior=prior, data=np.zeros(5))
    with pytest.raises(NotImplementedError):
        ss.SMC2(ssm_cls=ssm.Gordon_etal, prior=prior, data=np.zeros(5), fk_cls=ssm.GuidedPF)
    fk = ss.SMC2(ssm_cls=ssm.StochVol, prior=prior, data=np.zeros(7), smc_options={"ESSrmin": 0.7,
                                                                                   "resampling": "multinomial"})
    assert fk.T == 7 and fk.ESSrmin_inner == 0.7 and fk.resampling == "multinomial"
    assert fk.smc_options["collect"] == "off"
