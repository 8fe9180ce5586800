"""Particle MCMC on the device (particles_b200.mcmc, csrc/smcb_pmcmc.cu): the conditional filter against the filter
bank and a NumPy replay, and the samplers against exact answers."""
import numpy as np
import pytest
import torch
from scipy import stats

pytestmark = pytest.mark.gpu

from particles_b200 import _lib, mcmc                                      # noqa: E402
from particles_b200 import distributions as dists                          # noqa: E402
from particles_b200 import kalman, state_space_models as ssm               # noqa: E402
from particles_b200.bank import FilterBank, ThetaMap, _MAPS                 # noqa: E402
from particles_b200.device import as_device                                 # noqa: E402
from particles_b200.smc_samplers import _KeyCounter                         # noqa: E402


def _data(name, T, seed=0):
    r = np.random.RandomState(seed)
    if name == "DiscreteCox":
        return r.poisson(2.0, T).astype(np.float64)
    return r.standard_normal(T)


def _built():
    out = []
    for name, (_, _, proposal, _) in _MAPS.items():
        out.append((name, _lib.FK_BOOTSTRAP))
        if proposal:
            out.append((name, _lib.FK_GUIDED))
    return out


BUILT = _built()


def _tmap(name, T, seed=0):
    # a stand-in class with the stock model's name and module: the model's default parameters
    cls = type(name, (), {"__module__": "particles_b200.state_space_models"})
    return ThetaMap(cls, [], _data(name, T, seed))


def _runs(tmap, kind, N, R, draw="genealogy", essrmin=0.5, seed=7):
    runs = mcmc._CsmcRuns(tmap, kind, N, R, essrmin, draw)
    runs.set_rows(np.empty((R, 0)), _KeyCounter(seed))
    return runs


@pytest.mark.parametrize("name,kind", BUILT)
def test_pin_off_is_the_bank(name, kind):
    """The unconditional pass gives the bits of FilterBank.advance with the same keys, multinomial resampling."""
    N, T, R = 301, 40, 5
    m = _tmap(name, T)
    runs = _runs(m, kind, N, R, essrmin=0.8)
    summ = torch.zeros((R, T, 4), dtype=torch.float64, device="cuda")
    runs.run(pin=False, summaries=summ)
    bank = FilterBank(m.model, kind, "multinomial", N, R, as_device(m.data), m.n_params, 0.8,
                      shared_sc=None if m.shared_sc is None else as_device(m.shared_sc),
                      per_filter_sc=m.name == "Gordon_etal")
    bank.params.copy_(runs.params)
    bank.key.copy_(runs.key)
    if bank.sc is not None:
        bank.sc.copy_(runs.sc)
    bsumm = torch.zeros_like(summ)
    A = torch.full((R, bank.ld), -1, dtype=torch.int64, device="cuda")
    bank.advance(T, restart=True, summaries=bsumm, A=A)
    assert torch.equal(summ, bsumm)
    assert torch.equal(runs.logLt, bank.logLt)
    last = (T - 1) & 1
    assert torch.equal(runs.X[:, T - 1, :N], bank.X[:, last, :N])
    assert torch.equal(runs.lw[:, T - 1, :N], bank.lw[:, :N])
    rs_last = summ[:, T - 1, 2].cpu().numpy() > 0
    assert summ[:, :, 2].sum() > 0
    for r in np.flatnonzero(rs_last):
        assert torch.equal(runs.A[r, T - 1, :N], A[r, :N])


# ---------------------------------------------------------------------------------------------- oracle CSMC
@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("name,kind", BUILT)
def test_pin_on_matches_oracle(name, kind, backward):
    """8 chains against the oracle CSMC (corrected pinned weight) with injected noise: the pinned path bitwise, the
    ancestors of >= 99 % of (chain, t) rows, and on the chains whose ancestors all agree, logLt to 1e-12 and the
    drawn trajectory: the same particle index at every t, and the device's own particle there bit for bit."""
    from oracle import pmcmc_numpy as pmo, smc_numpy as orc
    from oracle.smoothing_numpy import px_logpt
    N, T, R, essrmin = 100, 30, 8, 0.7
    m = _tmap(name, T, seed=3)
    runs = _runs(m, kind, N, R, "backward" if backward else "genealogy", essrmin)
    r = np.random.RandomState(11)
    z, u, ud = r.standard_normal((R, T, N)), r.rand(R, T, N + 1), r.rand(R, T)
    xstar = np.empty((R, T))
    cols = {k: float(v[0]) for k, v in m.columns(np.empty((1, 0))).items()}
    model = getattr(orc, name)(**cols)
    fk = (orc.GuidedPF if kind == _lib.FK_GUIDED else orc.Bootstrap)(model, m.data)
    for c in range(R):                                   # reference paths: unconditional oracle runs
        h = pmo.CSMC(fk, N=N, ESSrmin=essrmin, noise=orc.InjectedNoise(z[(c + 1) % R], u[(c + 1) % R])).run().hist
        xstar[c] = pmo.draw_trajectory(h, None, ud[(c + 1) % R], False)[0]
    runs.xstar.copy_(torch.from_numpy(xstar))
    noise = {"z": as_device(z), "u": as_device(u), "ud": as_device(ud)}
    runs.run(pin=True, noise=noise)
    X, A = runs.X[:, :, :N].cpu().numpy(), runs.A[:, :, :N].cpu().numpy()
    traj_d, logLt_d = runs.traj.cpu().numpy(), runs.logLt.cpu().numpy()
    assert np.array_equal(X[:, :, 0], xstar)
    assert (A[:, 1:, 0] == 0).all()
    rows = agree = 0
    for c in range(R):
        o = pmo.CSMC(fk, N=N, ESSrmin=essrmin, xstar=xstar[c], noise=orc.InjectedNoise(z[c], u[c])).run()
        h = o.hist
        ok = (A[c] == np.array(h["A"])).all(axis=1)
        rows += ok.sum()
        if ok.all():
            agree += 1
            np.testing.assert_allclose(logLt_d[c], o.logLt, rtol=1e-12)
            traj, idx = pmo.draw_trajectory(h, px_logpt(model), ud[c], backward)
            assert np.array_equal(traj_d[c], X[c][np.arange(T), idx])
            np.testing.assert_allclose(traj_d[c], traj, rtol=1e-12, atol=1e-12)
    assert rows >= 0.99 * R * T
    assert agree >= R // 2


def test_csmc_surface():
    T, N = 25, 200
    y = [np.atleast_1d(v) for v in _data("LinearGauss", T, 5)]
    fk = ssm.Bootstrap(ssm=kalman.LinearGauss(rho=0.9, sigmaX=1.0, sigmaY=0.5), data=y)
    c0 = mcmc.CSMC(fk=fk, N=N, seed=3)
    c0.run()
    xstar = c0.hist.extract_one_trajectory()
    assert len(xstar) == T
    c1 = mcmc.CSMC(fk=fk, N=N, xstar=[float(v) for v in xstar], seed=4)
    c1.run()
    assert np.array_equal(torch.stack(c1.hist.X)[:, 0].cpu().numpy(), np.array([float(v) for v in xstar]))
    paths = c1.hist.backward_sampling_ON2(1)
    assert len(paths) == T
    # the same run through the kernel's own entry point gives the same logLt
    runs = mcmc._CsmcRuns(c1._map, c1._kind, N, 1, 0.5, "genealogy")
    runs.set_rows(c1._row, _KeyCounter(4))
    runs.xstar[0] = as_device(np.array([float(v) for v in xstar]))
    runs.run(pin=True)
    assert runs.logLt[0].item() == c1.logLt
    assert np.isfinite(c1.logLt)


# ---------------------------------------------------------------------------------------------- samplers
class _FixedTheta(mcmc.ParticleGibbs):
    def update_theta(self, theta, x):
        return theta


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("fk", ["Bootstrap", "GuidedPF"])
def test_particle_gibbs_leaves_the_smoother_invariant(fk, backward):
    """theta fixed: the Gibbs chain in x targets the smoothing distribution, known exactly (Kalman smoother)."""
    from oracle.smoothing_numpy import kalman_smoother
    T, K = 40, 4096
    th = dict(rho=0.9, sigmaX=1.0, sigmaY=0.5)
    model = kalman.LinearGauss(**th)
    _, y = model.simulate(T)
    y = np.array([float(v.reshape(-1)[0]) for v in y])
    prior = dists.StructDist({k: dists.Normal(loc=v) for k, v in th.items()})
    theta0 = np.array([tuple(th.values())], dtype=[(k, float) for k in th])
    pg = _FixedTheta(niter=50, ssm_cls=kalman.LinearGauss, prior=prior, data=y, theta0=theta0, Nx=128,
                     fk_cls=getattr(ssm, fk), backward_step=backward, nchains=K, seed=1)
    pg.run()
    x = pg.x
    mean, cov = kalman_smoother(model, y)
    mean, var = mean[:, 0], cov[:, 0, 0]
    zs = (x.mean(axis=0) - mean) / np.sqrt(var / K)
    assert np.abs(zs).max() < 5, zs
    assert np.abs(zs).mean() < 1.5
    ratio = x.var(axis=0) / var
    assert np.abs(ratio - 1).max() < 5 * np.sqrt(2 / K), ratio


def test_pmmh_posterior():
    """rho of LinearGauss under a Uniform(-1, 1) prior: posterior mean and sd against a 4000-point Kalman grid."""
    from oracle.smc_numpy import LinearGauss as OLG
    T, K, niter, burn = 50, 256, 2000, 500
    truth = OLG(rho=0.7, sigmaX=1.0, sigmaY=0.2)         # sigmaY: the class default, which PMMH keeps
    r = np.random.RandomState(2)
    x = np.empty(T)
    x[0] = truth.sigma0 * r.standard_normal()
    for t in range(1, T):
        x[t] = 0.7 * x[t - 1] + r.standard_normal()
    y = x + 0.2 * r.standard_normal(T)
    grid = np.linspace(-1, 1, 4002)[1:-1]
    ll = np.array([OLG(rho=g, sigmaX=1.0, sigmaY=0.2).kalman_loglik(y).sum() for g in grid])
    w = np.exp(ll - ll.max())
    w /= w.sum()
    pm = (w * grid).sum()
    psd = np.sqrt((w * (grid - pm) ** 2).sum())
    prior = dists.StructDist({"rho": dists.Uniform(a=-1.0, b=1.0)})
    th0 = np.array([(0.5,)], dtype=[("rho", float)])
    pmmh = mcmc.PMMH(niter=niter, ssm_cls=kalman.LinearGauss, prior=prior, data=y, Nx=200, theta0=th0,
                     adaptive=False, rw_cov=np.array([[0.15 ** 2]]), nchains=K, seed=5,
                     smc_options={"resampling": "systematic"})
    pmmh.run()
    rho = pmmh.chain.theta["rho"][burn:]                    # (niter - burn, K)
    cm, csd = rho.mean(axis=0), rho.std(axis=0)
    assert abs(cm.mean() - pm) < 4 * cm.std() / np.sqrt(K), (cm.mean(), pm)
    assert abs(csd.mean() - psd) < 4 * csd.std() / np.sqrt(K), (csd.mean(), psd)
    assert 0.05 < pmmh.acc_rate.mean() < 0.9


SIG0_PG = 2.0


class _PGStochVol(mcmc.ParticleGibbs):
    """Conjugate update of mu given x, rho and sigma fixed (the model of the PGStochVol example)."""

    def update_theta(self, theta, x):
        new = theta.copy()
        rho, sigma = theta["rho"], theta["sigma"]
        x = np.array(x)
        xlag = np.array([0.0] + list(x[:-1]))
        sig0 = sigma / np.sqrt(1 - rho ** 2)
        prec = 1 / SIG0_PG ** 2 + 1 / sig0 ** 2 + (len(x) - 1) * (1 - rho) ** 2 / sigma ** 2
        num = x[0] / sig0 ** 2 + ((1 - rho) * (x[1:] - rho * xlag[1:])).sum() / sigma ** 2
        new["mu"] = stats.norm.rvs(loc=num / prec, scale=1 / np.sqrt(prec))
        return new


def _pg_prior(rho=0.9, sigma=0.5):
    return dists.StructDist({"mu": dists.Normal(scale=SIG0_PG), "rho": dists.Dirac(rho),
                             "sigma": dists.Dirac(sigma)})


def test_particle_gibbs_recovers_the_prior():
    """Geweke: with the data re-simulated every iteration, (mu, x) follow the joint prior."""
    T, K, niter = 30, 512, 300
    np.random.seed(3)
    y = np.random.standard_normal(T)
    pg = _PGStochVol(niter=niter, ssm_cls=ssm.StochVol, prior=_pg_prior(), data=y, Nx=100,
                     regenerate_data=True, nchains=K, seed=9)
    pg.run()
    mu = pg.chain.theta["mu"][-1]
    assert stats.kstest(mu, stats.norm(scale=SIG0_PG).cdf).pvalue > 1e-3
    assert abs(mu.mean()) < 4 * SIG0_PG / np.sqrt(K)
    assert abs(mu.var() - SIG0_PG ** 2) < 4 * SIG0_PG ** 2 * np.sqrt(2 / (K - 1))
    jm = mu * pg.x.mean(axis=1)
    # direct simulation of prior and model: E[mu mean_t x_t]
    r = np.random.RandomState(4)
    S = 200000
    mus = SIG0_PG * r.standard_normal(S)
    rho, sigma = 0.9, 0.5
    xs = mus + sigma / np.sqrt(1 - rho ** 2) * r.standard_normal(S)
    acc = xs.copy()
    for t in range(1, T):
        xs = mus + rho * (xs - mus) + sigma * r.standard_normal(S)
        acc += xs
    ref = mus * acc / T
    se = np.sqrt(jm.var() / K + ref.var() / S)
    assert abs(jm.mean() - ref.mean()) < 4 * se, (jm.mean(), ref.mean(), se)


def test_seeds_fix_both_samplers():
    T, K = 20, 6
    y = _data("LinearGauss", T, 1)
    prior = dists.StructDist({"rho": dists.Uniform(a=-1.0, b=1.0)})

    def pmmh():
        p = mcmc.PMMH(niter=30, ssm_cls=kalman.LinearGauss, prior=prior, data=y, Nx=64, nchains=K, seed=21)
        p.run()
        return p.chain.theta["rho"].copy(), p.chain.lpost.copy()

    a, b = pmmh(), pmmh()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert len({tuple(c) for c in a[0].T}) == K

    def pg():
        np.random.seed(0)
        p = _PGStochVol(niter=20, ssm_cls=ssm.StochVol, prior=_pg_prior(), data=y, Nx=64, nchains=K, seed=22,
                        store_x=True)
        p.run()
        return p.chain.theta["mu"].copy(), p.chain.x.copy()

    a, b = pg(), pg()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert len({tuple(c) for c in a[0].T}) == K


def test_nx_above_the_bound_is_not_implemented():
    m = _tmap("StochVol", 10)
    with pytest.raises(NotImplementedError):
        mcmc._CsmcRuns(m, _lib.FK_BOOTSTRAP, 20000, 2, 0.5, "genealogy")
