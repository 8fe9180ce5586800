"""The laws of csrc/smcb_dists.cu on the device: log-densities against scipy / the host build of the same header
(tests/dists_host.cpp) / the live reference's values (tests/golden/golden_dists.npz), draws against the host
build's replay of the same Philox counters, goodness of fit at N = 10^6, VaryingCovNormal and Dirichlet against
NumPy / scipy, and end-to-end filters and a PMMH chain written with the new laws."""
import os

import numpy as np
import pytest
from scipy import stats
from scipy.special import gammaln, logsumexp

from test_dists_host import (BINOMIAL, DUNIFORM, GAMMA, GEOMETRIC, INVGAMMA, LAPLACE, LOGISTIC, LOGNORMAL,
                             NEGBINOMIAL, NORMAL, STUDENT, TRUNCNORMAL, chi2_p, close, host_dirichlet_rvs, host_logpdf,
                             host_rvs, ks_p, student_c0)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def D():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from particles_b200 import distributions
    return distributions


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "golden_dists.npz"))


def host(t):
    return t.detach().cpu().numpy()


def cuda(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float64), device="cuda")


# name -> (constructor, law code, parameter tuple in the kernel's order, a grid of x)
def cases(D):
    x = np.concatenate([[-1.0, 0.0, np.nan, 1e-3], np.linspace(0.05, 12.0, 60)])
    k = np.array([-1.0, 0.0, 0.5, 1.0, 2.0, 3.0, 5.0, 9.0, 30.0, 31.0, np.nan])
    return {
        "InvGamma": (lambda *p: D.InvGamma(*p), INVGAMMA, (2.5, 1.5), x),
        "LogNormal": (lambda *p: D.LogNormal(*p), LOGNORMAL, (-0.5, 0.8), x),
        "TruncNormal": (lambda *p: D.TruncNormal(*p), TRUNCNORMAL, (0.5, 2.0, -1.0, 4.0), x),
        "TruncNormalTail": (lambda *p: D.TruncNormal(*p), TRUNCNORMAL, (0.0, 1.0, 30.0, np.inf), 30.0 + x / 50),
        "Binomial": (lambda *p: D.Binomial(*p), BINOMIAL, (30.0, 0.35), k),
        "Geometric": (lambda *p: D.Geometric(*p), GEOMETRIC, (0.25,), k),
        "NegativeBinomial": (lambda *p: D.NegativeBinomial(*p), NEGBINOMIAL, (3.5, 0.3), k),
        "DiscreteUniform": (lambda *p: D.DiscreteUniform(*p), DUNIFORM, (-1.0, 7.0), k),
        "Normal": (lambda *p: D.Normal(*p), NORMAL, (0.5, 2.0), x),
        "Student": (lambda df, loc, s, c0: D.Student(df, loc, s), STUDENT, (2.5, 0.5, 2.0, student_c0(2.5)), x),
        "GammaSmallA": (lambda a, b, c0: D.Gamma(a, b), GAMMA, (0.4, 2.0, -gammaln(0.4)), x),
        "GammaExponential": (lambda a, b, c0: D.Gamma(a, b), GAMMA, (1.0, 0.7, -gammaln(1.0)), x),
        "Gamma": (lambda a, b, c0: D.Gamma(a, b), GAMMA, (3.5, 2.0, -gammaln(3.5)), x),
        "Laplace": (lambda *p: D.Laplace(*p), LAPLACE, (0.5, 2.0), x),
        "Logistic": (lambda *p: D.Logistic(*p), LOGISTIC, (0.5, 2.0), x),
    }


def test_logpdf_scalar_and_per_particle(D):
    r = np.random.RandomState(0)
    for name, (make, law, pars, x) in cases(D).items():
        got = host(make(*pars).logpdf(cuda(x)))
        close(got, host_logpdf(law, x, *pars))
        # per-particle parameters: each parameter jittered per element, x one value per particle
        n = 4096
        pp = [np.full(n, p) for p in pars]
        if law in (INVGAMMA, LOGNORMAL):
            pp = [pp[0] * r.uniform(0.5, 1.5, n), pp[1] * r.uniform(0.5, 1.5, n)]
        elif law == TRUNCNORMAL and np.isfinite(pars[3]):
            pp[0] = pp[0] + r.normal(size=n)
        elif law in (BINOMIAL, NEGBINOMIAL, GEOMETRIC):
            pp[-1] = r.uniform(0.05, 0.95, n)
        elif law in (NORMAL, LAPLACE, LOGISTIC):
            pp = [p * r.uniform(0.5, 1.5, n) for p in pp]
        elif law in (STUDENT, GAMMA):            # df, a and the constant c0 stay scalars, as in distributions.py
            pp = [pars[0]] + [p * r.uniform(0.5, 1.5, n) for p in pp[1:-1]] + [pars[-1]]
        xs = r.choice(x[np.isfinite(x)], n)
        got = host(make(*[cuda(p) for p in pp]).logpdf(cuda(xs)))
        close(got, host_logpdf(law, xs, *pp))
    # scipy directly, on per-particle parameters
    n = 2000
    a, b = r.uniform(0.3, 8.0, n), r.uniform(0.2, 3.0, n)
    xs = r.gamma(2.0, 1.0, n)
    close(host(D.InvGamma(cuda(a), cuda(b)).logpdf(cuda(xs))), stats.invgamma.logpdf(xs, a, scale=b))
    nn, p = r.randint(1, 500, n).astype(float), r.rand(n)
    ks = np.floor(r.rand(n) * (nn + 1))
    close(host(D.Binomial(cuda(nn), cuda(p)).logpdf(torch.as_tensor(ks, device="cuda").long())),
          stats.binom.logpmf(ks, nn, p))


def test_rvs_only_for_laws_with_a_sampler(D):
    """Normal, Student, Laplace and Logistic draw outside the law table: smcb_dist_rvs refuses their codes"""
    import ctypes as C
    from particles_b200 import _lib
    from particles_b200.device import context, empty, ptr
    ctx, out, s = context(), empty(8), np.ones(4)
    for law in (NORMAL, STUDENT, LAPLACE, LOGISTIC):
        with pytest.raises(ValueError, match="not a law with a sampler"):
            _lib.check(ctx.lib.smcb_dist_rvs(ctx.handle, law, None, None, None, None, s.ctypes.data_as(C.c_void_p),
                                             ptr(out), 8))


def test_logpdf_against_reference_golden(D, golden):
    mk = {"invgamma": D.InvGamma(a=2.5, b=1.5), "lognormal": D.LogNormal(mu=-0.5, sigma=0.8),
          "truncnormal": D.TruncNormal(mu=0.5, sigma=2.0, a=-1.0, b=4.0),
          "truncnormal_tail": D.TruncNormal(mu=0.0, sigma=1.0, a=8.0, b=np.inf),
          "binomial": D.Binomial(n=30, p=0.35), "geometric": D.Geometric(p=0.25),
          "discreteuniform": D.DiscreteUniform(lo=-1, hi=7),
          "logd_gamma": D.LogD(D.Gamma(a=2.0, b=3.0)),
          "lineard_normal": D.LinearD(D.Normal(loc=1.0), a=2.0, b=-1.0),
          "logitd_beta": D.LogitD(D.Beta(a=2.0, b=3.0), a=-1.0, b=2.0),
          "mixture": D.Mixture([0.3, 0.7], D.Normal(loc=-1.0), D.Normal(loc=2.0, scale=0.5))}
    for name, law in mk.items():
        x, ref = golden[f"logpdf/{name}/x"], golden[f"logpdf/{name}/y"]
        if name == "discreteuniform":          # the reference gives non-integer x the mass; every x here is integer
            assert np.all(x == np.floor(x))
        # tensors (state-space models) and NumPy arrays (priors) alike
        for xin in (cuda(x), x):
            got = law.logpdf(xin)
            got = host(got) if isinstance(got, torch.Tensor) else np.asarray(got)
            close(got, ref, rtol=1e-11, atol=1e-11)
    al = golden["logpdf/dirichlet/alphas"]
    close(host(D.Dirichlet(al).logpdf(cuda(golden["logpdf/dirichlet/x"]))), golden["logpdf/dirichlet/y"])


def test_draws_replay_host_counters(D):
    import particles_b200 as pb
    n = 200_000
    r = np.random.RandomState(1)
    per = {INVGAMMA: (r.uniform(0.2, 5, n), r.uniform(0.1, 3, n)), LOGNORMAL: (r.normal(size=n), r.uniform(0.1, 2, n)),
           TRUNCNORMAL: (r.normal(size=n), r.uniform(0.2, 2, n), r.choice([-np.inf, -1.0, 0.5, 3.0], n),
                         np.full(n, np.inf)),
           BINOMIAL: (r.randint(0, 100, n).astype(float), r.rand(n)), GEOMETRIC: (r.uniform(0.01, 1, n),),
           NEGBINOMIAL: (r.uniform(0.1, 30, n), r.uniform(0.05, 1, n)), DUNIFORM: (np.full(n, -5.0), np.full(n, 9.0)),
           GAMMA: (r.uniform(0.1, 20, n), r.uniform(0.5, 2, n))}
    mk = {INVGAMMA: D.InvGamma, LOGNORMAL: D.LogNormal, TRUNCNORMAL: D.TruncNormal, BINOMIAL: D.Binomial,
          GEOMETRIC: D.Geometric, NEGBINOMIAL: D.NegativeBinomial, DUNIFORM: D.DiscreteUniform}
    seed = 77
    for law, pars in per.items():
        pb.seed(seed)                          # the API call counter restarts at 0
        if law == GAMMA:                       # the sampler under InvGamma / NegativeBinomial / Dirichlet
            from particles_b200 import _lib
            from particles_b200.device import context, empty, ptr
            import ctypes as C
            ctx, out = context(), empty(n)
            s = np.zeros(4)
            ps = [cuda(p) for p in pars]
            _lib.check(ctx.lib.smcb_dist_rvs(ctx.handle, GAMMA, ptr(ps[0]), ptr(ps[1]), None, None,
                                             s.ctypes.data_as(C.c_void_p), ptr(out), n))
            dev = host(out)
        else:
            dev = host(mk[law](*[cuda(p) for p in pars]).rvs())
        ref = host_rvs(law, n, *pars, seed=seed, call=0)
        if law in (BINOMIAL, GEOMETRIC, NEGBINOMIAL, DUNIFORM):
            assert dev.dtype == np.int64
            assert np.mean(dev != ref) <= 1e-5, (law, np.mean(dev != ref))
        else:
            both = np.isfinite(ref)
            assert both.all()
            bad = ~np.isclose(dev, ref, rtol=1e-12, atol=1e-14)
            assert bad.mean() <= 1e-5, (law, dev[bad][:5], ref[bad][:5])


def test_goodness_of_fit_at_1e6(D):
    import particles_b200 as pb
    N = 1_000_000
    pb.seed(11)
    x = host(D.TruncNormal(mu=0.0, sigma=1.0, a=0.0, b=np.inf).rvs(size=N))
    assert ks_p(stats.truncnorm.cdf(x, 0.0, np.inf)) > 1e-4
    x = host(D.InvGamma(a=0.3, b=2.0).rvs(size=N))
    assert ks_p(stats.invgamma.cdf(x, 0.3, scale=2.0)) > 1e-4
    x = host(D.LogNormal(mu=1.0, sigma=0.5).rvs(size=N))
    assert ks_p(stats.lognorm.cdf(x, 0.5, scale=np.e)) > 1e-4
    for n, p in [(20, 0.2), (500, 0.4)]:
        x = host(D.Binomial(n=n, p=p).rvs(size=N))
        assert chi2_p(x, lambda k: stats.binom.pmf(k, n, p), 0) > 1e-4
    x = host(D.NegativeBinomial(n=2.5, p=0.4).rvs(size=N))
    assert chi2_p(x, lambda k: stats.nbinom.pmf(k, 2.5, 0.4), 0) > 1e-4
    a, b = np.random.RandomState(2).uniform(0.5, 5, N), np.random.RandomState(3).uniform(0.5, 2, N)
    x = host(D.InvGamma(a=cuda(a), b=cuda(b)).rvs())
    assert ks_p(stats.invgamma.cdf(x, a, scale=b)) > 1e-4


def test_seed_reproduces_draws(D):
    import particles_b200 as pb
    for law in (D.TruncNormal(0.0, 1.0, 40.0, np.inf), D.Binomial(1000, 0.3), D.NegativeBinomial(2.5, 0.4),
                D.Dirichlet(np.array([0.5, 1.5, 2.0])), D.Mixture([0.5, 0.5], D.InvGamma(), D.LogNormal())):
        pb.seed(5)
        a, b = host(law.rvs(size=10_000)), host(law.rvs(size=10_000))
        pb.seed(5)
        assert np.array_equal(a, host(law.rvs(size=10_000)))
        assert not np.array_equal(a, b)
    pb.seed(5)
    x = host(D.TruncNormal(0.0, 1.0, 40.0, np.inf).rvs(size=100_000))
    assert np.isfinite(x).all() and x.min() >= 40.0 and x.mean() < 40.1


def test_dirichlet(D):
    import particles_b200 as pb
    al = np.array([0.7, 2.0, 3.5])
    d = D.Dirichlet(al)
    x = np.random.RandomState(4).dirichlet(al, size=1000)
    close(host(d.logpdf(cuda(x))), stats.dirichlet.logpdf(x.T, al).T)
    for bad in ([0.5, 0.6, 0.1], [-0.1, 0.6, 0.5], [0.0, 0.5, 0.5]):
        with pytest.raises(ValueError):
            stats.dirichlet.logpdf(np.array(bad), al)
        with pytest.raises(ValueError):
            d.logpdf(cuda(np.vstack([x[:9], bad])))
    pb.seed(9)
    got = host(d.rvs(size=5000))
    np.testing.assert_allclose(got, host_dirichlet_rvs(al, 5000, seed=9, call=0), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("d", [1, 2, 4, 8])
def test_varying_cov_normal(D, d):
    import particles_b200 as pb
    r = np.random.RandomState(d)
    N = 3000
    A = r.normal(size=(N, d, d))
    cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(d)
    loc = r.normal(size=(N, d))
    law = D.VaryingCovNormal(loc=cuda(loc), cov=cuda(cov))
    Lref = np.linalg.cholesky(cov)
    np.testing.assert_allclose(host(law.L), Lref, rtol=1e-12, atol=1e-13)
    x = r.normal(size=(N, d)) * 2
    z = np.linalg.solve(Lref, (x - loc)[..., None])[..., 0]
    ref = -0.5 * np.sum(z * z, 1) - (d * 0.5 * np.log(2 * np.pi) + np.sum(np.log(np.diagonal(Lref, 0, 1, 2)), 1))
    close(host(law.logpdf(cuda(x))), ref, rtol=1e-11, atol=1e-11)
    pb.seed(3)
    draws = host(law.rvs())
    assert draws.shape == (N, d)
    zz = np.linalg.solve(Lref, (draws - loc)[..., None])[..., 0]      # standardised draws: N(0, I)
    assert ks_p(stats.norm.cdf(zz.ravel())) > 1e-4
    # one covariance shared row of loc, and the reference's ValueError for a non-positive-definite cov[n]
    assert host(D.VaryingCovNormal(loc=0.0, cov=cuda(cov)).rvs()).shape == (N, d)
    with pytest.raises(NotImplementedError):
        D.VaryingCovNormal(cov=cuda(np.tile(np.eye(9), (2, 1, 1))))


def test_varying_cov_normal_non_pd_raises(D):
    cov = np.tile(np.eye(3), (100_000, 1, 1))
    cov[71_234, 2, 2] = -1.0
    with pytest.raises(ValueError):
        D.VaryingCovNormal(cov=cuda(cov))


def test_dirichlet_scipy_checks_and_small_alphas(D):
    """scipy's tolerance (|sum - 1| <= 1e-9), its NaN behaviour, and finite draws for alphas near 0"""
    import particles_b200 as pb
    al = np.array([0.7, 2.0, 3.5])
    d = D.Dirichlet(al)
    x = np.random.RandomState(6).dirichlet(al, size=100)
    off = x.copy()
    off[17] *= 1.0 + 1e-6
    with pytest.raises(ValueError):
        stats.dirichlet.logpdf(off.T, al)
    with pytest.raises(ValueError):
        d.logpdf(cuda(off))
    nan = x.copy()
    nan[5, 1] = np.nan
    ref = stats.dirichlet.logpdf(nan.T, al).T
    close(host(d.logpdf(cuda(nan))), ref)
    assert np.isnan(ref[5]) and np.isfinite(np.delete(ref, 5)).all()
    tiny = np.array([1e-3, 1e-3, 2e-3])
    pb.seed(4)
    got = host(D.Dirichlet(tiny).rvs(size=100_000))
    assert np.isfinite(got).all()
    np.testing.assert_allclose(got.sum(1), 1.0, rtol=1e-14)
    np.testing.assert_allclose(got, host_dirichlet_rvs(tiny, 100_000, seed=4, call=0), rtol=1e-12, atol=1e-300)


def test_row_inputs_broadcast_or_raise(D):
    """A (1, d) observation and a (1, d) loc are one row for every particle (StateSpaceModel.simulate gives (1, d)
    observations); row counts other than 1 and N raise ValueError, as NumPy's broadcasting does.  Likewise a (1, k)
    pk of Mixture, and rvs(size) against N per-particle parameters."""
    import particles_b200 as pb
    r = np.random.RandomState(8)
    N, d = 500, 3
    A = r.normal(size=(N, d, d))
    cov = A @ A.transpose(0, 2, 1) + np.eye(d)
    Lref = np.linalg.cholesky(cov)
    y, m = r.normal(size=(1, d)), r.normal(size=(1, d))
    law = D.VaryingCovNormal(loc=cuda(m), cov=cuda(cov))
    z = np.linalg.solve(Lref, (y - m)[..., None])[..., 0]
    ref = -0.5 * np.sum(z * z, 1) - (d * 0.5 * np.log(2 * np.pi) + np.sum(np.log(np.diagonal(Lref, 0, 1, 2)), 1))
    close(host(law.logpdf(cuda(y))), ref, rtol=1e-11, atol=1e-11)
    close(host(law.logpdf(y)), ref, rtol=1e-11, atol=1e-11)
    pb.seed(1)
    assert np.isfinite(host(law.rvs())).all()
    for bad in (r.normal(size=(7, d)), r.normal(size=(N, d + 1)), r.normal(size=d + 1)):
        with pytest.raises(ValueError):
            law.logpdf(cuda(bad))
        with pytest.raises(ValueError):
            D.VaryingCovNormal(loc=cuda(bad), cov=cuda(cov)).rvs()
    x = r.normal(size=N)
    comps = (D.Normal(loc=cuda(x)), D.Normal(scale=3.0))
    pk1 = np.array([[0.2, 0.8]])
    ref = logsumexp(np.log(pk1) + np.column_stack([stats.norm.logpdf(0.5, x), np.full(N, stats.norm.logpdf(0.5, 0, 3))]),
                    -1)
    close(host(D.Mixture(cuda(pk1), *comps).logpdf(0.5)), ref)
    assert host(D.Mixture(cuda(pk1), *comps).rvs()).shape == (N,)
    with pytest.raises(ValueError):
        D.Mixture(cuda(np.full((7, 2), 0.5)), *comps).logpdf(0.5)
    with pytest.raises(ValueError):
        D.Mixture(cuda(np.full((7, 2), 0.5)), *comps).rvs()
    with pytest.raises(ValueError):
        D.TruncNormal(mu=cuda(x), sigma=1.0, a=0.0, b=np.inf).rvs(size=N + 1)
    assert host(D.TruncNormal(mu=cuda(x), sigma=1.0, a=0.0, b=np.inf).rvs(size=N)).shape == (N,)


def test_mixture_transforms_flat(D):
    r = np.random.RandomState(5)
    n = 5000
    x = r.normal(size=n) * 3
    pk = r.dirichlet([1.0, 1.0, 1.0], size=n)
    mix = D.Mixture(cuda(pk), D.Normal(loc=-1.0), D.Normal(loc=cuda(x / 2), scale=2.0), D.Logistic(loc=1.0))
    comps = np.column_stack([stats.norm.logpdf(x, -1.0), stats.norm.logpdf(x, x / 2, 2.0),
                             stats.logistic.logpdf(x, 1.0)])
    close(host(mix.logpdf(cuda(x))), logsumexp(np.log(pk) + comps, axis=-1))
    lg = D.LogitD(D.Beta(2.0, 3.0), a=0.0, b=1.0)
    xx = np.array([-800.0, -5.0, 0.0, 5.0, 710.0, 800.0])
    jac = host(lg.logJac(cuda(xx)))
    assert np.isfinite(jac).all()                    # the reference's log(1 + exp(x)) overflows above ~709
    np.testing.assert_allclose(jac[1:4], xx[1:4] - 2 * np.log1p(np.exp(xx[1:4])), rtol=1e-14)
    fl = D.FlatNormal(loc=cuda(x))
    assert host(fl.logpdf(0.5)).shape == (n,) and not host(fl.logpdf(0.5)).any()
    assert np.isnan(host(D.FlatNormal().rvs(size=7))).all()


# ------------------------------------------------------------------------------------------------------- end to end
def _neuro_model(ssm, D):
    class NeuroXp(ssm.StateSpaceModel):
        default_params = {'M': 50, 'rho': .99, 'sig2': .0121}

        def PX0(self):
            return D.Normal()

        def PX(self, t, xp):
            return D.Normal(loc=self.rho * xp, scale=np.sqrt(self.sig2))

        def PY(self, t, xp, x):
            return D.Binomial(n=self.M, p=torch.sigmoid(x))
    return NeuroXp


def test_neuro_bootstrap_filter(D, golden):
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    data = np.loadtxt(os.path.join(GOLDEN, "neuro_thaldata.csv"), delimiter=",")
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=_neuro_model(ssm, D)(), data=data), N=1000, seed=4)
    pf.run()
    assert abs(pf.logLt - float(golden["neuro/logLt_mean"])) < 3 * float(golden["neuro/logLt_sd"])


def test_positive_state_model(D, golden):
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm

    class PosState(ssm.StateSpaceModel):
        default_params = {'rho': 0.9, 'sigma': 0.5}

        def PX0(self):
            return D.LogD(D.Gamma(a=2.0, b=1.0))

        def PX(self, t, xp):
            return D.TruncNormal(mu=self.rho * xp, sigma=self.sigma, a=0.0, b=np.inf)

        def PY(self, t, xp, x):
            return D.Mixture([0.9, 0.1], D.Normal(loc=x), D.Normal(loc=x, scale=10.0))

    y = golden["posstate/data"]
    lls = []
    for s in range(3):
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=PosState(), data=y), N=1000, seed=10 + s)
        pf.run()
        lls.append(pf.logLt)
    m, sd = float(golden["posstate/logLt_mean"]), float(golden["posstate/logLt_sd"])
    assert all(abs(v - m) < 3 * sd for v in lls), (lls, m, sd)


def test_cond_logd_prior(D):
    """The Bayes_estimation_ssm dependent prior: rvs and logpdf against the reference's formulas on the same draws."""
    import particles_b200 as pb
    prior = D.StructDist({"rho": D.LogD(D.Gamma(a=2.0, b=1.0)),
                          "sigma": D.Cond(lambda th: D.Gamma(a=1.0, b=1.0 / np.exp(th["rho"])))})
    pb.seed(2)
    th = prior.rvs(size=20_000)
    assert np.isfinite(th["rho"]).all() and (th["sigma"] > 0).all()
    lp = prior.logpdf(th)
    rho, sig = th["rho"], th["sigma"]
    ref = stats.gamma.logpdf(np.exp(rho), 2.0) + rho + stats.gamma.logpdf(sig, 1.0, scale=np.exp(rho))
    close(lp, ref, rtol=1e-11, atol=1e-11)
    # exp(rho) ~ Gamma(2, 1)
    assert ks_p(stats.gamma.cdf(np.exp(rho), 2.0)) > 1e-4


def test_pmmh_truncnormal_prior(D):
    """rho of LinearGauss under a TruncNormal(0.5, 0.5, -1, 1) prior: posterior mean and sd against a Kalman grid."""
    from oracle.smc_numpy import LinearGauss as OLG
    from particles_b200 import kalman, mcmc
    T, K, niter, burn = 50, 256, 2000, 500
    r = np.random.RandomState(2)
    x = np.empty(T)
    x[0] = OLG(rho=0.7, sigmaX=1.0, sigmaY=0.2).sigma0 * r.standard_normal()
    for t in range(1, T):
        x[t] = 0.7 * x[t - 1] + r.standard_normal()
    y = x + 0.2 * r.standard_normal(T)
    grid = np.linspace(-1, 1, 4002)[1:-1]
    ll = np.array([OLG(rho=g, sigmaX=1.0, sigmaY=0.2).kalman_loglik(y).sum() for g in grid])
    ll += stats.truncnorm.logpdf(grid, -3.0, 1.0, loc=0.5, scale=0.5)
    w = np.exp(ll - ll.max())
    w /= w.sum()
    pm = (w * grid).sum()
    psd = np.sqrt((w * (grid - pm) ** 2).sum())
    prior = D.StructDist({"rho": D.TruncNormal(mu=0.5, sigma=0.5, a=-1.0, b=1.0)})
    th0 = np.array([(0.5,)], dtype=[("rho", float)])
    pmmh = mcmc.PMMH(niter=niter, ssm_cls=kalman.LinearGauss, prior=prior, data=y, Nx=200, theta0=th0,
                     adaptive=False, rw_cov=np.array([[0.15 ** 2]]), nchains=K, seed=5,
                     smc_options={"resampling": "systematic"})
    pmmh.run()
    rho = pmmh.chain.theta["rho"][burn:]
    cm, csd = rho.mean(axis=0), rho.std(axis=0)
    assert abs(cm.mean() - pm) < 4 * cm.std() / np.sqrt(K), (cm.mean(), pm)
    assert abs(csd.mean() - psd) < 4 * csd.std() / np.sqrt(K), (csd.mean(), psd)
