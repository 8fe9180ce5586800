"""Reference values for the laws added in particles_b200/csrc/smcb_dists.cuh, from the LIVE reference
(particles.distributions, particles.SMC): the data fixture tests/test_gpu_dists.py checks the device against.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_dists.py

Contents: (1) logpdf/<law>: the reference laws' log-densities on the test grids (x, then the values); (2) the mean and
sd of logLt over R = 30 seeded runs of the reference's bootstrap filter, N = 1000, for two models: the book's NeuroXp
(book/mle/mle_neuro.py: Binomial(50, expit(x)) observations) on the Neuro counts (tests/golden/neuro_thaldata.csv, a
copy of the reference's datasets/thaldata.csv), and a positive-state model -- X_0 ~ LogD(Gamma(2, 1)),
X_t | X_{t-1} ~ TruncNormal(0.9 x, 0.5, 0, inf), Y_t | X_t ~ Mixture([0.9, 0.1], N(x, 1), N(x, 10)) -- on T = 100
observations simulated from it (seed 3).  Writes tests/golden/golden_dists.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get("PARTICLES_REFERENCE", "/root/reference"))
import particles  # noqa: E402
from particles import distributions as dists, state_space_models as ssms  # noqa: E402
from scipy.special import expit  # noqa: E402

R, N = 30, 1000


class NeuroXp(ssms.StateSpaceModel):
    default_params = {'M': 50, 'rho': .99, 'sig2': .0121}

    def PX0(self):
        return dists.Normal()

    def PX(self, t, xp):
        return dists.Normal(loc=self.rho * xp, scale=np.sqrt(self.sig2))

    def PY(self, t, xp, x):
        return dists.Binomial(n=self.M, p=expit(x))


class PosState(ssms.StateSpaceModel):
    default_params = {'rho': 0.9, 'sigma': 0.5}

    def PX0(self):
        return dists.LogD(dists.Gamma(a=2.0, b=1.0))

    def PX(self, t, xp):
        return dists.TruncNormal(mu=self.rho * xp, sigma=self.sigma, a=0.0, b=np.inf)

    def PY(self, t, xp, x):
        return dists.Mixture([0.9, 0.1], dists.Normal(loc=x), dists.Normal(loc=x, scale=10.0))


def loglts(model, data):
    out = []
    for r in range(R):
        np.random.seed(1000 + r)
        pf = particles.SMC(fk=ssms.Bootstrap(ssm=model, data=data), N=N)
        pf.run()
        out.append(pf.logLt)
    return np.array(out)


def main():
    g = {}
    x = np.concatenate([np.linspace(-2.0, 12.0, 57), [0.0, 1e-3, 50.0]])
    k = np.arange(-1.0, 40.0)
    laws = {
        "invgamma": (dists.InvGamma(a=2.5, b=1.5), x),
        "lognormal": (dists.LogNormal(mu=-0.5, sigma=0.8), x),
        "truncnormal": (dists.TruncNormal(mu=0.5, sigma=2.0, a=-1.0, b=4.0), x),
        "truncnormal_tail": (dists.TruncNormal(mu=0.0, sigma=1.0, a=8.0, b=np.inf), np.linspace(8.0, 9.0, 11)),
        "binomial": (dists.Binomial(n=30, p=0.35), k),
        "geometric": (dists.Geometric(p=0.25), k),
        "discreteuniform": (dists.DiscreteUniform(lo=-1, hi=7), k),
        "logd_gamma": (dists.LogD(dists.Gamma(a=2.0, b=3.0)), x - 4.0),
        "lineard_normal": (dists.LinearD(dists.Normal(loc=1.0), a=2.0, b=-1.0), x),
        "logitd_beta": (dists.LogitD(dists.Beta(a=2.0, b=3.0), a=-1.0, b=2.0), x - 4.0),
        "mixture": (dists.Mixture([0.3, 0.7], dists.Normal(loc=-1.0), dists.Normal(loc=2.0, scale=0.5)), x),
    }
    for name, (law, xs) in laws.items():
        with np.errstate(all="ignore"):
            g[f"logpdf/{name}/x"] = xs
            g[f"logpdf/{name}/y"] = np.asarray(law.logpdf(xs), dtype=np.float64)
    alphas = np.array([0.7, 2.0, 3.5])
    xd = np.random.RandomState(0).dirichlet(alphas, size=50)
    g["logpdf/dirichlet/alphas"], g["logpdf/dirichlet/x"] = alphas, xd
    g["logpdf/dirichlet/y"] = dists.Dirichlet(alphas).logpdf(xd)

    data = np.loadtxt(os.path.join(HERE, "neuro_thaldata.csv"), delimiter=",")
    ll = loglts(NeuroXp(), data)
    g["neuro/logLt_mean"], g["neuro/logLt_sd"] = ll.mean(), ll.std(ddof=1)
    np.random.seed(3)
    _, y = PosState().simulate(100)
    y = np.array([float(np.ravel(v)[0]) for v in y])
    ll = loglts(PosState(), y)
    g["posstate/data"], g["posstate/logLt_mean"], g["posstate/logLt_sd"] = y, ll.mean(), ll.std(ddof=1)
    np.savez(os.path.join(HERE, "golden_dists.npz"), **g)
    print({k: v for k, v in g.items() if "logLt" in k})


if __name__ == "__main__":
    main()
