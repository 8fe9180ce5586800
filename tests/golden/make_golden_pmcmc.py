"""Particle MCMC outputs of the live reference (particles.mcmc), for tests/test_pmcmc_host.py.

CSMC: Bootstrap StochVol and LinearGauss (default parameters), Nx = 50, T = 30, data simulated under NumPy seed 1.
x* is the trajectory ``extract_one_trajectory()`` of an unconditional ``SMC(store_history=True)`` run after
``np.random.seed(2)``; then, after ``np.random.seed(3)``, one ``CSMC(xstar=x*)`` run, ``hist.extract_one_trajectory()``
and ``hist.backward_sampling_ON2(1)``, in that order.  Recorded: the history X / A / lw, logLt and both trajectories.

PMMH: LinearGauss with unknown rho, prior Uniform(-1, 1), theta0 = 0.2, T = 20, niter = 200, rw_cov = 0.3^2, for
adaptive True and False, after ``np.random.seed(4)``.  ``smc_cls`` is a stub whose ``logLt`` is the exact Kalman
log-likelihood of ``oracle.smc_numpy.LinearGauss``.  Recorded: the chain (theta, lpost, nacc) and the draws the run
consumed (the proposal normals and acceptance uniforms, re-drawn from the same seed in the same order).

    PYTHONPATH=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_pmcmc.py

Writes tests/golden/golden_pmcmc.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle.smc_numpy import LinearGauss as OLG          # noqa: E402

NX, T_CSMC, T_PMMH, NITER = 50, 30, 20, 200


def pmmh_data():
    r = np.random.RandomState(5)
    return r.standard_normal(T_PMMH)


class KalmanStub:
    """smc_cls for PMMH: logLt = the exact Kalman log-likelihood."""

    def __init__(self, fk=None, N=None, **kw):
        self.fk = fk

    def run(self):
        self.logLt = OLG(rho=float(self.fk.ssm.rho)).kalman_loglik(self.fk.data).sum()


def main():
    import scipy.stats as stats
    import particles
    from particles import distributions as dists, kalman, mcmc, state_space_models as ssms

    out = {}
    for name, model in (("sv", ssms.StochVol()), ("lg", kalman.LinearGauss())):
        np.random.seed(1)
        _, y = model.simulate(T_CSMC)
        fk = ssms.Bootstrap(ssm=model, data=y)
        np.random.seed(2)
        pf = particles.SMC(fk=fk, N=NX, store_history=True)
        pf.run()
        xstar = pf.hist.extract_one_trajectory()
        np.random.seed(3)
        c = mcmc.CSMC(fk=fk, N=NX, xstar=xstar)
        c.run()
        traj = c.hist.extract_one_trajectory()
        bwd = c.hist.backward_sampling_ON2(1)
        out[name + "_y"] = np.array([float(np.asarray(v).reshape(-1)[0]) for v in y])
        out[name + "_xstar"] = np.array([float(np.asarray(v).reshape(-1)[0]) for v in xstar])
        out[name + "_X"] = np.array([np.asarray(x, dtype=float).reshape(-1) for x in c.hist.X])
        out[name + "_A"] = np.array([np.asarray(a) for a in list(c.hist.A)[1:]])
        out[name + "_lw"] = np.array([w.lw for w in c.hist.wgts])
        out[name + "_logLt"] = np.array(c.logLt)
        out[name + "_traj"] = np.array([float(np.asarray(v).reshape(-1)[0]) for v in traj])
        out[name + "_bwd"] = np.array([float(np.asarray(v).reshape(-1)[0]) for v in bwd])

    y = pmmh_data()
    out["pmmh_y"] = y
    prior = dists.StructDist({"rho": dists.Uniform(a=-1.0, b=1.0)})
    rw_cov = np.array([[0.3 ** 2]])
    for tag, adaptive in (("ad", True), ("na", False)):
        # a fresh theta0 per run: the reference writes its proposals into the array it is given (prop_arr)
        th0 = np.array([(0.2,)], dtype=[("rho", float)])
        np.random.seed(4)
        p = mcmc.PMMH(niter=NITER, ssm_cls=kalman.LinearGauss, smc_cls=KalmanStub, prior=prior, data=y,
                      theta0=th0, adaptive=adaptive, rw_cov=rw_cov)
        p.run()
        np.random.seed(4)
        z, u = np.zeros((NITER, 1)), np.ones(NITER)
        for n in range(1, NITER):
            z[n] = stats.norm.rvs(size=1)
            u[n] = stats.uniform.rvs()
        out["pmmh_%s_theta" % tag] = p.chain.theta["rho"].copy()
        out["pmmh_%s_lpost" % tag] = p.chain.lpost.copy()
        out["pmmh_%s_nacc" % tag] = np.array(p.nacc)
        out["pmmh_%s_z" % tag], out["pmmh_%s_u" % tag] = z, u
    np.savez(os.path.join(HERE, "golden_pmcmc.npz"), **out)


if __name__ == "__main__":
    main()
