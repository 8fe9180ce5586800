"""SMC^2 statistics of the live reference (particles.smc_samplers.SMC2), for tests/test_gpu_smc2.py, and the GBP/USD
log-returns of the reference's book example (book/smc2/smc2_stochvol_leverage.py) as a data fixture.

Configuration: LinearGauss(rho=0.9, sigmaX=1) with sigmaY unknown, prior Gamma(a=2, b=4), T = 50 observations
simulated at sigmaY = 0.5 (NumPy seed 1), N = 200 theta-particles, Nx = 50, len_chain = 5:
    "std"   wastefree=False
    "wf"    wastefree=True
    "exch"  wastefree=False, init_Nx=20, ar_to_increase_Nx=1.0 (an exchange step after every move)
16 seeds each (np.random.seed(seed) before each run).  Per run: logLt at every t, the weighted posterior mean of
sigmaY at T, the Nx trajectory (shared['Nxs']).

    PYTHONPATH=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_smc2.py

Writes tests/golden/golden_smc2.npz (runs in parallel over the host's cores)."""
import os
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
T, N, NX, LEN_CHAIN, SEEDS = 50, 200, 50, 5, 16
CONFIGS = {"std": dict(wastefree=False), "wf": dict(wastefree=True),
           "exch": dict(wastefree=False, init_Nx=20, ar_to_increase_Nx=1.0)}


def data():
    rng = np.random.RandomState(1)
    x = np.empty(T)
    x[0] = rng.randn() / np.sqrt(1.0 - 0.81)
    for t in range(1, T):
        x[t] = 0.9 * x[t - 1] + rng.randn()
    return x + 0.5 * rng.randn(T)


def one(args):
    import particles
    from particles import distributions as dists, smc_samplers as ssp
    from particles.kalman import LinearGauss
    cfg, seed = args
    opts = dict(ssm_cls=LinearGauss, prior=dists.StructDist({"sigmaY": dists.Gamma(a=2.0, b=4.0)}),
                data=data(), init_Nx=NX, len_chain=LEN_CHAIN)
    opts.update(CONFIGS[cfg])
    np.random.seed(seed)
    pf = particles.SMC(fk=ssp.SMC2(**opts), N=N)
    pf.run()
    post = float(np.sum(pf.W * pf.X.theta["sigmaY"]))
    return cfg, seed, np.array(pf.summaries.logLts), post, np.array(pf.X.shared["Nxs"])


def gbp_usd():
    import particles
    path = os.path.join(os.path.dirname(particles.__file__), "datasets", "GBP_vs_USD_9798.txt")
    rate = np.loadtxt(path, skiprows=2, usecols=(3,), comments="(C)")
    return 100.0 * np.diff(np.log(rate))


def main():
    jobs = [(c, s) for c in CONFIGS for s in range(1, SEEDS + 1)]
    with Pool(os.cpu_count()) as pool:
        res = pool.map(one, jobs)
    out = {"data": data(), "gbp_usd": gbp_usd()}
    for c in CONFIGS:
        rows = [r for r in res if r[0] == c]
        out[c + "/logLts"] = np.array([r[2] for r in rows])
        out[c + "/post_mean"] = np.array([r[3] for r in rows])
        nxs = [r[4] for r in rows]
        width = max(len(v) for v in nxs)
        out[c + "/Nxs"] = np.array([np.pad(v, (0, width - len(v)), constant_values=-1) for v in nxs])
    np.savez(os.path.join(HERE, "golden_smc2.npz"), **out)
    for c in CONFIGS:
        ll = out[c + "/logLts"][:, -1]
        print(c, "logLt %.3f +- %.3f" % (ll.mean(), ll.std(ddof=1)), "post %.4f" % out[c + "/post_mean"].mean(),
              "Nx final", out[c + "/Nxs"].max(axis=1))


if __name__ == "__main__":
    main()
