"""Particle MCMC on one GPU: PMMH and Particle Gibbs for StochVol on the first 50 GBP/USD log-returns
(tests/golden/golden_smc2.npz), Nx = 200, niter = 1000.

PMMH: prior mu ~ N(0, 2^2), rho ~ U(-1, 1), sigma ~ Gamma(1, 1), adaptive random walk, bootstrap filters with
systematic resampling.  Particle Gibbs (``PGStochVol``): the conjugate update of mu given x with rho = 0.9 and
sigma = 0.5 fixed, with and without the backward step.  Each with nchains 1 and 64.

Prints one JSON line per run: wall time of ``run()``, chain-iterations/s, launches of the library, device time from
CUDA events around every bank / conditional-SMC launch, and the GPU's name, power limit and maximum SM clock read in
the same process.  Each configuration first runs once untimed (20 iterations).  With the live reference staged in
oracle/_ref (oracle/make_ref.sh), its own PMMH and ParticleGibbs run a TRUNCATED chain (--ref-niter iterations,
nchains 1) in this process on the host, labelled as such.

    python tools/bench_pmcmc.py [--niter 1000] [--Nx 200] [--ref-niter 50] [--seed 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
T = 50
RHO, SIGMA = 0.9, 0.5


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:          # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def mu_update(theta, x, mu_sd=2.0):
    """mu | x, rho, sigma for StochVol with mu ~ N(0, mu_sd^2): x_0 ~ N(mu, sig0^2), x_t - rho x_{t-1} =
    (1 - rho) mu + sigma eps."""
    from scipy import stats
    new = theta.copy()
    rho, sigma = theta["rho"], theta["sigma"]
    x = np.array(x, dtype=float)
    sig0 = sigma / np.sqrt(1 - rho ** 2)
    prec = 1 / mu_sd ** 2 + 1 / sig0 ** 2 + (len(x) - 1) * (1 - rho) ** 2 / sigma ** 2
    num = x[0] / sig0 ** 2 + ((1 - rho) * (x[1:] - rho * x[:-1])).sum() / sigma ** 2
    new["mu"] = stats.norm.rvs(loc=num / prec, scale=1 / np.sqrt(prec))
    return new


def device_run(kind, y, niter, Nx, K, seed, backward=False):
    import torch
    from particles_b200 import distributions as dists, mcmc, state_space_models as ssm
    from particles_b200.device import context
    if kind == "pmmh":
        prior = dists.StructDist({"mu": dists.Normal(scale=2.0), "rho": dists.Uniform(a=-1.0, b=1.0),
                                  "sigma": dists.Gamma(a=1.0, b=1.0)})
        th0 = np.array([(-1.0, 0.9, 0.3)], dtype=[("mu", float), ("rho", float), ("sigma", float)])
        s = mcmc.PMMH(niter=niter, ssm_cls=ssm.StochVol, prior=prior, data=y, Nx=Nx, theta0=th0, nchains=K,
                      seed=seed, smc_options={"resampling": "systematic"})
    else:
        class PGStochVol(mcmc.ParticleGibbs):
            def update_theta(self, theta, x):
                return mu_update(theta, x)

        prior = dists.StructDist({"mu": dists.Normal(scale=2.0), "rho": dists.Dirac(RHO), "sigma": dists.Dirac(SIGMA)})
        np.random.seed(seed)
        s = PGStochVol(niter=niter, ssm_cls=ssm.StochVol, prior=prior, data=y, Nx=Nx, nchains=K, seed=seed,
                       backward_step=backward)
    s.timer = []
    ctx = context()
    l0 = ctx.launches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    dev = sum(a.elapsed_time(b) for a, b in s.timer) / 1e3
    return {"wall_s": round(wall, 3), "chain_iters_per_s": niter * K / wall, "launches": int(ctx.launches - l0),
            "device_s": round(dev, 4), "timed_launches": len(s.timer)}


def reference_run(kind, y, niter, Nx, seed, backward=False):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import particles
    from particles import distributions as rd, mcmc as rm, state_space_models as rssm
    yl = [float(v) for v in y]
    np.random.seed(seed)
    if kind == "pmmh":
        prior = rd.StructDist({"mu": rd.Normal(scale=2.0), "rho": rd.Uniform(a=-1.0, b=1.0),
                               "sigma": rd.Gamma(a=1.0, b=1.0)})
        th0 = np.array([(-1.0, 0.9, 0.3)], dtype=[("mu", float), ("rho", float), ("sigma", float)])
        s = rm.PMMH(niter=niter, ssm_cls=rssm.StochVol, smc_cls=particles.SMC, prior=prior, data=yl, Nx=Nx,
                    theta0=th0, smc_options={"resampling": "systematic"})
    else:
        class PGStochVol(rm.ParticleGibbs):
            def update_theta(self, theta, x):
                return mu_update(theta, x)

        prior = rd.StructDist({"mu": rd.Normal(scale=2.0), "rho": rd.Dirac(RHO), "sigma": rd.Dirac(SIGMA)})
        s = PGStochVol(niter=niter, ssm_cls=rssm.StochVol, prior=prior, data=yl, Nx=Nx, backward_step=backward)
    t0 = time.perf_counter()
    s.run()
    wall = time.perf_counter() - t0
    return {"wall_s": round(wall, 3), "chain_iters_per_s": niter / wall}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--niter", type=int, default=1000)
    ap.add_argument("--Nx", type=int, default=200)
    ap.add_argument("--ref-niter", type=int, default=50)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    y = np.load(os.path.join(ROOT, "tests", "golden", "golden_smc2.npz"))["gbp_usd"][:T]
    info = gpu_info()
    runs = [("pmmh", False), ("pg", False), ("pg", True)]
    for kind, bwd in runs:
        for K in (1, 64):
            device_run(kind, y, 20, args.Nx, K, args.seed, bwd)          # untimed warm-up of this configuration
            res = {"run": kind + ("_backward" if bwd else ""), "impl": "device", "nchains": K, "niter": args.niter,
                   "Nx": args.Nx, "T": T}
            res.update(device_run(kind, y, args.niter, args.Nx, K, args.seed, bwd))
            res.update(info)
            print(json.dumps(res), flush=True)
    if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "particles")):
        for kind, bwd in runs:
            res = {"run": kind + ("_backward" if bwd else ""), "impl": "reference (host, truncated)", "nchains": 1,
                   "niter": args.ref_niter, "Nx": args.Nx, "T": T}
            res.update(reference_run(kind, y, args.ref_niter, args.Nx, args.seed, bwd))
            print(json.dumps(res), flush=True)
    else:
        print(json.dumps({"impl": "reference", "skipped": "oracle/_ref is not staged"}), flush=True)


if __name__ == "__main__":
    main()
