"""SMC^2 on one GPU: the book example (book/smc2/smc2_stochvol_leverage.py of the reference) on the GBP/USD
log-returns (tests/golden/golden_smc2.npz, 750 observations): N = 1000 theta-particles, init_Nx = 100,
ar_to_increase_Nx = 0.1, len_chain = 6, prior mu ~ N(0, 2^2), sigma ~ Gamma(2, 2), rho ~ Beta(9, 1),
phi ~ U(-1, 1) (StochVol drops phi), bootstrap inner filters, systematic resampling.

Runs: StochVolLeverage and StochVol with wastefree=False (the book's setting), and StochVolLeverage waste-free.
Prints one JSON line per run: wall time of ``SMC.run()``, device time of the filter-bank launches (CUDA events around
every ``smcb_bank_advance``), particle-steps the bank did, resample-move steps, Metropolis steps, final Nx, mean
acceptance rate, final logLt, and the GPU with its power limit.  A short untimed run of each model comes first.

    python tools/bench_smc2.py [--T 750] [--N 1000] [--seed 1]
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


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:          # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def run(name, ssm_cls, laws, y, N, seed, **kw):
    import torch
    import particles_b200 as pb
    from particles_b200 import distributions as dists, smc_samplers as ss
    fk = ss.SMC2(ssm_cls=ssm_cls, prior=dists.StructDist(laws), data=y, init_Nx=100, ar_to_increase_Nx=0.1,
                 len_chain=6, **kw)
    fk.timer = []
    steps = []                                      # particle-steps of every advance: filters x Nx x steps run
    from particles_b200 import bank
    orig = bank.FilterBank.advance

    def counted(self, t1, idx=None, restart=False, summaries=None, A=None):
        rows = self.R if idx is None else int(idx.shape[0])
        steps.append((rows, self.N, int(t1), bool(restart), self))
        return orig(self, t1, idx=idx, restart=restart, summaries=summaries, A=A)

    bank.FilterBank.advance = counted
    mh = []
    step0 = fk.move.mcmc.step
    fk.move.mcmc.step = lambda x, target: mh.append(1) or step0(x, target)
    torch.manual_seed(seed)
    pf = pb.SMC(fk=fk, N=N, seed=seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        pf.run()
    finally:
        bank.FilterBank.advance = orig
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    dev_ms = sum(a.elapsed_time(b) for a, b in fk.timer)
    # a restart runs t1 steps; a plain advance one step (every SMC^2 step advances by one)
    psteps = sum(r * nx * (t1 if rs else 1) for r, nx, t1, rs, _ in steps)
    rates = [float(v) for a in pf.X.shared.get("acc_rates", []) for v in (a if isinstance(a, list) else [a])
             for v in (v if isinstance(v, list) else [v])]
    res = {"run": name, "T": len(y), "N": N, "wastefree": kw.get("wastefree", True), "wall_s": round(wall, 3),
           "bank_device_s": round(dev_ms / 1e3, 3), "bank_launches": len(fk.timer),
           "particle_steps": int(psteps), "particle_steps_per_s_device": float(psteps / max(dev_ms / 1e3, 1e-12)),
           "resample_move_steps": int(sum(pf.summaries.rs_flags)), "mh_steps": len(mh),
           "final_Nx": int(pf.X.bank.N), "mean_acc_rate": float(np.mean(rates)) if rates else None,
           "logLt": float(pf.logLt)}
    res.update(gpu_info())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=750)
    ap.add_argument("--N", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    from particles_b200 import distributions as dists, state_space_models as ssm
    y = np.load(os.path.join(ROOT, "tests", "golden", "golden_smc2.npz"))["gbp_usd"][:args.T]
    sv = {"mu": dists.Normal(scale=2.0), "sigma": dists.Gamma(a=2.0, b=2.0), "rho": dists.Beta(a=9.0, b=1.0)}
    svl = dict(sv, phi=dists.Uniform(a=-1.0, b=1.0))
    for cls, laws in ((ssm.StochVolLeverage, svl), (ssm.StochVol, sv)):   # untimed: the kernels' first-use setup
        run("warmup", cls, laws, y[:20], args.N, args.seed, wastefree=False)
    for name, cls, laws, kw in (("smc2_svlev", ssm.StochVolLeverage, svl, dict(wastefree=False)),
                                ("smc2_sv", ssm.StochVol, sv, dict(wastefree=False)),
                                ("smc2_svlev_wastefree", ssm.StochVolLeverage, svl, dict(wastefree=True))):
        print(json.dumps(run(name, cls, laws, y, args.N, args.seed, **kw)), flush=True)


if __name__ == "__main__":
    main()
