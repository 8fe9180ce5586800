"""Device time per step and logLt variance of SMC and SQMC (``SMC(qmc=True)``) on the same workloads.

    python tools/bench_sqmc.py [--runs R] [--quick]

Prints the card's name and power limit, then one JSON line per workload: Gordon_etal Bootstrap at N = 2^6 .. 2^20 (the
grid of the book's sqmc_gordon.py), StochVol Bootstrap at N = 10^6 and 10^7, and two models whose Hilbert sort
standardises d > 1 columns (BearingsOnly, MVLinearGauss_Guarniero_etal dx = 2) at N = 2^16 and 2^20, each for SMC and
SQMC.  Where oracle/_ref holds the reference's package, the reference's own SQMC time per step (one run on one host
core) follows for Gordon_etal at N <= 2^16.  ``ms_per_step``
is the time of ``run()`` between two CUDA events, over T (after one warm-up run of the same shape); ``var_logLt`` is
the variance of logLt over R runs with different seeds; ``var_x_time`` is their product, the cost of a given accuracy.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import particles_b200 as pb  # noqa: E402
from particles_b200 import kalman  # noqa: E402
from particles_b200 import state_space_models as ssm  # noqa: E402

REF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def measure(fk, N, qmc, R, T):
    pb.SMC(fk=fk, N=N, qmc=qmc, seed=1, collect="off").run()          # warm-up of this shape
    ms, lls = [], []
    for r in range(R):
        pf = pb.SMC(fk=fk, N=N, qmc=qmc, seed=100 + r, collect="off")
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        pf.run()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / T)
        lls.append(pf.logLt)
    return float(np.median(ms)), float(np.var(lls))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=16)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--quick", action="store_true", help="Gordon grid 2^6, 2^12, 2^20 and StochVol at 10^6 only")
    a = ap.parse_args()
    print("# card, power limit:", card())
    np.random.seed(1)
    torch.manual_seed(1)
    gordon, sv = ssm.Gordon_etal(), ssm.StochVol()
    yg = [v.cpu().numpy() if torch.is_tensor(v) else v for v in gordon.simulate(a.T)[1]]
    ys = [v.cpu().numpy() if torch.is_tensor(v) else v for v in sv.simulate(a.T)[1]]
    grid = [2 ** k for k in ((6, 12, 20) if a.quick else range(6, 21, 2))]
    work = [("Gordon_etal", ssm.Bootstrap(ssm=gordon, data=yg), N) for N in grid]
    work += [("StochVol", ssm.Bootstrap(ssm=sv, data=ys), N) for N in ((10 ** 6,) if a.quick else (10 ** 6, 10 ** 7))]
    for name, m in (("BearingsOnly", ssm.BearingsOnly()), ("MVLinearGauss_Guarniero_etal dx=2",
                                                           kalman.MVLinearGauss_Guarniero_etal(dx=2))):
        y = [v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v) for v in m.simulate(a.T)[1]]
        work += [(name, ssm.Bootstrap(ssm=m, data=y), N) for N in (2 ** 16, 2 ** 20)]
    for name, fk, N in work:
        for qmc in (False, True):
            R = a.runs if N <= 2 ** 20 else max(4, a.runs // 4)
            ms, var = measure(fk, N, qmc, R, a.T)
            print(json.dumps({"model": name, "kind": "Bootstrap", "N": N, "T": a.T, "algo": "SQMC" if qmc else "SMC",
                              "ms_per_step": round(ms, 5), "runs": R, "var_logLt": var,
                              "var_x_time": var * ms}), flush=True)
    if os.path.isdir(os.path.join(REF_DIR, "particles")):
        import time
        sys.path.insert(0, REF_DIR)
        import particles
        from particles import state_space_models as rssm
        for N in (2 ** 6, 2 ** 10, 2 ** 14, 2 ** 16):
            pf = particles.SMC(fk=rssm.Bootstrap(ssm=rssm.Gordon_etal(), data=yg), N=N, qmc=True)
            t0 = time.perf_counter()
            pf.run()
            ms = 1e3 * (time.perf_counter() - t0) / a.T
            print(json.dumps({"model": "Gordon_etal", "kind": "Bootstrap", "N": N, "T": a.T,
                              "algo": "SQMC, reference on one host core", "ms_per_step": round(ms, 4)}), flush=True)


if __name__ == "__main__":
    main()
