#!/usr/bin/env python
"""tools/bench_ffbs_qmc.py -- QMC forward-filtering backward-sampling on the H100; prints one JSON line.

  python tools/bench_ffbs_qmc.py [--runs R] [--warmup W]

1. ``book``: the book's gold standard (compare_mcmc_samplers_stochvol.py): StochVol(mu=-1.02, sigma=0.178,
   rho=0.9702) on the first 200 GBP/USD returns (tests/golden/golden_smc2.npz), SMC(qmc=True, N=2048,
   store_history=True), then backward_sampling_qmc(2048).  CUDA-event times of the forward pass with and without
   history, of the T - 1 Hilbert sorts the history's ``h_orders`` cost, and of the backward pass, each after warm-up.
2. ``vs_on2``: N = M = 32768, T = 100, StochVol on BASELINE config 2's data: backward_sampling_qmc of an SQMC history
   against backward_sampling_ON2 of an SMC history, pair evaluations per second, alternated in one call.
3. ``variance``: LinearGauss(sigmaX=1, sigmaY=0.2, rho=0.9), T = 100, N = M in {2^10, 2^12, 2^14}, R runs: the
   variance over runs of sum_t mean_m x_t^m and the time of forward + backward pass, QMC-FFBS on SQMC against
   ON2-FFBS on SMC.
4. ``reference``: when oracle/_ref is staged, the reference's own backward_sampling_qmc at N = 2048, M = 32 on
   workload 1's data, pair evaluations per second on one host core.
Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import particles_b200 as pb  # noqa: E402
from particles_b200 import hilbert, kalman  # noqa: E402
from particles_b200 import state_space_models as ssm  # noqa: E402

REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, warmup):
    for _ in range(max(1, warmup)):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, r


def forward(model, y, N, qmc, hist, seed=1):
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, qmc=qmc, store_history=hist, seed=seed, collect="off")
    pf.run()
    return pf


def book(warmup):
    y = np.load(os.path.join(ROOT, "tests", "golden", "golden_smc2.npz"))["gbp_usd"][:200]
    y = [np.atleast_1d(v) for v in y]
    model = ssm.StochVol(mu=-1.02, sigma=0.178, rho=0.9702)
    N = 2048
    s_hist, pf = timed(lambda: forward(model, y, N, True, True), warmup)
    s_plain, _ = timed(lambda: forward(model, y, N, True, False), warmup)
    xs = [x.reshape(-1).contiguous() for x in pf.hist.X[:-1]]
    s_sorts, _ = timed(lambda: [hilbert.hilbert_order(x) for x in xs], warmup)
    s_bwd, _ = timed(lambda: pf.hist.backward_sampling_qmc(N, seed=2), warmup)
    T = len(y)
    return {"N": N, "M": N, "T": T, "forward_with_history_s": s_hist, "forward_without_history_s": s_plain,
            "h_orders_sorts_s": s_sorts, "backward_s": s_bwd,
            "backward_pair_evals_per_s": float(N) * N * (T - 1) / s_bwd}


def vs_on2(warmup, reps=3):
    from oracle import smc_numpy as orc
    T, N = 100, 32768
    y = [np.atleast_1d(v) for v in orc.config2_data(T, 1)]
    model = ssm.StochVol()
    hq = forward(model, y, N, True, True).hist
    hs = forward(model, y, N, False, True).hist
    q, s = [], []
    for r in range(reps):
        q.append(timed(lambda: hq.backward_sampling_qmc(N, seed=4 + r), warmup if r == 0 else 0)[0])
        s.append(timed(lambda: hs.backward_sampling_ON2(N, seed=4 + r), warmup if r == 0 else 0)[0])
    pairs = float(N) * N * (T - 1)
    return {"N": N, "M": N, "T": T, "qmc_s": min(q), "on2_s": min(s), "qmc_pair_evals_per_s": pairs / min(q),
            "on2_pair_evals_per_s": pairs / min(s), "qmc_s_all": q, "on2_s_all": s}


def variance(R, warmup):
    model = kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9)
    T = 100
    np.random.seed(8)
    _, y = model.simulate(T)
    y = [np.atleast_1d(v.cpu().numpy() if hasattr(v, "cpu") else v) for v in y]
    rows = []
    for N in (2 ** 10, 2 ** 12, 2 ** 14):
        row = {"N": N}
        for name, qmc in (("qmc", True), ("on2", False)):
            def one(r):
                pf = forward(model, y, N, qmc, True, seed=100 + r)
                h = pf.hist
                p = h.backward_sampling_qmc(N, seed=200 + r) if qmc else h.backward_sampling_ON2(N, seed=200 + r)
                return torch.stack(p).mean(1).sum()
            timed(lambda: one(0), warmup)
            est, secs = [], []
            for r in range(R):
                s, e = timed(lambda: one(r), 0)
                secs.append(s)
                est.append(float(e))
            row[name] = {"var": float(np.var(est, ddof=1)), "mean": float(np.mean(est)), "seconds": float(np.mean(secs))}
        row["var_ratio_qmc_over_on2"] = row["qmc"]["var"] / row["on2"]["var"]
        row["work_normalised_gain"] = (row["on2"]["var"] * row["on2"]["seconds"]) / (row["qmc"]["var"] *
                                                                                     row["qmc"]["seconds"])
        rows.append(row)
    return {"T": T, "R": R, "rows": rows}


def reference():
    if not os.path.isdir(os.path.join(REF_DIR, "particles")):
        return None
    sys.path.insert(0, REF_DIR)
    import particles
    from particles import state_space_models as rssm
    y = [float(v) for v in np.load(os.path.join(ROOT, "tests", "golden", "golden_smc2.npz"))["gbp_usd"][:200]]
    N, M = 2048, 32
    np.random.seed(5)
    pf = particles.SMC(fk=rssm.Bootstrap(ssm=rssm.StochVol(mu=-1.02, sigma=0.178, rho=0.9702), data=y), N=N,
                       qmc=True, store_history=True)
    pf.run()
    t0 = time.perf_counter()
    pf.hist.backward_sampling_qmc(M)
    s = time.perf_counter() - t0
    return {"kind": "the reference's own ParticleHistory (oracle/_ref), one host core", "N": N, "M": M,
            "seconds": s, "pair_evals_per_s": float(N) * M * (len(y) - 1) / s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=16, help="runs per N of the variance workload")
    ap.add_argument("--warmup", type=int, default=1, help="untimed passes before each timed one")
    a = ap.parse_args()
    out = {"metric": "ffbs_qmc", "card": card(), "book": book(a.warmup), "vs_on2": vs_on2(a.warmup),
           "variance": variance(a.runs, a.warmup), "reference": reference()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
