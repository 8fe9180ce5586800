#!/usr/bin/env python
"""tools/bench_online.py -- on-line smoothing throughput on the H100; prints one JSON line.

  python tools/bench_online.py [--n N] [--n-on2 N2] [--steps T] [--warmup W]

StochVol bootstrap filter on the observations of BASELINE config 2 (T = --steps, default 100), additive function
psi = (x_t - x_{t-1})^2, fused ``run()`` in one-step batches.  CUDA-event time per step of: the filter alone in
one-step batches, plus ``Online_smooth_naive`` and plus ``Paris(Nparis=2)`` at N = --n (default 1e6), plus
``Online_smooth_ON2`` at N = --n-on2 (default 16384, reported as pair evaluations per second over the time it adds to
the filter).  Each run is
timed after --warmup untimed runs.  Reference arm: the live reference's own collectors (oracle/_ref, staged by
oracle/make_ref.sh) at a small N, timed on one host core.  Writes nothing to the tree.
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
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--n-on2", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import particles_b200 as pb
    from particles_b200 import collectors as cols, state_space_models as ssm
    from oracle import smc_numpy as orc
    T = int(args.steps)
    y = [np.atleast_1d(v) for v in orc.config2_data(T, 1)]
    bound = -0.5 * np.log(2.0 * np.pi * ssm.StochVol().sigma ** 2)

    def psi(t, xp, x):
        return 0.0 * x if t == 0 else (x - xp) ** 2

    SV = type("SV", (ssm.StochVol,), {"add_func": lambda self, t, xp, x: psi(t, xp, x),
                                      "upper_bound_log_pt": lambda self, t: bound})

    def filter_alone(n):
        """The fused filter in one-step batches, as the smoothers run it."""
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=n, seed=1)
        for _ in range(T):
            pf._engine.step(1)
        return pf

    def smoothed(n, mk):
        def run():
            pf = pb.SMC(fk=ssm.Bootstrap(ssm=SV(), data=y), N=n, collect=[mk()], seed=1)
            assert pf.fused
            pf.run()
            return pf
        return run

    def timed(fn):
        for _ in range(max(1, int(args.warmup))):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / T, out

    N, N2 = int(args.n), int(args.n_on2)
    s_filter, _ = timed(lambda: filter_alone(N))
    s_naive, _ = timed(smoothed(N, cols.Online_smooth_naive))
    s_paris, pf = timed(smoothed(N, cols.Paris))
    acc = float(np.nanmean(pf.summaries._collectors[3].acc_rate))
    s_filter2, _ = timed(lambda: filter_alone(N2))
    s_on2, _ = timed(smoothed(N2, cols.Online_smooth_ON2))
    ref = None
    if os.path.isdir(os.path.join(REF_DIR, "particles")):
        sys.path.insert(0, REF_DIR)
        import particles
        from particles import collectors as rcols, state_space_models as rssm
        RSV = type("RSV", (rssm.StochVol,), {"add_func": lambda self, t, xp, x: psi(t, xp, x),
                                             "upper_bound_log_pt": lambda self, t: bound})
        ref = {"kind": "the reference's own collectors (oracle/_ref), one host core"}
        for key, mk, nr in (("naive", rcols.Online_smooth_naive, 10000), ("paris", rcols.Paris, 1000),
                            ("on2", rcols.Online_smooth_ON2, 200)):
            np.random.seed(5)
            rpf = particles.core.SMC(fk=rssm.Bootstrap(ssm=RSV(), data=[float(v[0]) for v in y]), N=nr,
                                     collect=[mk()])
            t0 = time.perf_counter()
            rpf.run()
            ref[key] = {"N": nr, "s_per_step": (time.perf_counter() - t0) / T}
    dev = torch.cuda.get_device_properties(0)
    out = {
        "metric": "online_smoothing_s_per_step",
        "config": {"workload": f"StochVol bootstrap, config-2 data, T={T}, psi=(x-xp)^2, fused run() in one-step "
                               f"batches; naive and PaRIS (Nparis=2, max_trials=N) at N={N}, ON2 at N={N2}",
                   "gpu": dev.name, "power_limit": power_limit()},
        "filter_alone": {"N": N, "s_per_step": s_filter},
        "naive": {"N": N, "s_per_step": s_naive},
        "paris": {"N": N, "s_per_step": s_paris, "mean_acc_rate": acc},
        "on2": {"N": N2, "s_per_step": s_on2, "filter_alone_s_per_step": s_filter2,
                "pair_evals_per_s": float(N2) * N2 / max(s_on2 - s_filter2, 1e-12)},
        "reference": ref,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
