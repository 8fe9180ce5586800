#!/usr/bin/env python
"""tools/bench_variance.py -- single-run variance estimators on the H100; prints one JSON line.

  python tools/bench_variance.py [--n N] [--steps T] [--warmup W] [--prof-steps P] [--n-ref NR]

StochVol bootstrap filter on the observations of BASELINE config 2 (T = --steps, default 1000) at N = --n (default
1e7), fused ``run()`` in one-step batches.  CUDA-event time per step of: the filter alone in one-step batches, plus
``Var_logLt()``, plus ``Var()`` (phi = identity, d = 1), plus both.  Each run is timed after --warmup untimed runs.

Then one separate run of both collectors over --prof-steps steps under ``torch.profiler`` (CUDA activities, nothing
written): the CUDA time of the estimator kernels (k_var_*), and their achieved bytes/s by the byte model below,
against the data sheet's 3.35 TB/s (H100 SXM, 700 W).  Byte model per particle and step: Var_logLt reads lw in
pass 1 and B, lw in pass 2 (24 B); Var reads lw, phi in pass 1 and B, lw, phi in pass 2 (40 B); the Eve update reads
A and B[A] and writes B on resampling steps only (24 B each, per collector).

Reference arm: the live reference's ``Var`` and ``Var_logLt`` (oracle/_ref, staged by oracle/make_ref.sh; they need
numba) at N = --n-ref (default 1e4), timed on one host core.  Writes nothing to the tree.
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
HBM_BYTES_PER_S = 3.35e12


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--prof-steps", type=int, default=200)
    ap.add_argument("--n-ref", type=int, default=10_000)
    args = ap.parse_args()
    import torch
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm, variance_estimators as ve
    from oracle import smc_numpy as orc
    T, N = int(args.steps), int(args.n)
    y = [np.atleast_1d(v) for v in orc.config2_data(T, 1)]

    def filter_alone():
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=N, seed=1)
        for _ in range(T):
            pf._engine.step(1)
        return pf

    def with_cols(mk, data=y):
        def run():
            pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=data), N=N, collect=mk(), seed=1)
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

    arms = {"logLt": lambda: [ve.Var_logLt()], "var": lambda: [ve.Var()],
            "both": lambda: [ve.Var(), ve.Var_logLt()]}
    res = {"filter_alone": {"s_per_step": timed(filter_alone)[0]}}
    nres = None
    for key, mk in arms.items():
        s, pf = timed(with_cols(mk))
        res[key] = {"s_per_step": s, "added_s_per_step": s - res["filter_alone"]["s_per_step"]}
        nres = int(sum(pf.summaries.rs_flags))

    # kernel time of the estimators, in a run of its own under the profiler
    P = min(int(args.prof_steps), T)
    run = with_cols(arms["both"], y[:P])
    run()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pf = run()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if "k_var_" in ev.key:
            name = ev.key.split("k_var_")[1].split("(")[0].split("<")[0]
            dt = getattr(ev, "device_time_total", None)
            if dt is None:
                dt = ev.cuda_time_total
            kern[name] = kern.get(name, 0.0) + dt / 1e6
    prs = int(sum(pf.summaries.rs_flags[1:]))
    sums_bytes = (24 + 40) * N * P                           # Var_logLt + Var (d = 1), every step
    eve_bytes = 2 * 24 * N * prs                             # one Eve tracker per collector
    sums_s = sum(v for k, v in kern.items() if k != "eve")
    prof_out = {"steps": P, "resampling_steps": prs, "kernel_s": kern,
                "sums_s_per_step": sums_s / P, "sums_bytes_per_s": sums_bytes / max(sums_s, 1e-12),
                "sums_share_of_hbm_peak": sums_bytes / max(sums_s, 1e-12) / HBM_BYTES_PER_S,
                "eve_bytes_per_s": eve_bytes / max(kern.get("eve", 0.0), 1e-12) if prs else None}

    ref = None
    if os.path.isdir(os.path.join(REF_DIR, "particles")):
        try:
            sys.path.insert(0, REF_DIR)
            import particles
            from particles import state_space_models as rssm, variance_estimators as rve
            Tr = min(T, 200)
            ref = {"kind": "the reference's own collectors (oracle/_ref), one host core", "N": int(args.n_ref),
                   "steps": Tr}
            for key, mk in (("filter_alone", lambda: None), ("both", lambda: [rve.Var(), rve.Var_logLt()])):
                np.random.seed(5)
                rpf = particles.core.SMC(fk=rssm.Bootstrap(ssm=rssm.StochVol(), data=[float(v[0]) for v in y[:Tr]]),
                                         N=int(args.n_ref), collect=mk())
                t0 = time.perf_counter()
                rpf.run()
                ref[key] = {"s_per_step": (time.perf_counter() - t0) / Tr}
        except ImportError as e:                              # numba missing
            ref = {"unavailable": str(e)}
    dev = torch.cuda.get_device_properties(0)
    out = {
        "metric": "variance_estimators_s_per_step",
        "config": {"workload": f"StochVol bootstrap, config-2 data, N={N}, T={T}, fused run() in one-step batches, "
                               f"phi = identity", "gpu": dev.name, "power_limit": power_limit()},
        "resampling_steps": nres, **res, "profile": prof_out, "reference": ref,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
