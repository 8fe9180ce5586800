#!/usr/bin/env python
"""tools/bench_fusion.py -- the bench.py workload (BASELINE config 2: StochVol bootstrap, systematic, ESSrmin 0.5,
N = 1e7) with and without fused pairs of streaming steps; prints one JSON line.

  python tools/bench_fusion.py [--n N] [--steps K] [--warmup W] [--modes 0,1,2]

Per SMCB_FUSE mode: the K-step run timed with CUDA events after W untimed steps on a throw-away filter, the device's
fusion counters, and -- from a second, profiled run of the same seed -- the device time of every step-kernel
launch by kind: "plain" (one streaming step), "fused" (two), "noop" (its step done by the previous launch),
"mispredicted" (its pre-computed step resampled after all), "resample".  The kinds are replayed on the host from
the run's summaries (core.fusion_schedule) and checked against the counters.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def launch_times(make, K):
    """Device microseconds of every k_step launch of one K-step run, in launch order (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    e = make()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.step(K)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    ev = sorted((x for x in trace["traceEvents"] if x.get("cat") == "kernel" and "k_step" in x.get("name", "")),
                key=lambda x: x["ts"])
    return e, [float(x["dur"]) for x in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--modes", default="0,1")
    args = ap.parse_args()
    import torch
    import bench
    from particles_b200 import state_space_models as ssm
    from particles_b200.core import _FusedEngine, fusion_schedule
    N, K, W = args.n, args.steps, max(args.warmup, 3)
    y = bench.load_data(K).reshape(-1, 1)
    spec = ssm.fused_spec(ssm.Bootstrap(ssm=ssm.StochVol(), data=[v for v in y]))
    essrmin, scheme = bench.ESSRMIN, bench.SCHEME

    def engine(nsteps, seed):
        sp = dict(spec)
        sp["data"] = np.ascontiguousarray(y[:nsteps])
        return _FusedEngine(sp, N, scheme, essrmin, seed)

    res = {"gpu": gpu_info(), "workload": f"StochVol bootstrap, N={N}, T={K}, {scheme}, ESSrmin={essrmin}",
           "modes": {}}
    for mode in (int(m) for m in args.modes.split(",")):
        os.environ["SMCB_FUSE"] = str(mode)
        wu = engine(W, 123)
        wu.step(W)
        torch.cuda.synchronize()
        wu.close()
        e = engine(K, 2024)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        e.step(K)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        counters = e.fusion_stats()
        e.close()
        e, dur = launch_times(lambda: engine(K, 2024), K)
        kinds = fusion_schedule(e.summ.cpu().numpy(), N, essrmin, mode, [K])
        replay_ok = (len(dur) == len(kinds) and e.fusion_stats() == {k: kinds.count(k) for k in counters})
        e.close()
        per_kind = {}
        for k in ("plain", "fused", "noop", "mispredicted", "resample"):
            d = [u for u, kk in zip(dur, kinds) if kk == k]
            if d:
                per_kind[k] = {"launches": len(d), "mean_us": float(np.mean(d)), "total_ms": float(np.sum(d)) / 1e3}
        res["modes"][str(mode)] = {"value": N * K / (ms * 1e-3), "unit": "particle-steps/s", "ms_per_step": ms / K,
                                   "counters": counters, "replay_matches_counters": bool(replay_ok),
                                   "profiled_step_kernel_ms": float(np.sum(dur)) / 1e3, "per_kind": per_kind}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
