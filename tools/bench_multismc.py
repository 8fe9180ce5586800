"""multiSMC throughput on one GPU: StochVol bootstrap filter on config-2 data (T = 1000, systematic, ESSrmin 0.5) at
N in {256, 1024, 4096, 16384, 65536} with R runs, R N >= 1e7.  Prints one JSON line with particle-steps/s of

  (a) the batched launch (csrc/smcb_batch.cu): device time from CUDA events around the launch, and the end-to-end wall
      time of ``core.run_batch`` (packing and upload of the per-run inputs, launch, the one read of the summary
      table), with the model's fused description computed once as ``multiSMC`` does for runs of one object;
  (b) the loop of single-engine ``SMC(seed=...)`` runs on the same seeds (a sample of LOOP runs, timed end to end);

then, for the routing rule of ``multiSMC`` (``core.batch_pays``), the end-to-end time of a batched group against the
loop at pairs (N, R) of few runs at large N (``--crossover``), with the rule's verdict next to the measured one;
plus, for the streaming tier, the algorithmic bytes per particle-step (32 on a plain step, 48 on a resampling step:
the CDF write and read and the ancestor gather) and the resulting fraction of the data-sheet HBM rate (3.35 TB/s,
H100 SXM).  The sampled batched runs are checked against their single-engine twins: the fraction that agrees in
every rs_flag, and the largest relative logLt difference among those.  Every shape is warmed up before it is timed.

    python tools/bench_multismc.py [--T 1000] [--loop 8] [--Ns 256,1024,...]
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

HBM = 3.35e12


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:          # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--loop", type=int, default=8)
    ap.add_argument("--Ns", default="256,1024,4096,16384,65536")
    ap.add_argument("--total", type=float, default=1e7)
    ap.add_argument("--crossover", default="16384x4,16384x16,65536x8,65536x32,65536x128,131072x32,131072x132,"
                                           "262144x64,262144x396,1048576x132")
    args = ap.parse_args()
    import torch
    import particles_b200 as pb
    from particles_b200 import core, state_space_models as ssm
    from oracle import smc_numpy as orc
    T = args.T
    y = [np.atleast_1d(v) for v in orc.config2_data(T, 1)]
    fk = ssm.Bootstrap(ssm=ssm.StochVol(), data=y)
    res = {"bench": "multismc", "model": "StochVol bootstrap, config-2 data", "T": T, **gpu_info(), "rows": []}
    for N in [int(v) for v in args.Ns.split(",")]:
        R = int(np.ceil(args.total / N))
        kws = [dict(fk=fk, N=N, resampling="systematic", ESSrmin=0.5)] * R
        seeds = list(range(1, R + 1))
        key, spec = core.batch_key(kws[0])
        core.run_batch(kws[:2], seeds[:2], _planned=(key, [spec] * 2))     # warm-up of this shape
        torch.cuda.synchronize()
        ev = []
        t0 = time.perf_counter()
        runs = core.run_batch(kws, seeds, timer=ev, _planned=(key, [spec] * R))
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        dev_s = ev[0][0].elapsed_time(ev[0][1]) / 1e3
        work = float(R) * N * T
        tier = {pb._lib.BATCH_RESIDENT: "resident", pb._lib.BATCH_STREAMING: "streaming"}[core.plan_group(key, R)[0]]
        rs_frac = float(np.mean([r.summaries.rs_flags for r in runs[:64]]))
        bytes_ps = 32 * (1 - rs_frac) + 48 * rs_frac
        # (b) the single-engine loop on the same seeds (sample)
        pb.SMC(fk=fk, N=N, seed=0).run()                        # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loop = []
        for s in seeds[:args.loop]:
            pf = pb.SMC(fk=fk, N=N, seed=s)
            pf.run()
            loop.append(pf)
        torch.cuda.synchronize()
        loop_s = (time.perf_counter() - t0) / len(loop)
        agree = [a.summaries.rs_flags == b.summaries.rs_flags for a, b in zip(loop, runs)]
        rel = [abs(a.logLt - b.logLt) / abs(a.logLt) for a, b, ok in zip(loop, runs, agree) if ok]
        row = {"N": N, "R": R, "tier": tier,
               "batched_device_ps": work / dev_s, "batched_wall_ps": work / wall,
               "batched_device_s": dev_s, "batched_wall_s": wall,
               "loop_ps": N * T / loop_s, "loop_s_per_run": loop_s,
               "speedup_device": (N * T / (dev_s / R)) / (N * T / loop_s) if dev_s > 0 else None,
               "rs_fraction": rs_frac, "agree_fraction": float(np.mean(agree)),
               "max_rel_logLt_diff_agreeing": max(rel) if rel else None}
        if tier == "streaming":
            row["bytes_per_particle_step"] = bytes_ps
            row["hbm_fraction"] = bytes_ps * work / dev_s / HBM
        res["rows"].append(row)
        del runs
        torch.cuda.empty_cache()
    # crossover of the routing rule (core.batch_pays): few runs at large N, batched launch against the loop, both
    # end to end; the loop's cost per run is taken from min(R, LOOP) runs
    res["crossover"] = []
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for N, R in [(int(a), int(b)) for a, b in (p.split("x") for p in args.crossover.split(","))]:
        kws = [dict(fk=fk, N=N, resampling="systematic", ESSrmin=0.5)] * R
        seeds = list(range(1, R + 1))
        key, spec = core.batch_key(kws[0])
        core.run_batch(kws[:1], seeds[:1], _planned=(key, [spec]), out_func=lambda pf: pf.logLt)
        pb.SMC(fk=fk, N=N, seed=0).run()
        torch.cuda.synchronize()
        ev = []
        t0 = time.perf_counter()
        core.run_batch(kws, seeds, timer=ev, _planned=(key, [spec] * R), out_func=lambda pf: pf.logLt)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        t0 = time.perf_counter()
        nl = min(R, args.loop)
        for s in seeds[:nl]:
            pb.SMC(fk=fk, N=N, seed=s).run()
        torch.cuda.synchronize()
        loop = (time.perf_counter() - t0) / nl * R
        tier, grid = core.plan_group(key, R)
        res["crossover"].append({"N": N, "R": R, "tier": tier, "grid": grid, "batched_wall_s": wall,
                                 "batched_device_s": ev[0][0].elapsed_time(ev[0][1]) / 1e3, "loop_wall_s": loop,
                                 "batched_faster": wall < loop,
                                 "rule_batches": core.batch_pays(N, R, tier, grid, n_sm=n_sm)})
    res["reference_cpu"] = "not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
