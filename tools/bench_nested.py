"""Nested sampling SMC against adaptive tempering on one GPU: the comparison of the reference's
papers/nested/tempering_vs_nested_logistic.py, on synthetic logistic-regression data of the shapes of its data sets
(Pima-like 768 x 9, EEG-like 14980 x 15, prior MvNormal(scale=5)), N = 1000 chains of len_chain = 100 (waste-free),
ESSrmin in {0.1, 0.3, 0.5, 0.7, 0.9}.

For every case the two samplers run ``--nruns`` times each, alternating, after one untimed run of each.  One JSON line
per case and sampler: wall time (mean per run), generations, likelihood evaluations N ((len_chain - 1) t + 1) as the
paper counts them, the estimate of log Z (mean and sd over the runs: X.shared['log_evid'][-1] for NS-SMC, logLt for
tempering), device->host reads (``Tensor.cpu`` / ``Tensor.item`` calls), libsmcb launches (``ctx.launches``) and
device time (sum of the CUDA kernel times in a separate torch.profiler run).  The GPU's name and power limit are read
in the same call.

``--threshold`` times the threshold step alone instead: ``smcb_ns_threshold`` at n = 1e5 (N len_chain at the paper's
sizes), 1e6 and 1e7 on log-likelihood-like values (one narrow band, so most keys share their top bits), device time
per call from CUDA events over 20 calls after 3 untimed ones, and the wall time of ``nested.threshold`` (the call
and its read) per call.

    python tools/bench_nested.py [--nruns 3] [--cases pima,eeg] [--alphas 0.1,0.3,0.5,0.7,0.9] [--out FILE]
    python tools/bench_nested.py --threshold
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_ibis import ReadCounter, gpu_info  # noqa: E402

CASES = {"pima": (768, 9), "eeg": (14980, 15)}


def make_pf(data, alg, alpha, N, lc, seed):
    import particles_b200 as pb
    from particles_b200 import nested
    from particles_b200 import smc_samplers as ssp
    model = ssp.LogisticRegression(data=data, prior_scale=5.0)
    if alg == "nested":
        fk = nested.NestedSamplingSMC(model=model, len_chain=lc, ESSrmin=alpha)
    else:
        fk = ssp.AdaptiveTempering(model=model, len_chain=lc, ESSrmin=alpha)
    return pb.SMC(fk=fk, N=N, seed=seed)


def estimate(pf):
    try:
        return pf.X.shared["log_evid"][-1]
    except (KeyError, IndexError):
        return pf.logLt


def one(data, alg, alpha, N, lc, seed):
    import torch
    from particles_b200.device import context
    pf = make_pf(data, alg, alpha, N, lc, seed)
    ctx = context()
    torch.cuda.synchronize()
    l0 = ctx.launches
    with ReadCounter() as rc:
        t0 = time.perf_counter()
        pf.run()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    return {"wall_s": wall, "reads": rc.n, "launches": ctx.launches - l0, "generations": pf.t,
            "nevals": N * ((lc - 1) * pf.t + 1), "est": estimate(pf)}


def device_ms(data, alg, alpha, N, lc, seed):
    import torch
    from torch.profiler import ProfilerActivity, profile
    pf = make_pf(data, alg, alpha, N, lc, seed)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pf.run()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages()) / 1e3


def threshold_times(n, alpha=0.5, reps=20):
    import torch
    from particles_b200 import _lib, nested
    from particles_b200.device import context, empty, ptr
    r = np.random.RandomState(n % 1000)
    llik = torch.from_numpy(-358.0 + 5.0 * r.standard_normal(n)).cuda()
    ctx = context()
    k0, k1, gamma = nested.percentile_rule(n, alpha)
    lw, out = empty(n), empty(3)

    def call():
        _lib.check(ctx.lib.smcb_ns_threshold(ctx.handle, ptr(llik), n, k0, k1, gamma, 0, float(np.log(alpha)), -np.inf,
                                             0.01, ptr(lw), ptr(out)))
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    dev = e0.elapsed_time(e1) / reps
    t0 = time.perf_counter()
    for _ in range(reps):
        nested.threshold(llik, alpha, 0, -np.inf, 0.01)
    wall = (time.perf_counter() - t0) / reps * 1e3
    want = np.percentile(llik.cpu().numpy(), 100.0 * (1.0 - alpha))
    return {"n": n, "device_ms_per_call": dev, "wall_ms_per_call_with_read": wall,
            "lt_equals_numpy": bool(out.cpu().numpy()[0] == want)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nruns", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--N", type=int, default=1000)
    ap.add_argument("--len-chain", type=int, default=100)
    ap.add_argument("--cases", default="pima,eeg")
    ap.add_argument("--alphas", default="0.1,0.3,0.5,0.7,0.9")
    ap.add_argument("--threshold", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from oracle.samplers_numpy import synthetic_logistic
    info = gpu_info()
    lines = []
    for n in ((100_000, 1_000_000, 10_000_000) if a.threshold else ()):
        rec = threshold_times(n)
        rec.update(info)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    for name in (a.cases.split(",") if not a.threshold else ()):
        T, d = CASES[name]
        data = synthetic_logistic(T, d, seed=0)
        for alpha in (float(s) for s in a.alphas.split(",")):
            recs = {"nested": [], "tempering": []}
            for alg in recs:
                one(data, alg, alpha, a.N, a.len_chain, a.seed)         # untimed
            for r in range(a.nruns):
                for alg in recs:
                    recs[alg].append(one(data, alg, alpha, a.N, a.len_chain, a.seed + 1 + r))
            for alg, rs in recs.items():
                est = np.array([x["est"] for x in rs])
                rec = {"case": name, "T": T, "d": d, "N": a.N, "len_chain": a.len_chain, "ESSrmin": alpha,
                       "alg": alg, "nruns": a.nruns,
                       "wall_s": float(np.mean([x["wall_s"] for x in rs])),
                       "generations": float(np.mean([x["generations"] for x in rs])),
                       "nevals": float(np.mean([x["nevals"] for x in rs])),
                       "est_mean": float(est.mean()), "est_sd": float(est.std(ddof=1)) if est.size > 1 else None,
                       "reads": float(np.mean([x["reads"] for x in rs])),
                       "launches": float(np.mean([x["launches"] for x in rs])),
                       "device_ms": device_ms(data, alg, alpha, a.N, a.len_chain, a.seed)}
                rec.update(info)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
