"""IBIS on one GPU: logistic regression on synthetic data of the shapes of the book's data sets
(book/smc_samplers/logistic_reg.py of the reference): Pima-like 768 x 9 (N = 1000, K = 3 Metropolis steps) and
EEG-like 14980 x 15 (N = 1000, K = 5), prior MvNormal(scale=5), ESSrmin = 0.5, standard (len_chain = K + 1, N
particles) and waste-free (N chains of length K + 1) moves.

For every case ``SMC.run()`` (stretches of reweighting steps, one host read each) and the per-step iterator
(``for _ in pf: pass``) run with the same seed, alternating, after one untimed run of each.  One JSON line per case
and path: wall time, device->host reads (``Tensor.cpu`` / ``Tensor.item`` calls), libsmcb launches
(``ctx.launches``), device time (sum of the CUDA kernel times in a separate torch.profiler run), steps, resampling
steps, stretches, and whether logLt, theta and lpost equal the other path's bit for bit.  ``--sweep`` times
``run()`` over starting stretch lengths and growth factors instead.  The GPU's name and power limit are read in the
same call.

    python tools/bench_ibis.py [--reps 2] [--sweep] [--out bench_ibis.jsonl]
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

CASES = [("pima", 768, 9, 3), ("eeg", 14980, 15, 5)]


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:          # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


class ReadCounter:
    """Counts device->host reads (Tensor.cpu / Tensor.item) while active."""

    def __enter__(self):
        import torch
        self.n, self._cpu, self._item = 0, torch.Tensor.cpu, torch.Tensor.item
        me = self

        def cpu(t, *a, **k):
            me.n += t.is_cuda
            return me._cpu(t, *a, **k)

        def item(t, *a, **k):
            me.n += t.is_cuda
            return me._item(t, *a, **k)

        torch.Tensor.cpu, torch.Tensor.item = cpu, item
        return self

    def __exit__(self, *exc):
        import torch
        torch.Tensor.cpu, torch.Tensor.item = self._cpu, self._item


def make_pf(data, wastefree, K, N, seed):
    import particles_b200 as pb
    from particles_b200 import smc_samplers as ssp
    fk = ssp.IBIS(model=ssp.LogisticRegression(data=data, prior_scale=5.0), wastefree=wastefree, len_chain=K + 1)
    return pb.SMC(fk=fk, N=N, ESSrmin=0.5, seed=seed)


def one(data, wastefree, K, N, seed, path):
    import torch
    from particles_b200.device import context
    pf = make_pf(data, wastefree, K, N, seed)
    ctx = context()
    torch.cuda.synchronize()
    l0 = ctx.launches
    with ReadCounter() as rc:
        t0 = time.perf_counter()
        if path == "run":
            pf.run()
        else:
            for _ in pf:
                pass
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    st = getattr(pf, "_ibis_stats", None) or {}
    return pf, {"wall_s": wall, "reads": rc.n, "launches": ctx.launches - l0, "steps": pf.t,
                "resamplings": int(sum(pf.summaries.rs_flags)), "stretches": st.get("stretches", 0),
                "stretch_rows": st.get("rows", 0), "scanned_rows": st.get("scanned", 0), "logLt": pf.logLt}


def device_ms(data, wastefree, K, N, seed, path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    pf = make_pf(data, wastefree, K, N, seed)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        if path == "run":
            pf.run()
        else:
            for _ in pf:
                pass
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages()) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--N", type=int, default=1000)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from oracle.samplers_numpy import synthetic_logistic
    from particles_b200 import core
    info = gpu_info()
    lines = []

    def emit(rec):
        rec.update(info)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    if a.sweep:
        name, T, d, K = CASES[1]
        data = synthetic_logistic(T, d, seed=0)
        one(data, False, K, a.N, a.seed, "run")
        for k0, growth in ((1, 1), (4, 1), (8, 1), (32, 1), (1, 2), (4, 2), (8, 2), (32, 2), (64, 2)):
            core.IBIS_K0, core.IBIS_K_GROWTH = k0, growth
            for wf in (False, True):
                walls = []
                for r in range(a.reps):
                    _, rec = one(data, wf, K, a.N, a.seed + r, "run")
                    walls.append(rec["wall_s"])
                emit({"case": name, "move": "wastefree" if wf else "standard", "K0": k0, "growth": growth,
                      "wall_s": min(walls), "scanned_rows": rec["scanned_rows"], "stretch_rows": rec["stretch_rows"],
                      "stretches": rec["stretches"]})
    else:
        for name, T, d, K in CASES:
            data = synthetic_logistic(T, d, seed=0)
            for wf in (False, True):
                move = "wastefree" if wf else "standard"
                one(data, wf, K, a.N, a.seed, "run")
                one(data, wf, K, a.N, a.seed, "iter")
                best = {}
                for r in range(a.reps):
                    for path in ("run", "iter"):
                        pf, rec = one(data, wf, K, a.N, a.seed, path)
                        if path not in best or rec["wall_s"] < best[path][1]["wall_s"]:
                            best[path] = (pf, rec)
                pr, pi = best["run"][0], best["iter"][0]
                same = (pr.logLt == pi.logLt and pr.summaries.ESSs == pi.summaries.ESSs
                        and torch.equal(pr.X.theta, pi.X.theta) and torch.equal(pr.X.lpost, pi.X.lpost))
                for path in ("run", "iter"):
                    rec = dict(best[path][1])
                    rec.update(case=name, T=T, d=d, N=a.N, K=K, move=move, path=path, identical=bool(same),
                               device_ms=device_ms(data, wf, K, a.N, a.seed, path),
                               K0=core.IBIS_K0, growth=core.IBIS_K_GROWTH, scratch_bytes=core.IBIS_SCRATCH_BYTES)
                    emit(rec)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
