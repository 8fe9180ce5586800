#!/usr/bin/env python
"""tools/bench_twofilter.py -- two-filter smoothing on the H100; prints one JSON line.

  python tools/bench_twofilter.py [--steps T] [--warmup W] [--reps R]

The book's configuration (book/smoothing/offline_smoothing.py): DiscreteCox (mu = 0, phi = 0.9, sigma = 0.5),
T = --steps (default 100) simulated observations, the additive function ``psit`` and a torch ``log_gamma``; the
forward and information filters are device runs with store_history=True.
  - two-filter O(N^2) per call at N = 3200, 12800, 32768 (t = T/2): with psit evaluated by torch on the pair
    blocks, and the kernel launches alone on a ready psi block (pair evaluations per second both ways);
  - two-filter O(N) and O(N) with the book's modifiers per call at N = 1e4, 1e5, 1e6;
  - smoothing_worker end to end (both runs, all T-1 estimates, one read) for every two-filter method next to
    FFBS_ON2, at N = 3200 and 12800.
Per-call times are CUDA-event times of --reps calls after --warmup untimed ones.  The card's name and power limit
are read in the same command.  Reference arm: the live reference's own two_filter_smoothing and smoothing_worker
(oracle/_ref, staged by oracle/make_ref.sh) at small N on one host core.  Writes nothing to the tree.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
MU, PHI, SIGMA = 0.0, 0.9, 0.5


def psit(t, x, xf, mu=MU, phi=PHI, sigma=SIGMA):
    if t == 0:
        return (-0.5 / sigma ** 2 + (0.5 * (1.0 - phi ** 2) / sigma ** 4) * (x - mu) ** 2
                + psit(1, x, xf, mu, phi, sigma))
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((xf - mu) - phi * (x - mu)) ** 2


def log_gamma(x, mu=MU, phi=PHI, sigma=SIGMA):
    scale = sigma / np.sqrt(1.0 - phi ** 2)
    z = (x - mu) / scale
    return -z * z / 2.0 - 0.5 * np.log(2.0 * np.pi) - np.log(scale)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def run(args):
    import torch
    import particles_b200 as pb
    from particles_b200 import _lib, collectors, state_space_models as ssm
    from particles_b200.collectors import _repeat_rows, _tile_rows
    from particles_b200.smoothing import _norm_logpdf, smoothing_worker
    from oracle import smc_numpy as orc

    class DiscreteCox_with_add_f(ssm.DiscreteCox):
        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi * self.sigma ** 2)

    T = int(args.steps)
    np.random.seed(1)
    _, y = orc.DiscreteCox(mu=MU, sigma=SIGMA, phi=PHI).simulate(T)
    y = [np.atleast_1d(v) for v in y]
    model = DiscreteCox_with_add_f(mu=MU, phi=PHI, sigma=SIGMA)
    fk, fk_info = ssm.Bootstrap(ssm=model, data=y), ssm.Bootstrap(ssm=model, data=y[::-1])

    def filters(n):
        pf = pb.SMC(fk=fk, N=n, store_history=True, seed=2)
        pf.run()
        info = pb.SMC(fk=fk_info, N=n, store_history=True, seed=3)
        info.run()
        torch.cuda.synchronize()
        return pf.hist, info

    def timed(fn):
        for _ in range(max(1, int(args.warmup))):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(int(args.reps)):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / int(args.reps)

    t = T // 2
    ti = T - 2 - t
    phi = lambda x, xf: psit(t, x, xf)                    # noqa: E731
    on2 = []
    for n in (3200, 12800, 32768):
        h, info = filters(n)
        s_call = timed(lambda: h.two_filter_smoothing(t, info, phi, log_gamma))
        # the kernel launches alone, on one ready psi block
        spec = ssm.transition_spec(h.fk)
        x, xi = h.X[t], info.hist.X[ti]
        R = max(1, min(n, collectors._ON2_PAIRS // n))
        psi = psit(t, _tile_rows(x, R), _repeat_rows(xi[:R], n)).reshape(R, n).contiguous()
        L, S = torch.empty(n, dtype=torch.float64, device=x.device), torch.empty_like(x)

        def kernels():
            for r0 in range(0, n, R):
                h._tf_desc(_lib.TF_ON2_ROWS, spec, t, x, xi, row0=r0, rows=min(R, n - r0), lw=h.wgts[t].lw,
                           psi=psi, L=L, S=S)
        s_kern = timed(kernels)
        pairs = float(n) * n
        on2.append({"N": n, "call_s": s_call, "pairs_per_s_with_phi": pairs / s_call, "kernel_s": s_kern,
                    "pairs_per_s_kernel": pairs / s_kern})
        del h, info, psi
    on = []
    for n in (10000, 100000, 1000000):
        h, info = filters(n)
        xa, xb = h.X[t + 1], info.hist.X[ti + 1]
        mf = _norm_logpdf(h.X[t], xb.mean(), xb.std(correction=0))       # the worker's '_prop' modifiers
        mi = _norm_logpdf(info.hist.X[ti], xa.mean(), xa.std(correction=0))
        s_on = timed(lambda: h.two_filter_smoothing(t, info, phi, log_gamma, linear_cost=True))
        s_prop = timed(lambda: h.two_filter_smoothing(t, info, phi, log_gamma, linear_cost=True, modif_forward=mf,
                                                      modif_info=mi))
        on.append({"N": n, "on_call_s": s_on, "on_prop_call_s": s_prop})
        del h, info
    methods = ["FFBS_ON2", "two-filter_ON2", "two-filter_ON", "two-filter_ON_prop"]
    worker = []
    for m in methods:                                          # warm every path once
        smoothing_worker(method=m, N=200, fk=fk, fk_info=fk_info, add_func=psit, log_gamma=log_gamma)
    for n in (3200, 12800):
        for m in methods:
            np.random.seed(4)
            r = smoothing_worker(method=m, N=n, fk=fk, fk_info=fk_info, add_func=psit, log_gamma=log_gamma)
            worker.append({"method": m, "N": n, "cpu_s": r["cpu"], "sum_est": float(np.sum(r["est"]))})
    ref = None
    if os.path.isdir(os.path.join(REF_DIR, "particles")):
        sys.path.insert(0, REF_DIR)
        import particles
        from particles import smoothing as rsm, state_space_models as rssm
        from scipy import stats

        class RCox(rssm.DiscreteCox):
            def upper_bound_log_pt(self, t):
                return -0.5 * np.log(2 * np.pi * self.sigma ** 2)
        rfk = rssm.Bootstrap(ssm=RCox(mu=MU, phi=PHI, sigma=SIGMA), data=[float(v[0]) for v in y])
        rlg = lambda x: stats.norm.logpdf(x, loc=MU, scale=SIGMA / np.sqrt(1.0 - PHI ** 2))   # noqa: E731
        nr = 800
        np.random.seed(5)
        rpf = particles.SMC(fk=rfk, N=nr, store_history=True)
        rpf.run()
        rinfo = particles.SMC(fk=rssm.Bootstrap(ssm=rfk.ssm, data=rfk.data[::-1]), N=nr, store_history=True)
        rinfo.run()
        t0 = time.perf_counter()
        rpf.hist.two_filter_smoothing(t, rinfo, phi, rlg)
        r_on2 = time.perf_counter() - t0
        t0 = time.perf_counter()
        for _ in range(10):
            rpf.hist.two_filter_smoothing(t, rinfo, phi, rlg, linear_cost=True)
        r_on = (time.perf_counter() - t0) / 10
        nw = 200
        rw = {}
        for m in methods:
            np.random.seed(6)
            with contextlib.redirect_stdout(io.StringIO()):         # the worker prints its time
                rw[m] = rsm.smoothing_worker(method=m, N=nw, fk=rfk, add_func=psit, log_gamma=rlg)["cpu"]
        ref = {"kind": "the reference's own ParticleHistory / smoothing_worker (oracle/_ref), one host core",
               "N": nr, "on2_call_s": r_on2, "on2_pairs_per_s": float(nr) * nr / r_on2, "on_call_s": r_on,
               "worker_N": nw, "worker_cpu_s": rw}
    print(json.dumps({
        "metric": "two_filter_on2_pairs_per_s",
        "config": {"workload": f"book DiscreteCox (mu={MU}, phi={PHI}, sigma={SIGMA}), T={T}, psit, torch log_gamma; "
                               f"per-call times at t={t} over {args.reps} calls after {args.warmup} warm-up",
                   "card": card(), "gpu": torch.cuda.get_device_properties(0).name},
        "on2": on2, "on": on, "worker": worker, "reference": ref,
    }))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100, help="time steps T")
    ap.add_argument("--warmup", type=int, default=1, help="untimed calls before each timed series")
    ap.add_argument("--reps", type=int, default=3, help="timed calls per series")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
