#!/usr/bin/env python
"""tools/bench_ffbs.py -- off-line smoothing (FFBS) throughput on the H100; prints one JSON line.

  python tools/bench_ffbs.py [--n N] [--steps T] [--warmup W]

Forward StochVol bootstrap filter with store_history=True (N particles, default 1e6; T = --steps, default 100) on the
observations of BASELINE config 2, then backward_sampling_mcmc and backward_sampling_reject with M = N, and
backward_sampling_ON2 at N = M = 32768 on its own history.  Every backward pass is CUDA-event timed after --warmup
untimed passes (at least one).  Reference arm: the live reference's own backward samplers (oracle/_ref, staged by
oracle/make_ref.sh) on a bounded sample, timed on one host core.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")        # the live reference's package, if staged


def have_live_reference():
    return os.path.isdir(os.path.join(REF_DIR, "particles"))


def run_ffbs(args):
    """The workload of the module docstring; prints its JSON line."""
    import torch
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    from oracle import smc_numpy as orc
    T, N = int(args.steps), int(args.n)
    y = [np.atleast_1d(v) for v in orc.config2_data(T, 1)]
    bound = -0.5 * np.log(2.0 * np.pi * ssm.StochVol().sigma ** 2)

    class SV(ssm.StochVol):
        def upper_bound_log_pt(self, t):
            return bound

    def history(n):
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=n, store_history=True, seed=1)
        pf.run()
        pf.hist.fk = ssm.Bootstrap(ssm=SV(), data=y)
        torch.cuda.synchronize()
        return pf.hist

    def timed(fn):
        for _ in range(max(1, int(args.warmup))):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    t0 = time.perf_counter()
    h = history(N)
    fwd_s = time.perf_counter() - t0
    s_mcmc = timed(lambda: h.backward_sampling_mcmc(N, seed=2))
    s_rej = timed(lambda: h.backward_sampling_reject(N, seed=3))
    acc = float(np.mean(h.acc_rate)) if T > 1 else None
    del h
    n2 = 32768
    h2 = history(n2)
    s_on2 = timed(lambda: h2.backward_sampling_ON2(n2, seed=4))
    del h2
    ref = None
    if have_live_reference():
        sys.path.insert(0, REF_DIR)
        import particles
        from particles import state_space_models as rssm

        class RSV(rssm.StochVol):
            def upper_bound_log_pt(self, t):
                return bound
        nr, m_on2 = 10000, 20
        np.random.seed(5)
        rpf = particles.SMC(fk=rssm.Bootstrap(ssm=RSV(), data=[float(v[0]) for v in y]), N=nr, store_history=True)
        rpf.run()
        t0 = time.perf_counter()
        rpf.hist.backward_sampling_mcmc(nr)
        r_mcmc = time.perf_counter() - t0
        t0 = time.perf_counter()
        rpf.hist.backward_sampling_ON2(m_on2)
        r_on2 = time.perf_counter() - t0
        ref = {"kind": "the reference's own ParticleHistory (oracle/_ref), one host core", "N": nr,
               "mcmc_traj_steps_per_s": nr * (T - 1) / r_mcmc, "on2_M": m_on2,
               "on2_pair_evals_per_s": float(nr) * m_on2 * (T - 1) / r_on2}
    dev = torch.cuda.get_device_properties(0)
    out = {
        "metric": "ffbs_trajectory_steps_per_s",
        "config": {"workload": f"StochVol bootstrap filter with store_history=True, N={N}, T={T}; "
                               f"MCMC (nsteps=1) and hybrid reject (max_trials=M) with M=N; ON2 at N=M={n2}",
                   "gpu": dev.name},
        "forward_with_history_s": fwd_s,
        "mcmc": {"seconds": s_mcmc, "traj_steps_per_s": N * (T - 1) / s_mcmc},
        "reject": {"seconds": s_rej, "traj_steps_per_s": N * (T - 1) / s_rej, "mean_acc_rate": acc},
        "on2": {"seconds": s_on2, "pair_evals_per_s": float(n2) * n2 * (T - 1) / s_on2},
        "reference": ref,
    }
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000, help="particles of the forward filter = trajectories M")
    ap.add_argument("--steps", type=int, default=100, help="time steps T")
    ap.add_argument("--warmup", type=int, default=1, help="untimed backward passes before each timed one")
    run_ffbs(ap.parse_args())


if __name__ == "__main__":
    main()
