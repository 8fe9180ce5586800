"""Baum-Welch on the device (particles_b200.hmm.BaumWelch) against the reference's algorithm on one host core.

    python tools/bench_hmm.py [--reps 5]

Prints the card name and power limit, then one JSON line per measurement.  Device times are CUDA events around
whole public calls (``run()``: emission table + forward launch + backward launch; ``forward()``; ``sample(N)``)
after a warm-up of the same shapes.  The host baseline is tests/hmm_oracle.py, a NumPy restatement of the
reference's BaumWelch with the same array operations, timed for ONE HMM (or N = 200 trajectories) and scaled
linearly to the device's batch: that scaling is stated in every line that uses it.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hmm_oracle as oh  # noqa: E402
from particles_b200 import hmm  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def model(rng, K, B=None):
    lead = () if B is None else (B,)
    trans = rng.dirichlet(np.ones(K), size=lead + (K,)) + np.eye(K)
    trans /= trans.sum(-1, keepdims=True)
    init = np.full(K, 1.0 / K)
    mus = np.broadcast_to(np.linspace(-3.0, 3.0, K), lead + (K,)).copy()
    sigmas = np.ones(lead + (K,))
    return trans, init, mus, sigmas


def dev_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def host_time(fn, reps=1):
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit: {pl}")
    rng = np.random.RandomState(0)

    B, T = 1024, 1000
    for K in (2, 8, 32, 64, 128):
        trans, init, mus, sigmas = model(rng, K, B)
        y = rng.normal(0.0, 2.0, size=(B, T))
        m = hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas)
        yd = torch.from_numpy(y).cuda()
        dt = dev_time(lambda: hmm.BaumWelch(hmm=m, data=yd).run(), args.reps)
        with np.errstate(divide="ignore"):
            ht = host_time(lambda: oh.run(init, trans[0], mus[0], sigmas[0], y[0]))
        print(json.dumps({"bench": "forward+backward", "B": B, "T": T, "K": K, "device_s": dt,
                          "transition_updates_per_s": 2 * B * T * K * K / dt, "host_one_hmm_s": ht,
                          "host_scaled_by_B_s": ht * B, "speedup_vs_host_scaled": ht * B / dt}))

    K, T = 8, 10 ** 4
    trans, init, mus, sigmas = model(rng, K)
    y = rng.normal(0.0, 2.0, size=T)
    m = hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas)
    yd = torch.from_numpy(y).cuda()
    dt = dev_time(lambda: hmm.BaumWelch(hmm=m, data=yd).forward(), args.reps)
    lf = oh.gaussian_logft(mus, sigmas, y)
    ht = host_time(lambda: oh.forward(init, trans, lf))
    print(json.dumps({"bench": "forward one long series", "B": 1, "T": T, "K": K, "device_s": dt,
                      "host_s": ht, "speedup": ht / dt}))

    K, T, N, Nh = 8, 1000, 10 ** 5, 200
    trans, init, mus, sigmas = model(rng, K)
    y = rng.normal(0.0, 2.0, size=T)
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas), data=y)
    bw.forward()
    dt = dev_time(lambda: bw.sample(N, seed=1), args.reps)
    filt = bw.filt.cpu().numpy()
    last, U = oh.reference_uniforms(1, Nh, T)
    with np.errstate(divide="ignore"):
        ht = host_time(lambda: oh.sample(trans, filt, last, U))
    print(json.dumps({"bench": "sample", "K": K, "T": T, "N": N, "device_s": dt,
                      "trajectory_steps_per_s": N * T / dt, "host_N": Nh, "host_s": ht,
                      "host_trajectory_steps_per_s": Nh * T / ht, "host_scaled_to_N_s": ht * N / Nh,
                      "speedup_vs_host_scaled": ht * N / Nh / dt}))


if __name__ == "__main__":
    main()
