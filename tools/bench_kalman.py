"""The Kalman filter and smoother on the device (particles_b200.kalman.Kalman) against the reference's algorithm on
one host core.

    python tools/bench_kalman.py [--reps 5]

Prints the card name and power limit, then one JSON line per workload.  Device times are CUDA events around whole
public calls (constructing ``Kalman`` -- the parameters' copy to the device -- then ``filter()`` and, where named,
``smoother()``) after a warm-up call of the same shapes.  The host column is tests/kalman_oracle.py, a
NumPy restatement of the reference's ``Kalman`` with the same array operations, timed for ONE model and multiplied by B:
a scaled estimate, labelled as such.  Workloads: the scalar tier (one thread per model) at the size of a PMMH or grid
evaluation over 10^5 theta; the warp tier at d = 4 and at its bound d = 32 (with a flop count); one long series,
which is latency-bound.
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
import kalman_oracle as ko  # noqa: E402
from particles_b200 import kalman  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


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


def host_time(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def flops(dx, dy, smooth):
    """fp64 operations of one filter step (and one smoother step) of one model, as the kernels run them."""
    f = (2 * dx * dx + 4 * dx ** 3 + 2 * dy * dx + 2 * dy * dx * dx + 2 * dy * dy * dx + dy ** 3 / 3
         + 2 * dx * dx * dy + 2 * dx * dy * dy + 2 * dx * dy + 2 * dx * dx * dy + 2 * dx ** 3)
    s = 2 * dx ** 3 + dx ** 3 / 3 + 2 * dx ** 3 + 2 * dx ** 3 + 2 * dx ** 3 + 2 * dx * dx
    return f + (s if smooth else 0)


def run(ssm, y, smooth):
    def call():
        kf = kalman.Kalman(ssm=ssm, data=y)
        kf.smoother() if smooth else kf.filter()
    return call


class _One:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def host_one(ssm1, y1, smooth):
    return host_time(lambda: ko.kalman_smoother(ssm1, y1) if smooth else ko.kalman_filter(ssm1, y1))


def random_batch(rng, B, d):
    A = rng.normal(size=(B, d, d))
    F = 0.9 * A / np.max(np.abs(np.linalg.eigvals(A)), axis=1)[:, None, None]
    M = rng.normal(size=(B, d, d))
    cov = 0.5 * (M @ np.swapaxes(M, 1, 2) / d + np.eye(d))
    return dict(F=F, G=rng.normal(size=(B, d, d)) / np.sqrt(d), covX=cov, covY=0.6 * cov, mu0=np.zeros(d), cov0=cov)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit: {pl}")
    rng = np.random.RandomState(0)
    ko.kalman_smoother(kalman.LinearGauss(), [0.0, 1.0])         # an untimed host warm-up, as on the device

    # 1. scalar tier: 10^5 theta of LinearGauss on one shared series
    B, T = 10 ** 5, 100
    rho = np.linspace(-0.99, 0.99, B)
    y = rng.normal(size=T)
    dt = dev_time(run(kalman.LinearGauss(rho=rho), torch.from_numpy(y).cuda(), False), args.reps)
    ht = host_one(kalman.LinearGauss(rho=0.5), list(y), False)
    print(json.dumps({"bench": "LinearGauss filter, shared data", "tier": "scalar", "B": B, "T": T,
                      "device_s": dt, "model_steps_per_s": B * T / dt, "host_one_model_s": ht,
                      "host_scaled_by_B_s": ht * B, "speedup_vs_host_scaled": ht * B / dt}))

    # 2. warp tier, Guarniero et al. dx = 4: B models, per-model data
    B, T, d = 1024, 1000, 4
    g1 = kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=d)
    gB = kalman.MVLinearGauss(F=np.repeat(g1.F[None], B, 0), G=g1.G, covX=g1.covX, covY=g1.covY)
    y = rng.normal(size=(B, T, d))
    yd = torch.from_numpy(y).cuda()
    for smooth in (False, True):
        dt = dev_time(run(gB, yd, smooth), args.reps)
        ht = host_one(g1, list(y[0]), smooth)
        print(json.dumps({"bench": "Guarniero dx=4 " + ("filter+smoother" if smooth else "filter"), "tier": "warp",
                          "B": B, "T": T, "device_s": dt, "model_steps_per_s": B * T / dt, "host_one_model_s": ht,
                          "host_scaled_by_B_s": ht * B, "speedup_vs_host_scaled": ht * B / dt}))

    # 3. warp tier at its bound, dx = dy = 32
    B, T, d = 256, 100, 32
    p = random_batch(rng, B, d)
    y = rng.normal(size=(B, T, d))
    yd = torch.from_numpy(y).cuda()
    m = kalman.MVLinearGauss(**p)
    m1 = _One(**{k: (v[0] if np.ndim(v) == 3 else v) for k, v in p.items()})
    for smooth in (False, True):
        dt = dev_time(run(m, yd, smooth), args.reps)
        ht = host_one(m1, list(y[0]), smooth)
        fl = B * T * flops(d, d, smooth)
        print(json.dumps({"bench": "dx=dy=32 " + ("filter+smoother" if smooth else "filter"), "tier": "warp",
                          "B": B, "T": T, "device_s": dt, "flop": fl, "flop_per_s": fl / dt,
                          "host_one_model_s": ht, "host_scaled_by_B_s": ht * B,
                          "speedup_vs_host_scaled": ht * B / dt}))

    # 4. one long series, dx = 4
    T, Th = 10 ** 5, 10 ** 4
    y = rng.normal(size=(T, 4))
    dt = dev_time(run(g1, torch.from_numpy(y).cuda(), False), max(1, args.reps // 2))
    ht = host_one(g1, list(y[:Th]), False)
    print(json.dumps({"bench": "Guarniero dx=4 filter, one long series", "tier": "warp", "B": 1, "T": T,
                      "device_s": dt, "device_us_per_step": dt / T * 1e6, "host_T": Th, "host_s": ht,
                      "host_us_per_step": ht / Th * 1e6, "speedup": (ht / Th) / (dt / T)}))


if __name__ == "__main__":
    main()
