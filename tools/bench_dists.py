"""The laws of csrc/smcb_dists.cu on the device: each law's logpdf and rvs at N = 10^7 with per-particle parameters,
and the book's NeuroXp bootstrap filter (Binomial observations) at N = 10^6 over the full Neuro series, against the
reference on one host core.

    python tools/bench_dists.py [--reps 20] [--n 10000000]

Prints the card name and power limit, then one JSON line per workload.  Kernel times are CUDA events around `reps`
back-to-back public calls after a warm-up call of the same shapes (the host enqueues faster than the kernels run at
this N, so the events time the device).  Bytes per element count what the kernel reads and writes: x (logpdf), each
per-particle parameter, and the output, 8 bytes each; achieved bandwidth is shown as a share of the data-sheet
3.35 TB/s of the H100 SXM.  The samplers are bounded by their fp64 arithmetic (Philox rounds, log / exp, rejection
loops), not by memory, so their share is low by design.  The reference lines time particles.distributions (scipy /
NumPy) and particles.SMC on one host core, at the sizes named in the line.
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
import particles_b200 as pb  # noqa: E402
from particles_b200 import distributions as D, state_space_models as ssm  # noqa: E402

HBM = 3.35e12


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


def laws(n, rng):
    """name -> (law with per-particle parameters, number of array parameters, x for logpdf)"""
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()   # noqa: E731
    u = lambda lo, hi: c(rng.uniform(lo, hi, n))                                         # noqa: E731
    mu = c(rng.normal(size=n))
    return {
        "InvGamma": (D.InvGamma(a=u(1.0, 5.0), b=u(0.5, 2.0)), 2, u(0.1, 4.0)),
        "LogNormal": (D.LogNormal(mu=mu, sigma=u(0.2, 2.0)), 2, u(0.1, 4.0)),
        "TruncNormal": (D.TruncNormal(mu=mu, sigma=1.0, a=0.0, b=np.inf), 1, u(0.0, 3.0)),
        "Binomial": (D.Binomial(n=50, p=u(0.01, 0.99)), 1, c(rng.randint(0, 51, n))),
        "Geometric": (D.Geometric(p=u(0.05, 0.95)), 1, c(rng.randint(1, 20, n))),
        "NegativeBinomial": (D.NegativeBinomial(n=u(0.5, 20.0), p=u(0.1, 0.9)), 2, c(rng.randint(0, 40, n))),
        "DiscreteUniform": (D.DiscreteUniform(lo=0, hi=c(rng.randint(1, 100, n))), 1, c(rng.randint(0, 100, n))),
    }


def neuro_model(base, dists, sigmoid):
    class NeuroXp(base):
        default_params = {'M': 50, 'rho': .99, 'sig2': .0121}

        def PX0(self):
            return dists.Normal()

        def PX(self, t, xp):
            return dists.Normal(loc=self.rho * xp, scale=np.sqrt(self.sig2))

        def PY(self, t, xp, x):
            return dists.Binomial(n=self.M, p=sigmoid(x))
    return NeuroXp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=10 ** 7)
    args = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit: {pl}")
    n, rng = args.n, np.random.RandomState(0)
    pb.seed(1)
    for lname, (law, npar, x) in laws(n, rng).items():
        dt = dev_time(lambda: law.logpdf(x), args.reps)
        b = 8 * (npar + 2)
        print(json.dumps({"bench": f"{lname}.logpdf", "N": n, "device_s": dt, "bytes_per_elem": b,
                          "GB_per_s": b * n / dt / 1e9, "share_of_3.35TB_s": b * n / dt / HBM}))
        dt = dev_time(lambda: law.rvs(), args.reps)
        b = 8 * (npar + 1)
        print(json.dumps({"bench": f"{lname}.rvs", "N": n, "device_s": dt, "bytes_per_elem": b,
                          "GB_per_s": b * n / dt / 1e9, "share_of_3.35TB_s": b * n / dt / HBM,
                          "draws_per_s": n / dt}))

    data = np.loadtxt(os.path.join(ROOT, "tests", "golden", "neuro_thaldata.csv"), delimiter=",")
    T, N = len(data), 10 ** 6
    model = neuro_model(ssm.StateSpaceModel, D, torch.sigmoid)
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model(), data=data[:10]), N=N, seed=1)    # warm-up of every shape
    pf.run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model(), data=data), N=N, seed=2)
    pf.run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(json.dumps({"bench": "NeuroXp bootstrap filter (Binomial PY), plugin path", "N": N, "T": T,
                      "end_to_end_s": dt, "ms_per_step": dt / T * 1e3, "logLt": pf.logLt}))

    # the reference on one host core (oracle/_ref, copied there by build(); absent -> skipped)
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "particles")):
        print(json.dumps({"bench": "reference", "skipped": "no oracle/_ref"}))
        return
    sys.path.insert(0, ref)
    import particles
    from particles import distributions as rd, state_space_models as rssm
    from scipy.special import expit
    nr = 10 ** 6
    rx = np.random.RandomState(1)
    for lname, law, x in [("Binomial", rd.Binomial(n=50, p=rx.uniform(0.01, 0.99, nr)), rx.randint(0, 51, nr)),
                          ("TruncNormal", rd.TruncNormal(mu=rx.normal(size=nr), sigma=1.0, a=0.0, b=np.inf),
                           rx.uniform(0.0, 3.0, nr)),
                          ("InvGamma", rd.InvGamma(a=2.0, b=rx.uniform(0.5, 2.0, nr)), rx.uniform(0.1, 4.0, nr))]:
        t0 = time.perf_counter()
        law.logpdf(x)
        t1 = time.perf_counter()
        print(json.dumps({"bench": f"reference {lname}.logpdf, one host core", "N": nr, "host_s": t1 - t0}))
    Nr = 10 ** 4
    np.random.seed(0)
    t0 = time.perf_counter()
    rpf = particles.SMC(fk=rssm.Bootstrap(ssm=neuro_model(rssm.StateSpaceModel, rd, expit)(), data=data), N=Nr)
    rpf.run()
    dt = time.perf_counter() - t0
    print(json.dumps({"bench": "reference NeuroXp bootstrap filter, one host core", "N": Nr, "T": T,
                      "end_to_end_s": dt, "ms_per_step": dt / T * 1e3, "logLt": rpf.logLt}))


if __name__ == "__main__":
    main()
