"""Baum-Welch of the LIVE reference (particles.hmm) on five seeded Gaussian HMMs: the data fixture that
tests/test_hmm_host.py checks the NumPy oracle (tests/hmm_oracle.py) against and tests/test_gpu_hmm.py runs the
device on.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_hmm.py

Cases: (a) the module docstring's K = 2 model, T = 100; (b) K = 5 with Dirichlet rows, T = 200; (c) K = 40 sticky,
T = 100; (d) K = 6 left-right, zeros in trans_mat and init_dist, T = 60; (e) K = 2, T = 1.  For each: the model,
the data, logft, pred, filt, logpyt, smth and ``sample(N)`` after ``numpy.random.seed(sample_seed)`` (the uniforms
are not stored: hmm_oracle.reference_uniforms regenerates them from the seed).  For (a) also ``smth`` after each
of the first 30 ``next()`` calls (the docstring's O(T^2) pattern), rows concatenated.
Writes tests/golden/golden_hmm.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")
from particles import hmm  # noqa: E402

N_SAMPLE = 24


def cases():
    rng = np.random.RandomState(20261018)
    out = {}
    out["a"] = dict(trans=np.array([[0.9, 0.1], [0.2, 0.8]]), init=np.full(2, 0.5), mus=np.array([0.0, 1.0]),
                    sigmas=np.ones(2), T=100)
    K = 5
    out["b"] = dict(trans=rng.dirichlet(np.ones(K), size=K), init=rng.dirichlet(np.ones(K)),
                    mus=np.linspace(-2.0, 2.0, K), sigmas=np.linspace(0.5, 1.0, K), T=200)
    K = 40
    out["c"] = dict(trans=0.9 * np.eye(K) + 0.1 / K, init=np.full(K, 1.0 / K), mus=np.linspace(-4.0, 4.0, K),
                    sigmas=np.full(K, 0.5), T=100)
    K = 6
    lr = np.zeros((K, K))
    for k in range(K - 1):
        lr[k, k], lr[k, k + 1] = 0.85, 0.15
    lr[K - 1, K - 1] = 1.0
    out["d"] = dict(trans=lr, init=np.array([0.6, 0.4, 0.0, 0.0, 0.0, 0.0]), mus=np.arange(K, dtype=float),
                    sigmas=np.full(K, 0.7), T=60)
    out["e"] = dict(trans=np.array([[0.7, 0.3], [0.4, 0.6]]), init=np.array([0.25, 0.75]), mus=np.array([-1.0, 1.0]),
                    sigmas=np.array([1.0, 2.0]), T=1)
    return out


def main():
    rec = {}
    for i, (name, c) in enumerate(sorted(cases().items())):
        m = hmm.GaussianHMM(trans_mat=c["trans"], init_dist=c["init"], mus=c["mus"], sigmas=c["sigmas"])
        np.random.seed(100 + i)
        _, y = m.simulate(c["T"])
        y = np.array(y, dtype=float).ravel()
        bw = hmm.BaumWelch(hmm=m, data=y)
        with np.errstate(divide="ignore"):
            bw.run()
            seed = 1000 + i
            np.random.seed(seed)
            paths = bw.sample(N_SAMPLE)
        p = name + "_"
        rec.update({p + "trans": c["trans"], p + "init": c["init"], p + "mus": c["mus"], p + "sigmas": c["sigmas"],
                    p + "y": y, p + "logft": np.array(bw.logft), p + "pred": np.array(bw.pred),
                    p + "filt": np.array(bw.filt), p + "logpyt": np.array(bw.logpyt), p + "smth": np.array(bw.smth),
                    p + "paths": paths.astype(np.int16), p + "sample_seed": np.int64(seed)})
        if name == "a":
            bw = hmm.BaumWelch(hmm=m, data=y)
            steps = []
            for _ in range(30):
                bw.next()
                bw.backward()
                steps.append(np.array(bw.smth))
            rec["a_smth_steps"] = np.concatenate(steps)
    rec["N_sample"] = np.int64(N_SAMPLE)
    np.savez_compressed(os.path.join(HERE, "golden_hmm.npz"), **rec)


if __name__ == "__main__":
    main()
