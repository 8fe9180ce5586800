"""On-line smoothing of the LIVE reference on small seeded problems: the data fixture that tests/test_online_host.py
checks the NumPy oracle (tests/online_oracle.py) against bit for bit, and that tests/test_gpu_online_smoothing.py
runs the device collectors on.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_online.py

For each case: simulate data, run a seeded ``particles.SMC(store_history=True)``, then replay the reference's
``Online_smooth_naive``, ``Online_smooth_ON2``, ``Paris(Nparis=2)`` and ``Paris(Nparis=3, max_trials=2)`` (which
exercises the exact fallback) over the stored history under fixed seeds, through a stub exposing
``t, N, X, Xp, A, W, wgts, fk``.  Records the history, every summary and ``nprop``.  Writes
tests/golden/golden_online.npz.

psi = x is written ``1.0 * x``: the reference's ON2 and PaRIS update Phi in place, and Phi_0 = add_func(0, None, X_0)
would otherwise be X_0 itself, which they still read at t = 1."""
import os
import sys

import numpy as np

sys.path.insert(0, "/root/reference")
import particles  # noqa: E402
from particles import collectors as cols  # noqa: E402
from particles import kalman  # noqa: E402
from particles import resampling as rs  # noqa: E402
from particles import state_space_models as ssms  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
T, N = 50, 200


def psit(t, xp, x, mu, phi, sigma):          # the book's score of the DiscreteCox model (online_smoothing.py)
    if t == 0:
        return -0.5 / sigma ** 2 + (0.5 * (1. - phi ** 2) / sigma ** 4) * (x - mu) ** 2
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((x - mu) - phi * (xp - mu)) ** 2


class LinearGaussA(kalman.LinearGauss):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigmaX ** 2)

    def add_func(self, t, xp, x):
        return 1.0 * x


class DiscreteCoxA(ssms.DiscreteCox):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2 * np.pi) - np.log(self.sigma)

    def add_func(self, t, xp, x):
        return psit(t, xp, x, self.mu, self.phi, self.sigma)


class StochVolA(ssms.StochVol):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigma ** 2)

    def add_func(self, t, xp, x):
        return 0.0 * x if t == 0 else (x - xp) ** 2


class GuarnieroA(kalman.MVLinearGauss_Guarniero_etal):
    def upper_bound_log_pt(self, t):          # covX = I
        return -0.5 * self.dx * np.log(2.0 * np.pi)

    def add_func(self, t, xp, x):             # (K, 2)-valued
        return 1.0 * x if t == 0 else x * xp


CASES = [("lg", lambda: LinearGaussA(sigmaX=1.0, sigmaY=0.2, rho=0.9), 21),
         ("cox", lambda: DiscreteCoxA(mu=0.0, sigma=0.5, phi=0.9), 22),
         ("sv", lambda: StochVolA(), 23),
         ("mvlg2", lambda: GuarnieroA(alpha=0.4, dx=2), 24)]

COLLECTORS = [("naive", lambda: cols.Online_smooth_naive()), ("on2", lambda: cols.Online_smooth_ON2()),
              ("paris", lambda: cols.Paris(Nparis=2)), ("paris2", lambda: cols.Paris(Nparis=3, max_trials=2))]


class Stub:
    """What the on-line collectors read from a running SMC (collectors.py:345-449)."""

    def __init__(self, fk, hist, t):
        self.fk, self.t, self.N = fk, t, N
        self.X = hist["X"][t].copy()
        self.wgts = rs.Weights(lw=hist["lw"][t].copy())
        self.W = self.wgts.W
        self.A = hist["A"][t].copy() if t > 0 else None
        self.Xp = hist["X"][t - 1][self.A] if t > 0 else None


def main():
    out = {}
    for name, make, seed in CASES:
        model = make()
        np.random.seed(seed)
        _, y = model.simulate(T)
        np.random.seed(seed + 100)
        fk = ssms.Bootstrap(ssm=model, data=y)
        pf = particles.SMC(fk=fk, N=N, store_history=True)
        pf.run()
        h = pf.hist
        hist = {"X": [np.array(x) for x in h.X], "lw": [np.array(w.lw) for w in h.wgts],
                "A": [np.zeros(N, dtype=np.int64)] + [np.asarray(a, dtype=np.int64) for a in h.A[1:]]}
        out[f"{name}/data"] = np.array([np.asarray(v, dtype=float).reshape(-1) for v in y])
        out[f"{name}/X"] = np.array(hist["X"])
        out[f"{name}/lw"] = np.array(hist["lw"])
        out[f"{name}/A"] = np.array(hist["A"])
        for i, (cname, mk) in enumerate(COLLECTORS):
            col = mk()
            np.random.seed(seed + 200 + i)
            for t in range(T):
                col.collect(Stub(fk, hist, t))
            out[f"{name}/{cname}"] = np.array(col.summary, dtype=float)
            if cname.startswith("paris"):
                out[f"{name}/{cname}_nprop"] = np.array(col.nprop, dtype=float)
        print(name, "paris nprop", out[f"{name}/paris_nprop"][1:].mean(), flush=True)
    out["meta/T_N"] = np.array([T, N])
    out["meta/seeds"] = np.array([s for _, _, s in CASES])
    np.savez_compressed(os.path.join(HERE, "golden_online.npz"), **out)


if __name__ == "__main__":
    main()
