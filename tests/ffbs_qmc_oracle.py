"""NumPy restatement of the reference's QMC forward-filtering backward-sampling (``ParticleHistory.
backward_sampling_qmc``, smoothing.py:425-455), and the models of tests/golden/golden_ffbs_qmc.npz on both sides.

A history is given as lists ``X`` (T arrays (N,) or (N, d)), ``lw`` (T log-weight arrays) and ``h_orders`` (T-1 int
arrays, ``h_orders[t]`` the Hilbert order of X[t]); ``logpt(t, xp, x)`` is the transition log-density and ``u`` the
(M, T) point set.  Returns the (T, M) particle indices of the paths."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import smc_numpy as orc  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_ffbs_qmc.npz")


def oracle_model(code):
    return {0: lambda: orc.StochVol(), 1: lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
            2: lambda: orc.Gordon_etal(), 3: lambda: orc.DiscreteCox(), 4: lambda: orc.BearingsOnly(),
            5: lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[code]()


def device_model(code):
    from particles_b200 import kalman
    from particles_b200 import state_space_models as ssm
    return {0: lambda: ssm.StochVol(), 1: lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
            2: lambda: ssm.Gordon_etal(), 3: lambda: ssm.DiscreteCox(), 4: lambda: ssm.BearingsOnly(),
            5: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=2)}[code]()


def hilbert_sort(x):
    """hilbert.hilbert_sort(x) through the host build of the device's Hilbert keys (tests/sqmc_host.cpp)."""
    import test_sqmc_host as hh
    if x.ndim == 1 or x.shape[1] == 1:
        return np.argsort(x.reshape(-1))
    return np.argsort(hh.host_hilbert_keys(hh.hilbert_ints(x)))


def backward_qmc(X, lw, h_orders, logpt, u, hT=None):
    """smoothing.py:443-455 with the recorded points u; ``hT``, the Hilbert order of X[T-1], is computed if None."""
    T, M = len(X), u.shape[0]
    hT = hilbert_sort(X[-1]) if hT is None else hT
    idx = np.empty((T, M), dtype=np.int64)
    i = np.searchsorted(np.cumsum(orc.exp_and_normalise(lw[-1])[hT]), u[:, T - 1])
    idx[-1] = hT[i]
    for t in reversed(range(T - 1)):
        h = h_orders[t]
        for m in range(M):
            lwm = lw[t] + logpt(t + 1, X[t], X[t + 1][idx[t + 1, m]])
            cw = np.cumsum(orc.exp_and_normalise(lwm[h]))
            idx[t, m] = h[np.searchsorted(cw, u[m, t])]
    return idx


def case(g, k):
    """(model code, N, T, M) and the arrays of golden case k."""
    mc, N, T, M = (int(v) for v in g[f"{k}/meta"])
    return (mc, N, T, M), {name: g[f"{k}/{name}"] for name in ("y", "ub", "X", "lw", "A", "h", "paths", "idx")}
