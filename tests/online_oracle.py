"""NumPy restatement of the reference's on-line smoothing collectors (particles/collectors.py:345-449): the naive
(genealogy) smoother, the O(N^2) smoother and hybrid PaRIS, replayed over a stored history.

PaRIS draws from the legacy global ``numpy.random`` stream in exactly the order the reference does (one
``MultinomialQueue`` over W_{t-1} per step, resampling.py:709-756, then one uniform per trial and per exact draw), so
a run after the same ``np.random.seed`` reproduces the reference's summaries and ``nprop`` bit for bit.  It also
returns, per step, the ancestors B (N, Nparis) and the randomness it consumed in the ``noise=`` layout of
``particles_b200.collectors.Paris``: ``prop`` / ``lu`` (N, Nparis, max_trials) and ``u_exact`` (N, Nparis).

A history is a dict with lists ``X`` (T arrays (N,) or (N, d)), ``lw`` (T log-weight arrays) and ``A`` (T ancestor
arrays, entry 0 unused); ``add_func(t, xp, x)`` is the additive function and ``logpt(t, xp, x)`` the transition
log-density, both called with the reference's broadcasting.
"""
import numpy as np

from oracle import smc_numpy as orc
from oracle.smoothing_numpy import MultinomialQueue


def _mean(Phi, W):
    return np.average(Phi, axis=0, weights=W)


def naive(hist, add_func):
    """collectors.py:368-370; returns the list of summaries."""
    X, lw, A = hist["X"], hist["lw"], hist["A"]
    out = []
    for t in range(len(X)):
        if t == 0:
            Phi = add_func(0, None, X[0])
        else:
            Phi = Phi[A[t]] + add_func(t, X[t - 1][A[t]], X[t])
        out.append(_mean(Phi, orc.exp_and_normalise(lw[t])))
    return out


def on2(hist, add_func, logpt):
    """collectors.py:373-387; returns the list of summaries."""
    X, lw = hist["X"], hist["lw"]
    out = []
    for t in range(len(X)):
        if t == 0:
            Phi = np.array(add_func(0, None, X[0]), dtype=float)
        else:
            prev = Phi.copy()
            for n in range(X[t].shape[0]):
                WXn = orc.exp_and_normalise(lw[t - 1] + logpt(t, X[t - 1], X[t][n]))
                Phi[n] = np.average(prev + add_func(t, X[t - 1], X[t][n]), axis=0, weights=WXn)
        out.append(_mean(Phi, orc.exp_and_normalise(lw[t])))
    return out


def paris(hist, add_func, logpt, log_bound, Nparis=2, max_trials=None):
    """collectors.py:390-449; returns (summaries, nprop, Bs, noises): Bs[t - 1] and noises[t - 1] belong to step
    t >= 1."""
    X, lw = hist["X"], hist["lw"]
    N = X[0].shape[0]
    mt = N if max_trials is None else max_trials
    out, nprop, Bs, noises = [], [0.0], [], []
    for t in range(len(X)):
        if t == 0:
            Phi = np.array(add_func(0, None, X[0]), dtype=float)
        else:
            prev = Phi.copy()
            Wp = orc.exp_and_normalise(lw[t - 1])
            mq = MultinomialQueue(Wp, N)
            B = np.empty((N, Nparis), dtype=np.int64)
            prop = np.zeros((N, Nparis, mt), dtype=np.int64)
            lu = np.zeros((N, Nparis, mt))
            u_exact = np.zeros((N, Nparis))
            tot = 0
            for n in range(N):
                for m in range(Nparis):
                    ntries, accepted = 0, False
                    while ntries < mt:
                        a = mq.dequeue(1)
                        lp = logpt(t, X[t - 1][a], X[t][n]) - log_bound(t)
                        v = np.log(np.random.rand())
                        prop[n, m, ntries], lu[n, m, ntries] = a[0], v
                        ntries += 1
                        if v < lp:
                            B[n, m] = a[0]
                            accepted = True
                            break
                    if not accepted:
                        WXn = orc.exp_and_normalise(lw[t - 1] + logpt(t, X[t - 1], X[t][n]))
                        u_exact[n, m] = np.random.rand()
                        B[n, m] = orc.multinomial_once(WXn, u_exact[n, m])
                    tot += ntries
                Phi[n] = np.average(prev[B[n]] + add_func(t, X[t - 1][B[n]], X[t][n]), axis=0)
            nprop.append(tot)
            Bs.append(B)
            noises.append({"prop": prop, "lu": lu, "u_exact": u_exact})
        out.append(_mean(Phi, orc.exp_and_normalise(lw[t])))
    return out, nprop, Bs, noises


# ----------------------------------------------------------------------------
# the cases of tests/golden/golden_online.npz (make_golden_online.py): additive functions and bounds, written as
# plain arithmetic so that they run on NumPy arrays and on CUDA tensors alike
# ----------------------------------------------------------------------------
SEEDS = {"lg": 21, "cox": 22, "sv": 23, "mvlg2": 24}
PARAMS = {"lg": dict(sigmaX=1.0, sigmaY=0.2, rho=0.9), "cox": dict(mu=0.0, sigma=0.5, phi=0.9), "sv": {},
          "mvlg2": dict(alpha=0.4, dx=2)}


def psit(t, xp, x, mu, phi, sigma):
    """The score of the DiscreteCox model (the reference's book/smoothing/online_smoothing.py)."""
    if t == 0:
        return -0.5 / sigma ** 2 + (0.5 * (1. - phi ** 2) / sigma ** 4) * (x - mu) ** 2
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((x - mu) - phi * (xp - mu)) ** 2


def add_func(name, m):
    if name == "lg":
        return lambda t, xp, x: 1.0 * x
    if name == "cox":
        return lambda t, xp, x: psit(t, xp, x, m.mu, m.phi, m.sigma)
    if name == "sv":
        return lambda t, xp, x: 0.0 * x if t == 0 else (x - xp) ** 2
    return lambda t, xp, x: 1.0 * x if t == 0 else x * xp


def log_bound(name, m):
    if name == "lg":
        return lambda t: -0.5 * np.log(2.0 * np.pi * m.sigmaX ** 2)
    if name == "cox":
        return lambda t: -0.5 * np.log(2 * np.pi) - np.log(m.sigma)
    if name == "sv":
        return lambda t: -0.5 * np.log(2.0 * np.pi * m.sigma ** 2)
    return lambda t: -0.5 * m.dx * np.log(2.0 * np.pi)


def history(g, name):
    return {"X": list(g[f"{name}/X"]), "lw": list(g[f"{name}/lw"]), "A": list(g[f"{name}/A"])}
