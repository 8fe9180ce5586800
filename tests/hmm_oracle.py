"""NumPy restatement of Baum-Welch for Gaussian HMMs (particles/hmm.py:143-268), operation for operation in the
reference's order, so that it reproduces the reference's outputs bit for bit on the same machine.  TEST
INFRASTRUCTURE: tests/golden/golden_hmm.npz is checked against it on the host.

Trajectory draws take their uniforms as arguments: ``last`` (N,) the sorted uniforms of the last row's multinomial
draw (``uniform_spacings``) and ``U`` (T-1, N) with U[t, n] the uniform of trajectory n at step t;
``reference_uniforms(seed, N, T)`` regenerates both from ``numpy.random.seed(seed)`` in the reference's draw order
(N + 1 ``rand`` for the spacings, then one ``rand`` per (t descending, n ascending))."""
import numpy as np
from scipy import stats


def gaussian_logft(mus, sigmas, y):
    """(T, K): log N(y_t; mus_k, sigmas_k^2) by scipy.stats.norm.logpdf, one t at a time."""
    mus, sigmas = np.asarray(mus, float), np.asarray(sigmas, float)
    return np.array([stats.norm.logpdf(yt, loc=mus, scale=sigmas) for yt in np.asarray(y, float).ravel()])


def _lse(v):
    m = v.max()
    return m + np.log(np.sum(np.exp(v - m)))


def _exp_and_normalise(lw):
    w = np.exp(lw - lw.max())
    return w / w.sum()


def forward(init, trans, logft):
    """pred, filt (T, K) and logpyt (T,)."""
    T, K = logft.shape
    pred, filt, logpyt = np.empty((T, K)), np.empty((T, K)), np.empty(T)
    for t in range(T):
        p = init if t == 0 else np.matmul(filt[t - 1], trans)
        lp = np.log(p) + logft[t]
        lpy = _lse(lp)
        pred[t], filt[t], logpyt[t] = p, np.exp(lp - lpy), lpy
    return pred, filt, logpyt


def backward(trans, logft, filt):
    """smth (T, K)."""
    T, K = filt.shape
    smth = np.empty((T, K))
    smth[-1] = filt[-1]
    log_trans = np.log(trans)
    ctg = np.zeros(K)
    for t in range(T - 2, -1, -1):
        new = np.empty(K)
        for k in range(K):
            new[k] = _lse(log_trans[k, :] + logft[t + 1] + ctg)
        ctg = new
        smth[t] = _exp_and_normalise(np.log(filt[t]) + ctg)
    return smth


def inverse_cdf(su, W):
    A = np.empty(su.shape[0], np.int64)
    j, s = 0, W[0]
    for n in range(su.shape[0]):
        while su[n] > s:
            j += 1
            s += W[j]
        A[n] = j
    return A


def reference_uniforms(seed, N, T):
    rng = np.random.RandomState(seed)
    z = np.cumsum(-np.log(rng.rand(N + 1)))
    last = z[:-1] / z[-1]
    U = np.empty((max(T - 1, 0), N))
    for t in range(T - 2, -1, -1):
        for n in range(N):
            U[t, n] = rng.rand()
    return last, U


def sample(trans, filt, last, U):
    """(T, N) int64 paths from the given uniforms (the reference's draw, unclipped)."""
    T = filt.shape[0]
    N = last.shape[0]
    paths = np.empty((T, N), np.int64)
    paths[-1] = inverse_cdf(last, filt[-1])
    log_trans = np.log(trans)
    for t in range(T - 2, -1, -1):
        lf = np.log(filt[t])
        for n in range(N):
            probs = _exp_and_normalise(log_trans[:, paths[t + 1, n]] + lf)
            paths[t, n] = np.searchsorted(np.cumsum(probs), U[t, n])
    return paths


def run(init, trans, mus, sigmas, y):
    """Every output of ``BaumWelch.run()``: logft, pred, filt, logpyt, smth."""
    logft = gaussian_logft(mus, sigmas, y)
    with np.errstate(divide="ignore"):
        pred, filt, logpyt = forward(np.asarray(init, float), np.asarray(trans, float), logft)
        smth = backward(np.asarray(trans, float), logft, filt)
    return dict(logft=logft, pred=pred, filt=filt, logpyt=logpyt, smth=smth)
