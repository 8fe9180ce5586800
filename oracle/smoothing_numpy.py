"""numpy restatement of the reference's off-line smoothers (TEST INFRASTRUCTURE, see ``oracle/__init__.py``):
FFBS backward sampling (particles/smoothing.py:278-423) and the Kalman (RTS) smoother (particles/kalman.py:266-290,
507-517).  Citations are relative to the reference's root.

The backward samplers draw from the legacy global ``numpy.random`` stream in exactly the order the reference does,
so a run after the same ``np.random.seed`` reproduces the reference's indices bit-for-bit.  Each also returns the
randomness it consumed in the ``noise=`` layout of ``particles_b200.smoothing.ParticleHistory`` (idx_T, and u for
ON2; prop / lu for MCMC; prop / lu / u_exact for reject), so the device samplers can be run on identical inputs.

A history is a dict with lists ``X`` (T arrays (N,) or (N, d)), ``lw`` (T log-weight arrays), ``A`` (T ancestor
arrays, entry 0 unused); ``logpt(t, xp, x)`` is the transition log-density.
"""
import numpy as np

from . import smc_numpy as orc


def _W(lw):
    return orc.exp_and_normalise(lw)


def _init(hist, M):
    T = len(hist["X"])
    idx = np.empty((T, M), dtype=np.int64)
    idx[-1, :] = orc.multinomial(_W(hist["lw"][-1]), M)          # smoothing.py:278-281
    return idx


def backward_ON2(hist, logpt, M):
    """smoothing.py:291-311; returns (idx, noise)."""
    X, lw = hist["X"], hist["lw"]
    T = len(X)
    idx = _init(hist, M)
    u = np.zeros((M, max(T - 1, 0)))
    for m in range(M):
        for t in reversed(range(T - 1)):
            lwm = lw[t] + logpt(t + 1, X[t], X[t + 1][idx[t + 1, m]])
            u[m, t] = np.random.rand()
            idx[t, m] = orc.multinomial_once(orc.exp_and_normalise(lwm), u[m, t])
    return idx, {"idx_T": idx[-1].copy(), "u": u}


def multinomial_iid(W, M):
    """resampling.py:561-571: multinomial, then random.shuffle."""
    A = orc.multinomial(W, M)
    np.random.shuffle(A)
    return A


def backward_mcmc(hist, logpt, M, nsteps=1):
    """smoothing.py:313-350; returns (idx, noise)."""
    X, lw, A = hist["X"], hist["lw"], hist["A"]
    T = len(X)
    idx = _init(hist, M)
    prop_all = np.zeros((max(T - 1, 0), nsteps, M), dtype=np.int64)
    lu_all = np.zeros((max(T - 1, 0), nsteps, M))
    for t in reversed(range(T - 1)):
        xn = X[t + 1][idx[t + 1, :]]
        idx[t, :] = A[t + 1][idx[t + 1, :]]
        for i in range(nsteps):
            prop = multinomial_iid(_W(lw[t]), M)
            lpr_acc = logpt(t + 1, X[t][prop], xn) - logpt(t + 1, X[t][idx[t, :]], xn)
            lu = np.log(np.random.rand(M))
            idx[t, :] = np.where(lu < lpr_acc, prop, idx[t, :])
            prop_all[t, i], lu_all[t, i] = prop, lu
    return idx, {"idx_T": idx[-1].copy(), "prop": prop_all, "lu": lu_all}


class MultinomialQueue:
    """resampling.py:709-756."""

    def __init__(self, W, M):
        self.W, self.M, self.j = W, M, 0
        self.enqueue()

    def enqueue(self):
        perm = np.random.permutation(self.M)
        self.A = orc.multinomial(self.W, self.M)[perm]

    def dequeue(self, k):
        if self.j + k <= self.M:
            out = self.A[self.j:(self.j + k)]
            self.j += k
        elif k <= self.M:
            out = np.empty(k, dtype=np.int64)
            nextra = self.j + k - self.M
            out[:(k - nextra)] = self.A[self.j:]
            self.enqueue()
            out[(k - nextra):] = self.A[:nextra]
            self.j = nextra
        else:
            raise ValueError("MultinomialQueue: k must be <= M")
        return out


def backward_reject(hist, logpt, M, log_bound, max_trials=None):
    """smoothing.py:352-423 (hybrid rejection); ``log_bound(t)`` = upper_bound_trans(t).
    Returns (idx, acc_rate, noise)."""
    X, lw = hist["X"], hist["lw"]
    T = len(X)
    idx = _init(hist, M)
    if max_trials is None:
        max_trials = M
    acc_rate = np.zeros(T - 1)
    prop_all = np.zeros((max(T - 1, 0), M, max_trials), dtype=np.int64)
    lu_all = np.zeros((max(T - 1, 0), M, max_trials))
    u_exact = np.zeros((max(T - 1, 0), M))
    for t in reversed(range(T - 1)):
        where_rejected = np.arange(M)
        who_rejected = X[t + 1][idx[t + 1, :]]
        nprops, ntrials, nrejected = 0, 0, M
        gen = MultinomialQueue(_W(lw[t]), M)
        while nrejected > 0 and ntrials < max_trials:
            nprops += nrejected
            nprop = gen.dequeue(nrejected)
            lpr_acc = logpt(t + 1, X[t][nprop], who_rejected) - log_bound(t + 1)
            lu = np.log(np.random.rand(nrejected))
            prop_all[t, where_rejected, ntrials] = nprop
            lu_all[t, where_rejected, ntrials] = lu
            ntrials += 1
            newly_accepted = lu < lpr_acc
            still_rejected = np.logical_not(newly_accepted)
            idx[t, where_rejected[newly_accepted]] = nprop[newly_accepted]
            where_rejected = where_rejected[still_rejected]
            who_rejected = who_rejected[still_rejected]
            nrejected -= np.sum(newly_accepted)
        for m in where_rejected:
            lwm = lw[t] + logpt(t + 1, X[t], X[t + 1][idx[t + 1, m]])
            u_exact[t, m] = np.random.rand()
            idx[t, m] = orc.multinomial_once(orc.exp_and_normalise(lwm), u_exact[t, m])
        acc_rate[t] = (M - nrejected) / nprops
    return idx, acc_rate, {"idx_T": idx[-1].copy(), "prop": prop_all, "lu": lu_all, "u_exact": u_exact}


def px_logpt(ssm):
    """Bootstrap.logpt, state_space_models.py:341-342."""
    return lambda t, xp, x: ssm.PX(t, xp).logpdf(x)


# ----------------------------------------------------------------------------
# Kalman filter + RTS smoother -- kalman.py:157-290, 455-517 (MVLinearGauss: F, G, covX, covY, mu0, cov0)
# ----------------------------------------------------------------------------
def _dotdotinv(a, b, c):
    """a b c^{-1}, c symmetric positive (kalman.py:161-163)."""
    import scipy.linalg
    return scipy.linalg.solve(c, np.dot(a, b).T, assume_a="pos").T


def kalman_smoother(ssm, data):
    """Kalman.smoother, kalman.py:507-517: lists of smoothing means (dx,) and covariances (dx, dx)."""
    F, G, covX, covY = (np.atleast_2d(v) for v in (ssm.F, ssm.G, ssm.covX, ssm.covY))
    pred, filt = [], []
    for t, yt in enumerate(data):
        yt = np.atleast_1d(np.asarray(yt, dtype=np.float64))
        if t == 0:
            pm, pc = np.atleast_1d(np.asarray(ssm.mu0, dtype=np.float64)), np.atleast_2d(ssm.cov0)
        else:                                                   # predict_step, kalman.py:169-193
            fm, fc = filt[-1]
            pm, pc = np.matmul(fm, F.T), np.dot(np.dot(F, fc), F.T) + covX
        pred.append((pm, pc))
        dpm = np.matmul(pm, G.T)                                # filter_step, kalman.py:196-229
        dpc = np.dot(np.dot(G, pc), G.T) + covY
        gain = _dotdotinv(pc, G.T, dpc)
        filt.append((pm + np.matmul(yt - dpm, gain.T), pc - np.dot(np.dot(gain, G), pc)))
    smth = [filt[-1]]
    for t in reversed(range(len(filt) - 1)):                    # smoother_step, kalman.py:266-290
        fm, fc = filt[t]
        pm, pc = pred[t + 1]
        sm, sc = smth[-1]
        J = _dotdotinv(fc, F.T, pc)
        smth.append((fm + np.matmul(sm - pm, J.T), fc + np.dot(np.dot(J, sc - pc), J.T)))
    smth.reverse()
    return np.array([m for m, _ in smth]), np.array([c for _, c in smth])
