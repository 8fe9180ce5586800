"""NumPy restatement of the reference's two-filter smoothing (particles/smoothing.py:487-566), test infrastructure.

``on2`` is the O(N^2) estimate in the reference's own loop (one forward particle n at a time, weights shifted by
the same upper bound); ``on_given`` is the O(N) estimate given the draws I (information filter) and J (forward
filter) the reference made, in its order of operations, so that it reproduces the reference's estimate and ESS
bit for bit.  ``on2_rows`` is the row decomposition the device computes (per information particle m: the
log-sum-exp L[m] over n and the omega-weighted mean S[m] of phi), chunked, in float64: a replay of the device's
algorithm at sizes where the reference's loop is too slow.

``logpt(t, xp, x)`` is the transition log-density, ``phi(x, xf)`` the test function.

``LOG_GAMMA`` and ``prop_modifiers`` are what the golden fixture (tests/golden/make_golden_twofilter.py) fed the
reference; the fixture does not store their values, as they follow bit for bit from the stored particles.
"""
import numpy as np
from scipy import stats

from oracle import smc_numpy as orc

# (loc, scale) of the Normal log_gamma of each golden case: the book's DiscreteCox (mu = 0, phi = 0.9, sigma = 0.5)
# and LinearGauss (sigmaX = 1, rho = 0.9) at their stationary laws; a Normal for StochVol
LOG_GAMMA = {"cox": (0.0, 0.5 / np.sqrt(1.0 - 0.9 ** 2)), "lg": (0.0, 1.0 / np.sqrt(1.0 - 0.9 ** 2)),
             "sv": (-1.0, 0.15 / np.sqrt(1.0 - 0.9 ** 2))}


def log_gamma(name, x):
    loc, scale = LOG_GAMMA[name]
    return stats.norm.logpdf(x, loc=loc, scale=scale)


def prop_modifiers(X, Xinfo, t):
    """The book's '_prop' modifiers of smoothing_worker (smoothing.py:649-660) at time t: Normal log-densities at the
    other filter's particle mean and population (ddof = 0) standard deviation.  X, Xinfo: (T, N) histories."""
    ti = X.shape[0] - 2 - t
    mf = stats.norm.logpdf(X[t], loc=np.mean(Xinfo[ti + 1]), scale=np.std(Xinfo[ti + 1]))
    mi = stats.norm.logpdf(Xinfo[ti], loc=np.mean(X[t + 1]), scale=np.std(X[t + 1]))
    return mf, mi


def on2(t, X, lw, Xinfo, lwinfo, logpt, phi, upb=0.0):
    """smoothing.py:527-547; ``upb`` = fk.upper_bound_trans(t + 1) when the model has one."""
    sp, sw = 0.0, 0.0
    shift = lwinfo.max() + lw.max() + upb
    for n in range(X.shape[0]):
        om = np.exp(lwinfo + lw[n] - shift + logpt(t + 1, X[n], Xinfo))
        sp += np.sum(om * phi(X[n], Xinfo))
        sw += np.sum(om)
    return sp / sw


def on_given(t, X, Xinfo, I, J, logpt, phi, modif_forward=None, modif_info=None):
    """smoothing.py:549-566 after the two multinomial draws: (estimate, ESS)."""
    log_omega = logpt(t + 1, X[J], Xinfo[I])
    if modif_forward is not None:
        log_omega -= modif_forward[J]
    if modif_info is not None:
        log_omega -= modif_info[I]
    Om = orc.exp_and_normalise(log_omega)
    est = np.average(phi(X[J], Xinfo[I]), axis=0, weights=Om)
    return est, 1.0 / np.sum(Om ** 2)


def on2_rows(t, X, lw, Xinfo, lwinfo, logpt, phi, chunk=256):
    """The O(N^2) estimate by rows of the information filter, as the device forms it, in float64 on the host."""
    L = np.empty(Xinfo.shape[0])
    S = np.empty(Xinfo.shape[0])
    for m0 in range(0, Xinfo.shape[0], chunk):
        xi = Xinfo[m0:m0 + chunk]
        xa, xb = np.broadcast_to(X[None, :], (xi.shape[0], X.shape[0])), np.broadcast_to(xi[:, None], (xi.shape[0],
                                                                                                     X.shape[0]))
        v = lw[None, :] + logpt(t + 1, xa, xb)
        mx = v.max(axis=1)
        ok = mx > -np.inf
        e = np.exp(v - np.where(ok, mx, 0.0)[:, None])
        s = e.sum(axis=1)
        L[m0:m0 + chunk] = np.where(ok, mx + np.log(s), -np.inf)
        with np.errstate(invalid="ignore"):
            S[m0:m0 + chunk] = np.where(ok, (e * phi(xa, xb)).sum(axis=1) / s, 0.0)
    return np.dot(orc.exp_and_normalise(lwinfo + L), S)
