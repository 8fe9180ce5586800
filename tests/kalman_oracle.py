"""NumPy restatement of the reference's Kalman filter (particles/kalman.py:169-229, 483-505) with its log-likelihood
factors.  TEST INFRASTRUCTURE for tests/test_kalman_host.py, tests/test_gpu_kalman.py and tools/bench_kalman.py.

``kalman_filter`` runs the same array operations as ``oracle.smoothing_numpy.kalman_smoother``'s forward loop and
adds ``logpyt``: scipy.stats.norm.logpdf with scale sqrt(S) for dy = 1, ``distributions.MvNormal.logpdf``'s form
(kalman.py:218-223) otherwise.  ``kalman_smoother`` is that oracle's backward loop over this filter's output, so its
bits are the oracle's (tests/test_kalman_host.py checks it)."""
import numpy as np
import scipy.linalg
import scipy.stats

HALFLOG2PI = 0.5 * np.log(2.0 * np.pi)                          # particles/distributions.py


def _dotdotinv(a, b, c):
    """a b c^{-1}, c symmetric positive (kalman.py:161-163)."""
    return scipy.linalg.solve(c, np.dot(a, b).T, assume_a="pos").T


def kalman_filter(ssm, data):
    """Kalman.filter: lists of (mean (dx,), cov (dx, dx)) pairs ``pred`` and ``filt``, and ``logpyt`` (floats)."""
    F, G, covX, covY = (np.atleast_2d(v) for v in (ssm.F, ssm.G, ssm.covX, ssm.covY))
    pred, filt, logpyt = [], [], []
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
        if covY.shape[0] == 1:
            lp = scipy.stats.norm.logpdf(yt, loc=dpm, scale=np.sqrt(dpc))
        else:
            L = np.linalg.cholesky(dpc)
            z = scipy.linalg.solve_triangular(L, np.transpose(yt - dpm), lower=True)
            lp = -0.5 * np.sum(z * z, axis=0) - np.sum(np.log(np.diag(L))) - dpc.shape[-1] * HALFLOG2PI
        logpyt.append(float(np.asarray(lp).reshape(-1)[0]))
        gain = _dotdotinv(pc, G.T, dpc)
        filt.append((pm + np.matmul(yt - dpm, gain.T), pc - np.dot(np.dot(gain, G), pc)))
    return pred, filt, logpyt


def kalman_smoother(ssm, data):
    """Kalman.smoother, kalman.py:507-517: arrays of smoothing means (T, dx) and covariances (T, dx, dx)."""
    F = np.atleast_2d(ssm.F)
    pred, filt, _ = kalman_filter(ssm, data)
    smth = [filt[-1]]
    for t in reversed(range(len(filt) - 1)):                    # smoother_step, kalman.py:266-290
        fm, fc = filt[t]
        pm, pc = pred[t + 1]
        sm, sc = smth[-1]
        J = _dotdotinv(fc, F.T, pc)
        smth.append((fm + np.matmul(sm - pm, J.T), fc + np.dot(np.dot(J, sc - pc), J.T)))
    smth.reverse()
    return np.array([m for m, _ in smth]), np.array([c for _, c in smth])
