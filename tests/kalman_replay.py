"""Replay of csrc/smcb_kalman.cu in the device's operation order, vectorised over a batch of models.  TEST
INFRASTRUCTURE for tests/test_kalman_host.py and tests/test_gpu_kalman.py.

Every sum runs over its index in order from 0.0, one term at a time, as one device thread runs it; products of
matrices keep the parenthesisation of particles/kalman.py ((F Sig) F', (G P) G', P - (K G) P, (J D) J').  The
Cholesky factor is left-looking (L_ij = (A_ij - sum_{k<j} L_ik L_jk) / L_jj, a non-positive pivot is NaN), and
every solve through it is a forward then a backward substitution.  In long double (the default) the replay is the
reference the device is checked against; in float64 it performs the device's own roundings (the library is built
with -fmad=false and its +, -, *, / and sqrt are IEEE), so it predicts the device's means and covariances bit for
bit and its log-likelihoods up to the last bits of ``log``.

Shapes: parameters (B, r, c) (mu0 (B, dx)), observations (B, T, dy); results (B, T, dx), (B, T, dx, dx), (B, T)."""
import numpy as np

LD = np.longdouble
HALFLOG2PI = 0.5 * np.log(2.0 * np.pi)          # == np.log(np.sqrt(2 pi)) in fp64 (scipy's _norm_pdf_logC)


def _ab(A, B, dt):
    """A B, the sum over k in order: A (B, n, m), B (B, m, p)."""
    out = np.zeros(A.shape[:-1] + (B.shape[-1],), dt)
    for k in range(A.shape[-1]):
        out = out + A[..., :, k:k + 1] * B[..., k:k + 1, :]
    return out


def _abt(A, B, dt):
    """A B'."""
    return _ab(A, np.swapaxes(B, -1, -2), dt)


def _pivot(v):
    with np.errstate(invalid="ignore"):
        return np.where(v > 0, np.sqrt(np.where(v > 0, v, 1)), np.nan)


def chol(A, dt):
    """Left-looking Cholesky of A (B, n, n), the device's order."""
    n = A.shape[-1]
    L = np.zeros_like(A)
    for j in range(n):
        acc = np.zeros(A.shape[:-2], dt)
        for k in range(j):
            acc = acc + L[..., j, k] * L[..., j, k]
        L[..., j, j] = _pivot(A[..., j, j] - acc)
        acc = np.zeros(A.shape[:-2] + (n - j - 1,), dt)             # rows i > j, each summed over k in order
        for k in range(j):
            acc = acc + L[..., j + 1:, k] * L[..., j, k:k + 1]
        L[..., j + 1:, j] = (A[..., j + 1:, j] - acc) / L[..., j, j:j + 1]
    return L


def chol_solve_rows(L, X, dt):
    """Each row x of X (B, r, n) replaced by (L L')^-1 x."""
    X = X.copy()
    n = L.shape[-1]
    for j in range(n):
        acc = np.zeros(X.shape[:-1], dt)
        for k in range(j):
            acc = acc + L[..., None, j, k] * X[..., k]
        X[..., j] = (X[..., j] - acc) / L[..., None, j, j]
    for j in range(n - 1, -1, -1):
        acc = np.zeros(X.shape[:-1], dt)
        for k in range(j + 1, n):
            acc = acc + L[..., None, k, j] * X[..., k]
        X[..., j] = (X[..., j] - acc) / L[..., None, j, j]
    return X


def _as(v, dt, nd):
    """v with nd + 1 axes: a leading batch axis (of 1 when shared), and scalars as 1 x 1."""
    v = np.asarray(v, dt)
    return v.reshape((1,) * (nd - v.ndim) + v.shape) if v.ndim < nd else (v if v.ndim == nd else v[None])


def filter(F, G, covX, covY, mu0, cov0, y, dtype=LD):
    """SMCB_KALMAN_FILTER over every row of y: dict of pred_mean, pred_cov, filt_mean, filt_cov, logpyt."""
    dt = dtype
    F, G, covX, covY, cov0 = (_as(v, dt, 3) for v in (F, G, covX, covY, cov0))
    mu0, y = _as(mu0, dt, 2), _as(y, dt, 3)
    B = max(v.shape[0] for v in (F, G, covX, covY, mu0, cov0, y))
    T, dy, dx = y.shape[1], G.shape[-2], F.shape[-1]
    out = {k: np.empty((B, T) + s, dt) for k, s in (("pred_mean", (dx,)), ("pred_cov", (dx, dx)),
                                                    ("filt_mean", (dx,)), ("filt_cov", (dx, dx)), ("logpyt", ()))}
    m = S = None
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(T):
            if t == 0:
                pm, P = np.broadcast_to(mu0, (B, dx)).copy(), np.broadcast_to(cov0, (B, dx, dx)).copy()
            else:
                pm = _ab(F, m[..., None], dt)[..., 0]
                P = _abt(_ab(F, S, dt), F, dt) + covX
            dpm = _ab(G, pm[..., None], dt)[..., 0]
            r = y[:, t] - dpm
            L = chol(_abt(_ab(G, P, dt), G, dt) + covY, dt)
            K = chol_solve_rows(L, _abt(P, np.broadcast_to(G, (B, dy, dx)), dt), dt)      # (B, dx, dy)
            if dy == 1:
                z = r[..., 0] / L[..., 0, 0]
                lp = -(z * z) / dt(2.0) - dt(HALFLOG2PI) - np.log(L[..., 0, 0])
            else:
                w = np.zeros((B, dy), dt)
                for j in range(dy):
                    acc = np.zeros(B, dt)
                    for k in range(j):
                        acc = acc + L[:, j, k] * w[:, k]
                    w[:, j] = (r[:, j] - acc) / L[:, j, j]
                ssq, hld = np.zeros(B, dt), np.zeros(B, dt)
                for j in range(dy):
                    ssq = ssq + w[:, j] * w[:, j]
                for j in range(dy):
                    hld = hld + np.log(L[:, j, j])
                lp = dt(-0.5) * ssq - hld - dt(dy) * dt(HALFLOG2PI)
            m = pm + _ab(K, r[..., None], dt)[..., 0]
            S = P - _ab(_ab(K, np.broadcast_to(G, (B, dy, dx)), dt), P, dt)
            out["pred_mean"][:, t], out["pred_cov"][:, t] = pm, P
            out["filt_mean"][:, t], out["filt_cov"][:, t], out["logpyt"][:, t] = m, S, lp
    return out


def smooth(F, res, dtype=LD):
    """SMCB_KALMAN_SMOOTH over the rows of ``res`` (filter's output): smth_mean, smth_cov."""
    dt = dtype
    F = _as(F, dt, 3)
    fm, fc, pm, pc = (np.asarray(res[k], dt) for k in ("filt_mean", "filt_cov", "pred_mean", "pred_cov"))
    B, T, dx = fm.shape
    F = np.broadcast_to(F, (B, dx, dx))
    sm, sc = np.empty_like(fm), np.empty_like(fc)
    sm[:, -1], sc[:, -1] = fm[:, -1], fc[:, -1]
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(T - 2, -1, -1):
            J = chol_solve_rows(chol(pc[:, t + 1], dt), _abt(fc[:, t], F, dt), dt)
            D = sc[:, t + 1] - pc[:, t + 1]
            dm = sm[:, t + 1] - pm[:, t + 1]
            sc[:, t] = fc[:, t] + _abt(_ab(J, D, dt), J, dt)
            sm[:, t] = fm[:, t] + _ab(J, dm[..., None], dt)[..., 0]
    return {"smth_mean": sm, "smth_cov": sc}


def run(F, G, covX, covY, mu0, cov0, y, dtype=LD):
    out = filter(F, G, covX, covY, mu0, cov0, y, dtype)
    out.update(smooth(F, out, dtype))
    return out
