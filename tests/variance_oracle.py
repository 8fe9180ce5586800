"""NumPy oracle of the single-run variance estimators (particles/variance_estimators.py) and of
``Fixed_lag_smooth`` (particles/collectors.py:324-342), written from their definitions:

    var_estimate(W, phi, B) = sum_b (sum_{m: B_m = b} W_m (phi_m - m))^2,  m = sum W phi / sum W,
                              zeros when B[0] == B[-1] (whether or not B is sorted);
    var_logLt(W, B)         = sum_b (sum_{B_m = b} W_m)^2;
    Eve indices             B_0 = arange(N), B_t = B_{t-1}[A_t].
"""
import numpy as np


def normalise(lw):
    W = np.exp(lw - lw.max())
    return W / W.sum()


def branch_sums(v, B, N=None):
    """(sum_{B_m = b} v_m)_b for (N,) or (N, k) v, accumulated in index order."""
    N = v.shape[0] if N is None else N
    s = np.zeros((N,) + v.shape[1:])
    np.add.at(s, B, v)
    return s


def var_estimate(W, phi, B):
    m = np.average(phi, weights=W, axis=0)
    if B[0] == B[-1]:
        return np.zeros_like(m)
    v = (W[:, None] if phi.ndim == 2 else W) * (phi - m)
    return np.sum(branch_sums(v, B) ** 2, axis=0)


def var_logLt(W, B):
    return np.sum(branch_sums(W, B) ** 2, axis=0)


def eve_rows(A):
    """B_t for every t, from the per-step ancestors A (A[0] unused)."""
    B = [np.arange(A[0].shape[0])]
    for a in A[1:]:
        B.append(B[-1][a])
    return B


def trajectories(A, t, lag):
    """Rows of the rolling history's compute_trajectories() after step t (window of ``lag`` steps)."""
    rows = [np.arange(A[t].shape[0])]
    for s in range(t, max(t - lag + 1, 0), -1):
        rows.append(A[s][rows[-1]])
    return np.array(rows[::-1])


def replay(X, lw, A, phi, lag, phi_fl=None):
    """Every estimate of a run from its history: var, var_logLt, lag_based_var (lists of lag rows) and
    fixed_lag_smooth."""
    out = {"var": [], "var_logLt": [], "lag_based_var": [], "fixed_lag_smooth": []}
    for t, B in enumerate(eve_rows(A)):
        W = normalise(lw[t])
        px = phi(X[t])
        out["var"].append(var_estimate(W, px, B))
        out["var_logLt"].append(var_logLt(W, B))
        Bt = trajectories(A, t, lag)
        out["lag_based_var"].append([var_estimate(W, px, b) for b in Bt][::-1])
        if phi_fl is not None:
            xs = [X[t - Bt.shape[0] + 1 + i][b] for i, b in enumerate(Bt)]
            out["fixed_lag_smooth"].append(np.average(phi_fl(xs), weights=W))
    return out
