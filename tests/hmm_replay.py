"""Long-double replay of csrc/smcb_hmm.cu, in the device's summation orders, and of its Philox draws.  TEST
INFRASTRUCTURE for tests/test_hmm_host.py and tests/test_gpu_hmm.py.

Orders: pred_k sums over j in index order; a sum over states k is the device's group reduction -- K <= 32: one
warp, lanes padded with zeros and folded by the xor butterfly (x[i] += x[i + h], h = 16 .. 1); K > 32:
ceil(K / 32) such warps, whose partials add in warp order; the backward cost-to-go and the sampling CDFs sum over
j or k in index order inside one thread.  Trajectory draw n at step t of HMM b takes the uniform
u53(Philox4x32-10(seed; n, t, b, 7)) and returns #{k : C[path_{t+1}][k] < u}, clipped to K - 1."""
import numpy as np

import philox_ref as pr

LD = np.longdouble
PURPOSE_HMM = 7


def group_sum(v):
    """The device's sum over states of v (K,)."""
    K = v.shape[0]
    nw = 1 if K <= 32 else (K + 31) // 32
    x = np.zeros(32 * nw, dtype=LD)
    x[:K] = v
    total = None
    for w in range(nw):
        y = x[32 * w:32 * (w + 1)]
        h = 16
        while h:
            y = y[:h] + y[h:2 * h]
            h //= 2
        total = y[0] if total is None else total + y[0]
    return total


def forward(init, trans, logft):
    init, P, lf = LD(1) * np.asarray(init, LD), np.asarray(trans, LD), np.asarray(logft, LD)
    T, K = lf.shape
    pred, filt, logpyt = np.empty((T, K), LD), np.empty((T, K), LD), np.empty(T, LD)
    with np.errstate(divide="ignore", invalid="ignore"):
        for t in range(T):
            if t == 0:
                p = init.copy()
            else:
                p = np.zeros(K, LD)
                for j in range(K):
                    p = p + filt[t - 1, j] * P[j]
            lp = np.log(p) + lf[t]
            m = lp.max()
            lpy = m + np.log(group_sum(np.exp(lp - m)))
            pred[t], filt[t], logpyt[t] = p, np.exp(lp - lpy), lpy
    return pred, filt, logpyt


def backward(trans, logft, filt):
    P, lf, filt = np.asarray(trans, LD), np.asarray(logft, LD), np.asarray(filt, LD)
    T, K = filt.shape
    smth = np.empty((T, K), LD)
    smth[-1] = filt[-1]
    ctg = np.zeros(K, LD)
    with np.errstate(divide="ignore", invalid="ignore"):
        logP = np.log(P)
        for t in range(T - 2, -1, -1):
            v = (logP + lf[t + 1][None, :]) + ctg[None, :]                  # [k, j]
            mx = v.max(axis=1)
            ctg = mx + np.log(np.exp(v - mx[:, None]).sum(axis=1))
            lv = np.log(filt[t]) + ctg
            e = np.exp(lv - lv.max())
            smth[t] = e / group_sum(e)
    return smth


def run(init, trans, logft):
    pred, filt, logpyt = forward(init, trans, logft)
    return dict(pred=pred, filt=filt, logpyt=logpyt, smth=backward(trans, logft, filt))


def column_cdfs(trans, filt_t):
    """C[j, k] = cumsum_k exp_and_normalise_k(log P[k, j] + log filt_t[k])."""
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.log(np.asarray(trans, LD)).T + np.log(np.asarray(filt_t, LD))[None, :]
        w = np.exp(v - v.max(axis=1, keepdims=True))
        return np.cumsum(w / w.sum(axis=1, keepdims=True), axis=1)


def device_uniforms(seed, N, T, b=0):
    """U[t, n] of HMM b, t < T - 1, as the device draws them without injected uniforms."""
    U = np.empty((max(T - 1, 0), N))
    n = np.arange(N)
    for t in range(T - 1):
        r = pr.philox4x32_10(n, t, b, PURPOSE_HMM, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        U[t] = pr.u53(r[0], r[1])
    return U


def sample(trans, filt, last_row, U):
    """Rows T-2 .. 0 from the given last row and uniforms; also the distance of each uniform to the nearest CDF
    entry of the column it was drawn from (a mismatch with the device is only expected where that is tiny)."""
    T, K = np.asarray(filt).shape
    N = last_row.shape[0]
    paths = np.empty((T, N), np.int64)
    gap = np.full((T, N), np.inf)
    paths[-1] = last_row
    for t in range(T - 2, -1, -1):
        C = column_cdfs(trans, filt[t])
        col = C[paths[t + 1]]                                             # (N, K)
        u = np.asarray(U[t], LD)
        paths[t] = np.minimum((col < u[:, None]).sum(axis=1), K - 1)
        gap[t] = np.abs(col - u[:, None]).min(axis=1).astype(float)
    return paths, gap


def two_slice(trans, pred, filt, smth):
    """xi[t, i, j] = P(x_t = i, x_{t+1} = j | y_{0:T-1}) = filt_t[i] P[i, j] smth_{t+1}[j] / pred_{t+1}[j]."""
    P = np.asarray(trans, LD)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(pred[1:] > 0, smth[1:] / pred[1:], 0)                 # (T-1, K)
    return filt[:-1, :, None] * P[None] * r[:, None, :]
