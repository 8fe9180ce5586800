"""Single-run variance estimators -- particles/variance_estimators.py (Chan & Lai 2013; Lee & Whiteley 2018; Olsson &
Douc 2019) on the device.

``var_estimate(W, phi_x, B)`` is  sum_b (sum_{m: B_m = b} W_m (phi_m - m))^2  with m = sum W phi / sum W, and zeros
whenever B[0] == B[-1] (also for an unsorted B, as the reference).  The collectors keep the reference's names,
signatures and summary names:

* ``Var(phi=None)``: that estimate for the Eve indices B_t = B_{t-1}[A_t] (B_0 = arange(N)); ``phi`` is called on the
  CUDA tensor ``smc.X`` and returns (N,) or (N, k); the summary is a float, or a (k,) array.
* ``Var_logLt()``:  sum_b (sum_{B_m = b} W_m)^2, the variance estimate of log L_t.
* ``Lag_based_var(phi=None)``: a list whose element i is the estimate for the Eve indices i steps back, from
  ``smc.hist.compute_trajectories()`` (needs ``store_history=k``).

Every estimate runs through csrc/smcb_variance.cu.  It reduces a sorted row of Eve indices, whose branches are
contiguous runs: every inverse-CDF scheme (multinomial, stratified, systematic), ``ssp`` and ``idiotic`` give
non-decreasing ancestors, so the rows of a run using them stay sorted.  For any other scheme the rows are first put
in order by a stable sort, and the B[0] == B[-1] rule is decided on the rows as they were.  On the fused path the
Eve update reads the step's resampling flag on the device: ``Var`` and ``Var_logLt`` keep ``SMC.run()`` free of
host syncs, and their rows reach the host once per run.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from . import collectors as col
from .device import as_device, context

# schemes whose ancestors are non-decreasing: Eve rows stay sorted
SORTED_SCHEMES = ("multinomial", "stratified", "systematic", "ssp", "idiotic")


def _as_phi(v, N):
    """phi's (N,) or (N, k) output -> ((N, k) contiguous fp64 on the device, vector?)."""
    v = as_device(v)
    if v.ndim == 0 or v.ndim > 2 or v.shape[0] != N:
        raise ValueError(f"phi must return an array of shape (N,) or (N, k) with N = {N}, got {tuple(v.shape)}")
    return (v.reshape(N, 1) if v.ndim == 1 else v).contiguous(), v.ndim > 1


class _Sums:
    """The device buffers of one estimator: scratch, the sticky per-row "not sorted" flags and, for an Eve tracker,
    the ping-pong pair of rows and its parity word."""

    def __init__(self, N, L, k, device, eve=False):
        ctx = context(device)
        self.ctx, self.N, self.L, self.k = ctx, N, L, k
        self.scratch = torch.empty(int(ctx.lib.smcb_variance_scratch_doubles(N, L, k)), dtype=torch.float64,
                                   device=device)
        self.unsorted = torch.zeros(L, dtype=torch.int32, device=device)
        if eve:
            self.B = torch.empty((2, N), dtype=torch.int64, device=device)
            self.B[0] = torch.arange(N, device=device)
            self.parity = torch.zeros(1, dtype=torch.int32, device=device)

    def eve(self, A, rs_flag=None, rs_host=False):
        """B <- B[A] on the device when the step resampled (``rs_flag``: a device double, or the host's flag)."""
        d = self._desc(_lib.VAR_EVE, rs_flag, rs_host)
        d.A = A.data_ptr()
        _lib.check(self.ctx.lib.smcb_variance(self.ctx.handle, C.byref(d)))

    def run(self, mode, lw, B=None, phi=None, rows=None, zero=None, lin_w=False, rs_flag=None, rs_host=False):
        """Enqueue the branch sums of the L rows of B (None: this tracker's Eve row); returns the (L, k) estimates.
        ``rows`` = (lw_rows, phi_rows): per-row permuted copies (L, N) and (L, N, k) of lw and phi."""
        d = self._desc(_lib.VAR_SUMS, rs_flag, rs_host)
        d.mode, d.lin_w = mode, int(lin_w)
        if B is not None:
            d.parity, d.B[0], d.B[1] = None, B.data_ptr(), 0
        d.lw = lw.data_ptr()
        d.phi = phi.data_ptr() if phi is not None else None
        if rows is None:
            d.lw_rows, d.phi_rows, d.row_ld = d.lw, d.phi, 0
        else:
            d.lw_rows, d.row_ld = rows[0].data_ptr(), self.N
            d.phi_rows = rows[1].data_ptr() if rows[1] is not None else None
        d.zero = zero.data_ptr() if zero is not None else None
        out = torch.empty((self.L, self.k), dtype=torch.float64, device=lw.device)
        d.unsorted, d.scratch, d.out = self.unsorted.data_ptr(), self.scratch.data_ptr(), out.data_ptr()
        _lib.check(self.ctx.lib.smcb_variance(self.ctx.handle, C.byref(d)))
        return out

    def _desc(self, method, rs_flag, rs_host):
        d = _lib.VarDesc()
        d.method, d.N, d.k, d.L = method, self.N, self.k, self.L
        d.rs_flag = rs_flag
        d.rs_host = int(bool(rs_host))
        if hasattr(self, "parity"):
            d.parity, d.B[0], d.B[1] = self.parity.data_ptr(), self.B[0].data_ptr(), self.B[1].data_ptr()
        return d

    def check(self, flags):
        if flags.any():
            raise RuntimeError("variance estimate: a row of Eve indices is not sorted (its resampling scheme does "
                               "not give non-decreasing ancestors)")


def _sorted_rows(B, lw, phi):
    """Stable sort of each row of B (L, N); lw and phi permuted alike, and the B[0] == B[-1] rule of the rows as
    given."""
    Bs, idx = torch.sort(B, dim=1, stable=True)
    zero = (B[:, 0] == B[:, -1]).to(torch.uint8)
    return Bs.contiguous(), (lw[idx].contiguous(), None if phi is None else phi[idx].contiguous()), zero


def _row_value(r, vector):
    return r.copy() if vector else float(r[0])


def _estimate(mode, lw, B, phi=None, lin_w=False, sorted_rows=None):
    """The branch sums of the L rows of B (L, N) in one set of launches; returns ((L, k) host array, sums)."""
    L, N = B.shape
    k = 1 if phi is None else phi.shape[1]
    s = _Sums(N, L, k, lw.device)
    if sorted_rows is None:
        sorted_rows = N < 2 or bool((B[:, 1:] >= B[:, :-1]).all())
    if sorted_rows:
        out = s.run(mode, lw, B=B.contiguous(), phi=phi, lin_w=lin_w)
    else:
        Bs, rows, zero = _sorted_rows(B, lw, phi)
        out = s.run(mode, lw, B=Bs, phi=phi, rows=rows, zero=zero, lin_w=lin_w)
    res, flags = out.cpu().numpy(), s.unsorted.cpu().numpy()
    s.check(flags)
    return res


def var_estimate(W, phi_x, B):
    """particles/variance_estimators.py:93-130 on the device: ``W`` (N,) weights (used as given), ``phi_x`` (N,) or
    (N, k), ``B`` (N,) int Eve indices.  Returns a float, or a (k,) array."""
    W = as_device(W)
    N = W.shape[0]
    phi, vector = _as_phi(phi_x, N)
    B = as_device(B, dtype=torch.int64)
    if B.shape != (N,):
        raise ValueError(f"B must have shape ({N},), got {tuple(B.shape)}")
    return _row_value(_estimate(_lib.VAR_CENTRED, W, B.reshape(1, N), phi, lin_w=True)[0], vector)


def _scheme_sorted(smc):
    return getattr(smc, "resampling", None) in SORTED_SCHEMES


class _PhiMixin:
    signature = {"phi": None}

    def test_func(self, x):
        return x if self.phi is None else self.phi(x)


class _EveCollector(col.DeviceRowsMixin, col.Collector):
    """The Eve-index collectors: per step one EVE launch, one set of branch-sum launches and at most one call to
    phi, no host sync; the rows reach ``summary`` in ``_flush``."""
    mode = _lib.VAR_CENTRED

    def _phi(self, X):
        return None, False

    def _step(self, smc, t):
        if smc.fused:
            e = smc._engine
            X = e.X[t & 1]
            X, lw = (X if X.ndim == 1 else X.t()), e.lw[t & 1]
            A, rs_host = e.A, False
            rs_flag = e.summ.data_ptr() + (t * _lib.SUMMARY_STRIDE + 2) * 8 if t > 0 else None
        else:
            X, lw = as_device(smc.X), as_device(smc.wgts.lw).contiguous()
            A, rs_flag, rs_host = smc.A, None, bool(smc.rs_flag) if t > 0 else False
        phi, self._vector = self._phi(X)
        N = lw.shape[0]
        if t == 0 or not hasattr(self, "_sums"):                  # variance_estimators.py:143-147
            self._rows = []
            self._sorted = smc.fused or _scheme_sorted(smc)
            self._sums = _Sums(N, 1, 1 if phi is None else phi.shape[1], lw.device, eve=self._sorted)
            self._B = None if self._sorted else torch.arange(N, device=lw.device)
        elif self._sorted:
            self._sums.eve(A, rs_flag, rs_host)
        elif rs_host:
            self._B = self._B.index_select(0, as_device(A, dtype=torch.int64))
        s = self._sums
        if self._sorted:
            out = s.run(self.mode, lw, phi=phi, rs_flag=rs_flag, rs_host=rs_host)
        else:
            Bs, rows, zero = _sorted_rows(self._B.reshape(1, N), lw, phi)
            out = s.run(self.mode, lw, B=Bs, phi=phi, rows=rows, zero=zero if self.mode == _lib.VAR_CENTRED else None)
        self._rows.append(out[0])

    def _flush(self):
        if hasattr(self, "_sums"):
            flags = self._sums.unsorted.cpu().numpy()
            col.DeviceRowsMixin._flush(self)
            self._sums.check(flags)


class Var(_PhiMixin, _EveCollector):
    """variance_estimators.py:150-169: the estimate of the variance of sum_n W_t^n phi(X_t^n)."""

    def _phi(self, X):
        return _as_phi(self.test_func(X), X.shape[0])


class Var_logLt(_EveCollector):
    """variance_estimators.py:172-179: the estimate of the variance of log L_t."""
    signature = {}
    mode = _lib.VAR_WEIGHTS


class Lag_based_var(_PhiMixin, col.Collector):
    """variance_estimators.py:182-201 (Olsson & Douc 2019): element i of each summary is the estimate for the Eve
    indices at lag i, row T - 1 - i of ``smc.hist.compute_trajectories()`` (``store_history=k``)."""

    def fetch(self, smc):
        B = smc.hist.compute_trajectories()
        lw = col._lw_of(smc)
        phi, vector = _as_phi(self.test_func(as_device(smc.X)), lw.shape[0])
        res = _estimate(_lib.VAR_CENTRED, lw, B, phi, sorted_rows=smc.fused or _scheme_sorted(smc))
        return [_row_value(r, vector) for r in res][::-1]
