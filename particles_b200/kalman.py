"""Linear-Gaussian state-space models and the Kalman filter / RTS smoother of ``particles/kalman.py`` on the device.

* ``MVLinearGauss``, ``MVLinearGauss_Guarniero_etal`` and ``LinearGauss`` (kalman.py:296-452) are state-space models
  over device arrays; the stock ones run on the fused kernels (``state_space_models.fused_spec``).
* ``Kalman`` (kalman.py:459-517) computes the exact predictive and filtering distributions, the log-likelihood
  factors ``logpyt`` and the smoothing distributions with csrc/smcb_kalman.cu: ``filter()`` is one launch over every
  remaining row, ``next()`` one launch per row, ``smoother()`` one launch.  Results are CUDA tensors with ``kf.t``
  rows on their time axis (sum the log-likelihood with ``kf.logpyt.sum()``).  ``pred``, ``filt`` and ``smth`` are
  sequences: ``kf.filt[3].mean`` and ``kf.pred[-1].cov`` are row t's ``MeanAndCov``; ``kf.filt.mean`` and
  ``kf.filt.cov`` are the stacked (T, dx) and (T, dx, dx) tensors.  The reference's means are (dx,) or (1, dx)
  depending on the shape of its data rows; here they are always (T, dx).  dx and dy are at most 32
  (``_lib.KALMAN_MAX_D``): above that ``Kalman`` raises ``NotImplementedError``.
* Batches, for ``Kalman`` only: ``MVLinearGauss`` with any of F, G, covX, covY, cov0 given (B, r, c) or mu0 (B, dx)
  (the others shared), or ``LinearGauss`` with any of rho, sigmaX, sigmaY, sigma0 an array or tensor of more than one
  element (a one-element array stays a scalar model; a batch of one is a 3-D ``MVLinearGauss``), is B models run
  side by side: every result gains a leading B.  Data (B, T, dy) is per model; any other data is shared by all.
  ``PX0``, ``PX``, ``PY``, the proposals, ``logeta``, ``simulate`` and ``fused_spec`` refuse a batched model.
* ``MeanAndCov``, ``predict_step``, ``filter_step``, ``filter_step_asarray`` and ``smoother_step`` are the
  reference's single steps with torch operations on CUDA tensors (N predictive means at once, as there).

One deliberate difference: where S = G P G' + covY (or P_{t+1} in the smoother) is not positive definite, the
reference raises; ``Kalman`` cannot without a host read, so that model's rows are NaN from that step on.
"""
import collections
import ctypes as C

import numpy as np
import torch

from . import _lib
from . import distributions as dists
from . import state_space_models as ssms
from .device import as_device, context

_HALFLOG2PI = 0.5 * np.log(2.0 * np.pi)          # == scipy.stats.norm's _norm_pdf_logC in fp64


def _h(y):
    return np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y, dtype=np.float64).reshape(-1)


def _host(v):
    return np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=np.float64)


# ----------------------------------------------------------------------------------------------------------------
# single steps (kalman.py:157-290) on CUDA tensors
# ----------------------------------------------------------------------------------------------------------------
MeanAndCov = collections.namedtuple("MeanAndCov", "mean cov")


def _mat(a):
    x = as_device(a)
    return x.reshape(1, 1) if x.ndim < 2 else x


def predict_step(F, covX, filt):
    """kalman.py:169-193: the predictive distribution at t from the filtering one at t - 1; ``filt.mean`` (dx,) or
    (N, dx)."""
    F, covX = _mat(F), _mat(covX)
    return MeanAndCov(mean=torch.matmul(as_device(filt.mean), F.T), cov=(F @ _mat(filt.cov)) @ F.T + covX)


def filter_step(G, covY, pred, yt):
    """kalman.py:196-229: (filtering ``MeanAndCov``, log-density of y_t given the past)."""
    G, covY = _mat(G), _mat(covY)
    pm, pc, yt = as_device(pred.mean), _mat(pred.cov), as_device(yt)
    dpm = torch.matmul(pm, G.T)
    dpc = (G @ pc) @ G.T + covY
    if covY.shape[0] == 1:                                    # scipy.stats.norm.logpdf(yt, dpm, sqrt(dpc))
        scale = torch.sqrt(dpc)
        z = (yt - dpm) / scale
        logpyt = -(z * z) / 2.0 - _HALFLOG2PI - torch.log(scale)
    else:                                                     # distributions.MvNormal.logpdf
        L = torch.linalg.cholesky(dpc)
        xc = yt - dpm
        zt = xc.T if xc.ndim == 2 else xc[:, None]
        z = torch.linalg.solve_triangular(L, zt, upper=False)
        z = z if xc.ndim == 2 else z[:, 0]
        logpyt = -0.5 * torch.sum(z * z, dim=0) - torch.sum(torch.log(torch.diagonal(L))) - dpc.shape[-1] * _HALFLOG2PI
    gain = torch.cholesky_solve((pc @ G.T).T, torch.linalg.cholesky(dpc)).T
    residual = yt - dpm
    return MeanAndCov(mean=pm + torch.matmul(residual, gain.T), cov=pc - (gain @ G) @ pc), logpyt


def filter_step_asarray(G, covY, pred, yt):
    """kalman.py:232-263: ``filter_step`` for N predictive means (N,) or (N, dx).  As in the reference, a mean of
    shape (N,) comes back (N, 1)."""
    pm = as_device(pred.mean)
    return filter_step(G, covY, MeanAndCov(mean=pm[:, None] if pm.ndim == 1 else pm, cov=pred.cov), yt)


def smoother_step(F, filt, next_pred, next_smth):
    """kalman.py:266-290: the smoothing distribution at t."""
    F = _mat(F)
    fc, pc = _mat(filt.cov), _mat(next_pred.cov)
    J = torch.cholesky_solve((fc @ F.T).T, torch.linalg.cholesky(pc)).T
    cov = fc + (J @ (_mat(next_smth.cov) - pc)) @ J.T
    mean = as_device(filt.mean) + torch.matmul(as_device(next_smth.mean) - as_device(next_pred.mean), J.T)
    return MeanAndCov(mean=mean, cov=cov)


# ----------------------------------------------------------------------------------------------------------------
# models (kalman.py:296-452)
# ----------------------------------------------------------------------------------------------------------------
def _batched_mv(F, G, covX, covY, mu0, cov0):
    return any(np.ndim(v) == 3 for v in (F, G, covX, covY, cov0) if v is not None) or (
        mu0 is not None and np.ndim(mu0) == 2)


class MVLinearGauss(ssms.StateSpaceModel):
    """kalman.py:296-361: X_0 ~ N(mu0, cov0); X_t = F X_{t-1} + U_t; Y_t = G X_t + V_t.  A (B, r, c) matrix or a
    (B, dx) mu0 makes a batch of B models (``batch`` = B) for ``Kalman``."""

    batch = None

    def __init__(self, F=None, G=None, covX=None, covY=None, mu0=None, cov0=None):
        if _batched_mv(F, G, covX, covY, mu0, cov0):
            self._init_batch(F, G, covX, covY, mu0, cov0)
            return
        self.covX, self.covY = np.atleast_2d(covX), np.atleast_2d(covY)
        self.dx, self.dy = self.covX.shape[0], self.covY.shape[0]
        self.mu0 = np.zeros(self.dx) if mu0 is None else mu0
        self.cov0 = self.covX if cov0 is None else np.atleast_2d(cov0)
        self.F = np.eye(self.dx) if F is None else np.atleast_2d(F)
        self.G = np.eye(self.dy, self.dx) if G is None else np.atleast_2d(G)
        assert self.F.shape == (self.dx, self.dx) and self.G.shape == (self.dy, self.dx)

    def _init_batch(self, F, G, covX, covY, mu0, cov0):
        def mat(v):
            v = _host(v)
            return v if v.ndim == 3 else np.atleast_2d(v)

        self.covX, self.covY = mat(covX), mat(covY)
        self.dx, self.dy = self.covX.shape[-1], self.covY.shape[-1]
        self.mu0 = np.zeros(self.dx) if mu0 is None else _host(mu0)
        self.cov0 = self.covX if cov0 is None else mat(cov0)
        self.F = np.eye(self.dx) if F is None else mat(F)
        self.G = np.eye(self.dy, self.dx) if G is None else mat(G)
        dx, dy = self.dx, self.dy
        want = {"F": (dx, dx), "G": (dy, dx), "covX": (dx, dx), "covY": (dy, dy), "mu0": (dx,), "cov0": (dx, dx)}
        sizes = set()
        for name, shape in want.items():
            v = getattr(self, name)
            if v.shape != shape:
                if v.shape[1:] != shape:
                    raise ValueError(f"MVLinearGauss: {name} has shape {v.shape}; expected {shape} or (B,) + {shape}")
                sizes.add(v.shape[0])
        if len(sizes) != 1:
            raise ValueError(f"MVLinearGauss: batched parameters disagree on B: {sorted(sizes)}")
        self.batch = sizes.pop()

    def _unbatched(self, what):
        if self.batch is not None:
            raise ValueError(f"{type(self).__name__}.{what}: a batch of B = {self.batch} models runs in "
                             "kalman.Kalman only")

    def _dev(self, M):
        return as_device(np.ascontiguousarray(M))

    def simulate(self, T):
        self._unbatched("simulate")
        return ssms.StateSpaceModel.simulate(self, T)

    def PX0(self):
        self._unbatched("PX0")
        return dists.MvNormal(loc=self.mu0, cov=self.cov0)

    def PX(self, t, xp):
        self._unbatched("PX")
        return dists.MvNormal(loc=xp @ self._dev(self.F.T), cov=self.covX)

    def PY(self, t, xp, x):
        self._unbatched("PY")
        return dists.MvNormal(loc=x @ self._dev(self.G.T), cov=self.covY)

    # Kalman update with a common predictive covariance (kalman.py:196-229, 232-262)
    def _gain(self, pred_cov):
        dpc = self.G @ pred_cov @ self.G.T + self.covY
        gain = np.linalg.solve(dpc, (pred_cov @ self.G.T).T).T
        fcov = pred_cov - gain @ self.G @ pred_cov
        return dpc, gain, fcov

    def proposal0(self, data):
        self._unbatched("proposal0")
        dpc, gain, fcov = self._gain(self.cov0)
        resid = _h(data[0]) - self.mu0 @ self.G.T
        return dists.MvNormal(loc=self.mu0 + resid @ gain.T, cov=fcov)

    def proposal(self, t, xp, data):
        self._unbatched("proposal")
        dpc, gain, fcov = self._gain(self.covX)
        pm = xp @ self._dev(self.F.T)
        resid = as_device(_h(data[t])) - pm @ self._dev(self.G.T)
        return dists.MvNormal(loc=pm + resid @ self._dev(gain.T), cov=fcov)

    def logeta(self, t, x, data):
        self._unbatched("logeta")
        dpc, _, _ = self._gain(self.covX)
        pm = x @ self._dev(self.F.T)
        return dists.MvNormal(loc=pm @ self._dev(self.G.T), cov=dpc).logpdf(_h(data[t + 1]))


class MVLinearGauss_Guarniero_etal(MVLinearGauss):
    """kalman.py:364-394: F_ij = alpha^(1 + |i - j|), G = covX = covY = cov0 = I."""

    def __init__(self, alpha=0.4, dx=2):
        F = np.empty((dx, dx))
        for i in range(dx):
            for j in range(dx):
                F[i, j] = alpha ** (1 + abs(i - j))
        MVLinearGauss.__init__(self, F=F, G=np.eye(dx), covX=np.eye(dx), covY=np.eye(dx))


def _multi(v):
    return isinstance(v, (np.ndarray, torch.Tensor)) and int(np.prod(v.shape)) > 1


class LinearGauss(MVLinearGauss):
    """kalman.py:397-452.  rho, sigmaX, sigmaY or sigma0 given as an array or tensor of B > 1 elements (the others
    scalars or B elements) makes a batch of B models for ``Kalman``; sigma0 = None is then sigmaX / sqrt(1 - rho^2)
    per model."""
    default_params = {"sigmaY": 0.2, "rho": 0.9, "sigmaX": 1.0, "sigma0": None}

    def __init__(self, **kwargs):
        ssms.StateSpaceModel.__init__(self, **kwargs)
        if any(_multi(v) for v in (self.rho, self.sigmaX, self.sigmaY, self.sigma0)):
            given = [_host(v).reshape(-1) for v in (self.rho, self.sigmaX, self.sigmaY, self.sigma0) if v is not None]
            try:
                rho, sX, sY, *s0 = np.broadcast_arrays(*given)
            except ValueError:
                raise ValueError("LinearGauss: rho, sigmaX, sigmaY and sigma0 must have one or B elements each")
            s0 = sX / np.sqrt(1.0 - rho ** 2) if self.sigma0 is None else s0[0]
            self.rho, self.sigmaX, self.sigmaY, self.sigma0 = (np.ascontiguousarray(v) for v in (rho, sX, sY, s0))
            c = lambda v: np.ascontiguousarray(v[:, None, None])         # noqa: E731
            MVLinearGauss.__init__(self, F=c(rho), G=np.ones((1, 1)), covX=c(sX ** 2), covY=c(sY ** 2),
                                   cov0=c(s0 ** 2))
            return
        if self.sigma0 is None:
            self.sigma0 = self.sigmaX / np.sqrt(1.0 - self.rho ** 2)
        MVLinearGauss.__init__(self, F=self.rho, G=1.0, covX=self.sigmaX ** 2,
                               covY=self.sigmaY ** 2, cov0=self.sigma0 ** 2)

    def PX0(self):
        self._unbatched("PX0")
        return dists.Normal(scale=self.sigma0)

    def PX(self, t, xp):
        self._unbatched("PX")
        return dists.Normal(loc=self.rho * xp, scale=self.sigmaX)

    def PY(self, t, xp, x):
        self._unbatched("PY")
        return dists.Normal(loc=x, scale=self.sigmaY)

    def proposal0(self, data):
        self._unbatched("proposal0")
        sig2post = 1.0 / (1.0 / self.sigma0 ** 2 + 1.0 / self.sigmaY ** 2)
        mupost = sig2post * (_h(data[0])[0] / self.sigmaY ** 2)
        return dists.Normal(loc=mupost, scale=np.sqrt(sig2post))

    def proposal(self, t, xp, data):
        self._unbatched("proposal")
        sig2post = 1.0 / (1.0 / self.sigmaX ** 2 + 1.0 / self.sigmaY ** 2)
        mupost = sig2post * (self.rho * xp / self.sigmaX ** 2 + _h(data[t])[0] / self.sigmaY ** 2)
        return dists.Normal(loc=mupost, scale=np.sqrt(sig2post))

    def logeta(self, t, x, data):
        self._unbatched("logeta")
        law = dists.Normal(loc=self.rho * x, scale=np.sqrt(self.sigmaX ** 2 + self.sigmaY ** 2))
        return law.logpdf(_h(data[t + 1])[0])


# ----------------------------------------------------------------------------------------------------------------
# the Kalman filter / smoother (kalman.py:459-517)
# ----------------------------------------------------------------------------------------------------------------
_PARAMS = ("F", "G", "covX", "covY", "mu0", "cov0")


def model_layout(ssm):
    """(dx, dy, B, {name: per-model shape}) of any object with F, G, covX, covY, mu0, cov0 (duck typing); B is
    None for one model.  Reads shapes only.  ``NotImplementedError`` above ``_lib.KALMAN_MAX_D``."""
    shp = {k: tuple(np.shape(getattr(ssm, k))) for k in _PARAMS}
    dx = shp["covX"][-1] if shp["covX"] else 1
    dy = shp["covY"][-1] if shp["covY"] else 1
    if max(dx, dy) > _lib.KALMAN_MAX_D:
        raise NotImplementedError(f"Kalman: dx = {dx}, dy = {dy}; the device filter has a bound of "
                                  f"{_lib.KALMAN_MAX_D} on both")
    want = {"F": (dx, dx), "G": (dy, dx), "covX": (dx, dx), "covY": (dy, dy), "mu0": (dx,), "cov0": (dx, dx)}
    sizes = set()
    for k, w in want.items():
        s = shp[k]
        if len(s) == len(w) + 1 and s[1:] == w:
            sizes.add(s[0])
        elif not (s == w or (len(s) < len(w) and int(np.prod(s)) == int(np.prod(w)))):
            raise ValueError(f"Kalman: {k} has shape {s}; expected {w} or (B,) + {w}")
    if len(sizes) > 1:
        raise ValueError(f"Kalman: batched parameters disagree on B: {sorted(sizes)}")
    return dx, dy, (sizes.pop() if sizes else None), want


def data_layout(data, B, dy):
    """(per_model, T) of ``data``: (B, T, dy) arrays or tensors are per model when the model is a batch of B;
    anything else -- (T,), (T, dy), a list of rows -- is one series shared by every model."""
    if isinstance(data, (np.ndarray, torch.Tensor)):
        if B is not None and data.ndim == 3:
            if tuple(data.shape[0:1]) + tuple(data.shape[2:]) != (B, dy):
                raise ValueError(f"Kalman: per-model data must be (B, T, dy) = ({B}, T, {dy}); got {tuple(data.shape)}")
            return True, int(data.shape[1])
        return False, int(data.shape[0]) if data.ndim else 0
    return False, len(data)


def data_rows(data, per_model, t0, t1, dy):
    """Rows [t0, t1) of ``data`` as an array of shape (B or 1, t1 - t0, dy): a NumPy array, or a tensor when the
    data holds tensors."""
    n = t1 - t0
    if per_model:
        x = data[:, t0:t1]
    elif isinstance(data, (np.ndarray, torch.Tensor)):
        x = data[t0:t1]
    else:
        items = data[t0:t1]
        if any(isinstance(v, torch.Tensor) for v in items):
            x = torch.cat([as_device(v).reshape(-1) for v in items]) if items else torch.empty(0)
        else:
            x = np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in items])
    size = int(np.prod(x.shape))
    if size != (x.shape[0] if per_model else 1) * n * dy:
        raise ValueError(f"Kalman: data rows [{t0}, {t1}) do not hold {dy} value(s) each")
    return x.reshape(-1, n, dy)


class _Seq:
    """``pred``, ``filt`` or ``smth``: stacked ``mean`` (T, dx) and ``cov`` (T, dx, dx) (a leading B for a batch);
    ``seq[t]`` is row t's ``MeanAndCov``."""

    def __init__(self, mean, cov, batched):
        self.mean, self.cov, self._batched = mean, cov, batched

    def __len__(self):
        return int(self.mean.shape[-2])

    def __getitem__(self, t):
        if self._batched:
            return MeanAndCov(mean=self.mean[:, t], cov=self.cov[:, t])
        return MeanAndCov(mean=self.mean[t], cov=self.cov[t])

    def __iter__(self):
        return (self[t] for t in range(len(self)))


class Kalman:
    """kalman.py:459-517: Kalman filter and smoother of one linear-Gaussian model or a batch of B (see the module
    docstring).  ``ssm`` is any object with F, G, covX, covY, mu0 and cov0; ``data`` a list of rows, a (T,) or
    (T, dy) array or tensor, or (B, T, dy) for a batch.  ``next()`` reads ``data[kf.t]``, so data appended between
    steps is picked up; storage grows by doubling."""

    def __init__(self, ssm=None, data=None):
        self.ssm = ssm
        self.data = data
        self.dx, self.dy, self.B, want = model_layout(ssm)
        self._nb = 1 if self.B is None else self.B
        self._per_model, _ = data_layout(data, self.B, self.dy)
        self._p = {}
        for k in _PARAMS:
            v = getattr(ssm, k)
            v = as_device(v if isinstance(v, torch.Tensor) else _host(v))
            batched = v.ndim == len(want[k]) + 1
            self._p[k] = (v.reshape((-1,) + want[k]).contiguous(), int(np.prod(want[k])) if batched else 0)
        self._t, self._cap = 0, 0
        self._dev = self._p["F"][0].device
        self._buf = self._alloc(0)

    # -- storage ------------------------------------------------------------------------------------------------
    @property
    def t(self):
        return self._t

    def _alloc(self, cap):
        nb, dx, dev = self._nb, self.dx, self._dev
        e = lambda *s: torch.empty(s, dtype=torch.float64, device=dev)       # noqa: E731
        return {"pred_mean": e(nb, cap, dx), "pred_cov": e(nb, cap, dx, dx), "filt_mean": e(nb, cap, dx),
                "filt_cov": e(nb, cap, dx, dx), "logpyt": e(nb, cap),
                "y": e(nb if self._per_model else 1, cap, self.dy)}

    def _reserve(self, rows):
        if rows <= self._cap:
            return
        cap = max(rows, 2 * self._cap, 16)
        new = self._alloc(cap)
        if self._t:
            for k, v in new.items():
                v[:, :self._t] = self._buf[k][:, :self._t]
        self._buf, self._cap = new, cap

    def _view(self, k):
        v = self._buf[k][:, :self._t]
        return v if self.B is not None else v[0]

    @property
    def logpyt(self):
        return self._view("logpyt")

    @property
    def pred(self):
        return _Seq(self._view("pred_mean"), self._view("pred_cov"), self.B is not None)

    @property
    def filt(self):
        return _Seq(self._view("filt_mean"), self._view("filt_cov"), self.B is not None)

    # -- kernels --------------------------------------------------------------------------------------------------
    def _launch(self, method, **kw):
        d = _lib.KalmanDesc()
        d.method, d.dx, d.dy, d.B, d.ld = method, self.dx, self.dy, self._nb, self._cap
        for k, (v, stride) in self._p.items():
            setattr(d, k, v.data_ptr())
            setattr(d, k + "_stride", stride)
        d.y_stride = self._cap * self.dy if self._per_model else 0
        for k, v in self._buf.items():
            setattr(d, k, v.data_ptr())
        for k, v in kw.items():
            setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        ctx = context(self._dev)
        _lib.check(ctx.lib.smcb_kalman(ctx.handle, C.byref(d)))

    def _advance(self, t1):
        t0 = self._t
        self._reserve(t1)
        self._buf["y"][:, t0:t1] = as_device(data_rows(self.data, self._per_model, t0, t1, self.dy))
        self._launch(_lib.KALMAN_FILTER, t0=t0, t1=t1)
        self._t = t1

    def _data_len(self):
        return data_layout(self.data, self.B, self.dy)[1]

    # -- the reference's surface ----------------------------------------------------------------------------------
    def __next__(self):
        if self._t >= self._data_len():
            raise StopIteration
        self._advance(self._t + 1)

    def next(self):
        return self.__next__()

    def __iter__(self):
        return self

    def filter(self):
        """Forward recursion over every data point not yet processed, in one launch."""
        n = self._data_len()
        if n > self._t:
            self._advance(n)

    def smoother(self):
        """Backward recursion over the rows filtered so far, in one launch: ``smth``.  Filters first if no step has
        been taken."""
        if self._t == 0:
            self.filter()
        if self._t == 0:
            raise IndexError("Kalman.smoother: there is no data to smooth")
        nb, cap, dx = self._nb, self._cap, self.dx
        sm = torch.empty(nb, cap, dx, dtype=torch.float64, device=self._dev)
        sc = torch.empty(nb, cap, dx, dx, dtype=torch.float64, device=self._dev)
        self._launch(_lib.KALMAN_SMOOTH, t1=self._t, smth_mean=sm, smth_cov=sc)
        sm, sc = sm[:, :self._t], sc[:, :self._t]
        self.smth = _Seq(sm if self.B is not None else sm[0], sc if self.B is not None else sc[0], self.B is not None)
