"""Hidden Markov models (particles/hmm.py:107-268) on the device: ``HMM``, ``GaussianHMM`` and ``BaumWelch``.

``HMM`` is a finite-state ``StateSpaceModel``: ``PX0`` / ``PX`` are ``Categorical`` laws, so ``SMC`` and
``simulate`` run it on the plugin path like any user model.  ``BaumWelch`` computes the exact filter, predictive,
likelihood factors, smoother and posterior trajectory draws with csrc/smcb_hmm.cu: a forward over any number of
rows is one launch, the backward pass one launch, and ``sample`` one launch after the last row's multinomial draw.

Batches: ``trans_mat`` (B, K, K), with ``init_dist`` / ``mus`` / ``sigmas`` (B, K) or shared (K,), makes one
object of B HMMs that ``BaumWelch`` runs together on (B, T) data; every result then has a leading B.  A batched HMM
is for ``BaumWelch`` only.  K is at most 128 (``_lib.HMM_MAX_K``): above it ``BaumWelch`` raises
``NotImplementedError``, while ``SMC`` on such a model still runs on the plugin path.

Results are CUDA tensors whose time axis has length ``bw.t`` -- (T, K) or (T,), (B, T, K) or (B, T) when
batched -- so a call never waits on the host.  Two deliberate differences from the reference: ``pred`` sums over
the previous state in index order (the reference's ``np.matmul`` uses a BLAS order, so the two agree to rounding,
not to the bit), and a trajectory draw whose uniform lies above a column CDF that rounds below 1 takes the last
state instead of failing with an ``IndexError``.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from . import distributions as dists
from . import resampling as rs
from . import state_space_models as ssms
from .device import as_device, context

_LOG_SQRT_2PI = np.log(np.sqrt(2 * np.pi))       # scipy.stats.norm's _norm_pdf_logC


class HMM(ssms.StateSpaceModel):
    """hmm.py:107-131: subclass it and define ``PY``.  Parameters become CUDA fp64 tensors."""

    default_params = {"init_dist": None, "trans_mat": None}

    def __init__(self, **kwargs):
        ssms.StateSpaceModel.__init__(self, **kwargs)
        if self.trans_mat is None:
            raise ValueError("Transition Matrix is missing")
        err_msg = "Wrong shape for trans_mat or init_dist"
        tm = as_device(self.trans_mat)
        assert tm.ndim in (2, 3), err_msg
        self.dim = int(tm.shape[-2])
        self.batch = int(tm.shape[0]) if tm.ndim == 3 else None
        if self.init_dist is None:
            self.init_dist = np.full(self.dim, 1.0 / self.dim)
        init = as_device(self.init_dist)
        assert tuple(tm.shape[-2:]) == (self.dim, self.dim), err_msg
        assert tuple(init.shape) == (self.dim,) or (self.batch is not None
                                                    and tuple(init.shape) == (self.batch, self.dim)), err_msg
        self.trans_mat, self.init_dist = tm, init

    def _unbatched(self, what):
        if self.batch is not None:
            raise ValueError(f"{type(self).__name__}.{what}: a batched HMM (B = {self.batch}) runs in BaumWelch only")

    def PX0(self):
        self._unbatched("PX0")
        return dists.Categorical(p=self.init_dist)

    def PX(self, t, xp):
        self._unbatched("PX")
        return dists.Categorical(p=self.trans_mat[as_device(xp, dtype=torch.int64), :])

    def logft(self, data, t0=0):
        """The (T, K) table of ``PY(t0 + i, None, k).logpdf(data[i])``: one call of the user's ``PY`` per step, on
        CUDA tensors.  Override it with a vectorised evaluation (``GaussianHMM`` does); a batched HMM needs one."""
        if self.batch is not None:
            raise NotImplementedError(f"{type(self).__name__}.logft: a batched HMM needs a vectorised logft "
                                      "(GaussianHMM has one)")
        ks = torch.arange(self.dim, dtype=torch.int64, device=self.trans_mat.device)
        rows = [as_device(self.PY(t0 + i, None, ks).logpdf(data[i:i + 1])).reshape(self.dim)
                for i in range(data.shape[0])]
        if not rows:
            return torch.empty(0, self.dim, dtype=torch.float64, device=ks.device)
        return torch.stack(rows)


class GaussianHMM(HMM):
    r"""hmm.py:134-141: :math:`Y_t | X_t = k \sim N(\mu_k, \sigma_k^2)`."""

    default_params = {"mus": None, "sigmas": None}
    default_params.update(HMM.default_params)

    def __init__(self, **kwargs):
        HMM.__init__(self, **kwargs)
        if self.mus is not None and self.sigmas is not None:
            sig = self.sigmas.detach().cpu().numpy() if isinstance(self.sigmas, torch.Tensor) else self.sigmas
            self._log_sigmas = as_device(np.log(np.asarray(sig, dtype=np.float64)))    # NumPy's log, as scipy
            self.mus, self.sigmas = as_device(self.mus), as_device(self.sigmas)

    def PY(self, t, xp, x):
        return dists.Normal(loc=self.mus[x], scale=self.sigmas[x])

    def logft(self, data, t0=0):
        """scipy.stats.norm.logpdf over every (t, k) at once, in its operation order:
        z = (y - mu) / sigma, -z**2 / 2 - log(sqrt(2 pi)) - log(sigma).  ``data`` (T,), or (B, T) when batched."""
        y = as_device(data)
        mu, sig, lsig = self.mus, self.sigmas, self._log_sigmas
        if y.ndim == 1:
            z = (y[:, None] - mu[None, :]) / sig[None, :]
            return -(z * z) / 2.0 - _LOG_SQRT_2PI - lsig[None, :]
        mu, sig, lsig = (v[None, :] if v.ndim == 1 else v for v in (mu, sig, lsig))
        z = (y[:, :, None] - mu[:, None, :]) / sig[:, None, :]
        return -(z * z) / 2.0 - _LOG_SQRT_2PI - lsig[:, None, :]


class BaumWelch:
    """hmm.py:143-268: Baum-Welch filter, smoother and posterior trajectory sampler.

    ``pred``, ``filt``, ``logft``, ``logpyt`` (and ``smth`` after ``backward``) are CUDA tensors with ``bw.t``
    rows along their time axis.  ``next()`` reads ``data[bw.t]``, so data appended between steps is picked up;
    storage grows by doubling.  ``data``: a list of scalars or of (1,) tensors, a (T,) array or tensor, or (B, T)
    for a batched HMM."""

    def __init__(self, hmm=None, data=None):
        self.hmm = hmm
        self.data = data
        K = hmm.dim
        if K > _lib.HMM_MAX_K:
            raise NotImplementedError(f"BaumWelch: K = {K} states is above the device bound of {_lib.HMM_MAX_K} "
                                      "(SMC on this model still runs on the plugin path)")
        self.K, self.B = K, hmm.batch
        self._nb = 1 if hmm.batch is None else hmm.batch
        self._trans = hmm.trans_mat.contiguous()
        self._init = hmm.init_dist.contiguous()
        self._t, self._cap = 0, 0
        dev = self._trans.device
        self._pred, self._filt, self._logft = (torch.empty(self._nb, 0, K, dtype=torch.float64, device=dev)
                                               for _ in range(3))
        self._logpyt = torch.empty(self._nb, 0, dtype=torch.float64, device=dev)

    # -- storage ------------------------------------------------------------------------------------------------
    @property
    def t(self):
        return self._t

    def _view(self, buf):
        v = buf[:, :self._t]
        return v if self.B is not None else v[0]

    pred = property(lambda self: self._view(self._pred))
    filt = property(lambda self: self._view(self._filt))
    logft = property(lambda self: self._view(self._logft))
    logpyt = property(lambda self: self._view(self._logpyt))

    def _reserve(self, rows):
        if rows <= self._cap:
            return
        cap = max(rows, 2 * self._cap, 16)
        nb, K, dev, t = self._nb, self.K, self._trans.device, self._t

        def grow(old, shape):
            new = torch.empty(shape, dtype=torch.float64, device=dev)
            if t:
                new[:, :t] = old[:, :t]
            return new

        self._pred = grow(self._pred, (nb, cap, K))
        self._filt = grow(self._filt, (nb, cap, K))
        self._logft = grow(self._logft, (nb, cap, K))
        self._logpyt = grow(self._logpyt, (nb, cap))
        self._cap = cap

    # -- data -----------------------------------------------------------------------------------------------------
    def _data_len(self):
        d = self.data
        return int(d.shape[-1]) if isinstance(d, (np.ndarray, torch.Tensor)) else len(d)

    def _rows(self, t0, t1):
        """data[t0:t1] as a (nb, t1 - t0) CUDA fp64 tensor."""
        d = self.data
        if isinstance(d, (np.ndarray, torch.Tensor)):
            x = as_device(d[..., t0:t1])
        else:
            items = d[t0:t1]
            if any(isinstance(v, torch.Tensor) for v in items):
                x = torch.cat([as_device(v).reshape(-1) for v in items])
            else:
                x = as_device(np.asarray(items, dtype=np.float64).reshape(-1))
        return x.reshape(self._nb, t1 - t0)

    # -- kernels --------------------------------------------------------------------------------------------------
    def _launch(self, method, **kw):
        d = _lib.HmmDesc()
        d.method, d.K, d.B, d.ld = method, self.K, self._nb, self._cap
        d.trans = self._trans.data_ptr()
        d.trans_stride = self.K * self.K if self._trans.ndim == 3 else 0
        d.init = self._init.data_ptr()
        d.init_stride = self.K if self._init.ndim == 2 else 0
        d.logft, d.pred, d.filt, d.logpyt = (b.data_ptr() for b in (self._logft, self._pred, self._filt,
                                                                      self._logpyt))
        for k, v in kw.items():
            setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        ctx = context(self._trans.device)
        _lib.check(ctx.lib.smcb_hmm(ctx.handle, C.byref(d)))

    def _advance(self, t1):
        """Forward rows [t, t1): the emission table of the new rows, then one launch."""
        t0 = self._t
        self._reserve(t1)
        y = self._rows(t0, t1)
        lf = self.hmm.logft(y[0] if self.B is None else y, t0)
        self._logft[:, t0:t1] = as_device(lf).reshape(self._nb, t1 - t0, self.K)
        self._launch(_lib.HMM_FORWARD, t0=t0, t1=t1)
        self._t = t1

    # -- the reference's surface ----------------------------------------------------------------------------------
    def __next__(self):
        if self._t >= self._data_len():
            raise StopIteration
        self._advance(self._t + 1)

    def next(self):
        return self.__next__()

    def __iter__(self):
        return self

    def forward(self):
        """Forward recursion over every data point not yet processed (one launch): ``filt``, ``pred``,
        ``logpyt`` and ``logft`` then have ``len(data)`` rows."""
        n = self._data_len()
        if n > self._t:
            self._advance(n)

    def backward(self):
        """Backward recursion: ``smth``, the marginal smoothing probabilities of the rows filtered so far.  Runs
        ``forward`` first only if no step has been taken."""
        if self._t == 0:
            self.forward()
        if self._t == 0:
            raise IndexError("BaumWelch.backward: there is no data to smooth")
        smth = torch.empty(self._nb, self._cap, self.K, dtype=torch.float64, device=self._trans.device)
        self._launch(_lib.HMM_BACKWARD, t1=self._t, smth=smth)
        self.smth = self._view(smth)

    def run(self):
        self.forward()
        self.backward()

    def sample(self, N=1, seed=None, noise=None):
        """N trajectories from the posterior of X_{0:T-1}: int64 (T, N), or (B, T, N).  The last row is
        ``resampling.multinomial(filt[T-1], M=N)`` (sorted), the rows before it one device launch.
        ``seed`` re-keys the draws; ``noise={"last": sorted uniforms (N,) or (B, N), "U": (T-1, N) or
        (B, T-1, N)}`` injects them (U[t, n] is the uniform of trajectory n at step t)."""
        if self._t == 0:
            self.forward()
        T, nb, N = self._t, self._nb, int(N)
        dev = self._trans.device
        nz = noise or {}
        if seed is not None:
            context(dev).seed(seed)
        paths = torch.empty(nb, T, N, dtype=torch.int64, device=dev)
        last = nz.get("last")
        if last is not None:
            last = as_device(last).reshape(nb, N)
        for b in range(nb):
            W = self._filt[b, T - 1].clone()                # the resampling kernels want 16-byte aligned rows
            paths[b, T - 1] = rs.multinomial(W, M=N) if last is None else rs.inverse_cdf(last[b], W)
        U = nz.get("U")
        U = None if U is None or T == 1 else as_device(U).reshape(nb, T - 1, N)
        key = int(seed) if seed is not None else int(np.random.randint(0, 2 ** 63, dtype=np.int64))
        self._launch(_lib.HMM_SAMPLE, t1=T, N=N, seed=key & (2 ** 64 - 1), U=0 if U is None else U, paths=paths)
        return paths if self.B is not None else paths[0]
