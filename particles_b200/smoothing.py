"""Particle history containers (``hist.save(smc)``, core.py:362-363; classes at smoothing.py:151-270) and the
off-line FFBS smoothers of ``ParticleHistory`` (smoothing.py:278-423) on the device.

The reference stores references to ``smc.X / A / wgts`` (it allocates new arrays every step).
The device loop ping-pongs two buffers instead, so a history OWNS what it saves: ``save`` clones
the device arrays (8(d+2) bytes per particle per saved step -- at N = 1e7 keep the window short).

Backward sampling (``backward_sampling_ON2 / _mcmc / _reject / _qmc``): when the transition density is a stock
model's ``PX`` (``state_space_models.transition_spec``) the whole backward pass is ONE kernel launch
(csrc/smcb_smooth.cu; QMC adds the final-time draw); otherwise the same algorithms run with ``fk.logpt`` called on CUDA
tensors, with the library's sampling, CDF and gather kernels underneath.  There is no CPU path.

Two-filter smoothing (``two_filter_smoothing``, O(N^2) and O(N), one-dimensional states) works the same way:
csrc/smcb_twofilter.cu on a stock model's transition, ``fk.logpt`` on CUDA tensors otherwise; ``smoothing_worker``
drives every off-line method as the reference's book scripts do.
"""
import ctypes as C
from collections import deque

import numpy as np
import torch

from . import _lib
from . import resampling as rs
from .device import as_device, context, ptr


def _flat(x):
    """A 1-D particle array as the two-filter kernels read it: (N,) fp64 on the device, element stride kept."""
    x = x if isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float64 else as_device(x)
    return x.reshape(x.shape[0]) if x.ndim > 1 else x


def _own(x):
    return x.clone() if isinstance(x, torch.Tensor) else x


def _np(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


class HilbertOrdersError(NotImplementedError, ValueError):
    """QMC backward sampling of a history that kept no Hilbert orders (not an SQMC run).  A NotImplementedError, and a
    ValueError as the reference's ``_check_h_orders`` raises."""


def _own_weights(w):
    if w.lw is None:
        return rs.Weights()
    return rs.Weights._from_device_stats(w.lw.clone(), w._stats.clone())


def generate_hist_obj(option, smc):
    """smoothing.py:151-161."""
    if option is True:
        return ParticleHistory(smc.fk, smc.qmc)
    elif option is False:
        return None
    elif callable(option):
        return PartialParticleHistory(option)
    elif isinstance(option, int) and option >= 0:
        return RollingParticleHistory(option)
    raise ValueError("store_history: invalid option")


class PartialParticleHistory:
    """smoothing.py:164-178: records the particle system at the times ``func(t)`` selects."""

    def __init__(self, func):
        self.is_save_time = func
        self.X, self.wgts = {}, {}

    def save(self, smc):
        t = smc.t
        if self.is_save_time(t):
            self.X[t] = _own(smc.X)
            self.wgts[t] = _own_weights(smc.wgts)


class RollingParticleHistory:
    """smoothing.py:181-219: keeps the k most recent particle systems."""

    def __init__(self, length):
        self.X = deque([], length)
        self.A = deque([], length)
        self.wgts = deque([], length)

    @property
    def N(self):
        return self.X[0].shape[0]

    @property
    def T(self):
        return len(self.X)

    def save(self, smc):
        self.X.append(_own(smc.X))
        self.A.append(_own(smc.A))
        self.wgts.append(_own_weights(smc.wgts))

    def compute_trajectories(self):
        """(T, N) int64 tensor B with B[t, n] = index at time t of the ancestor of X_T^n
        (smoothing.py:209-219); iterated gathers ``A[B]`` on the device."""
        Bs = [torch.arange(self.N, device=self.X[0].device)]
        for A in list(self.A)[-1:0:-1]:
            Bs.append(A[Bs[-1]])
        Bs.reverse()
        return torch.stack(Bs)


class ParticleHistory(RollingParticleHistory):
    """smoothing.py:222-270 (storage + ``extract_one_trajectory``).

    With ``qmc`` (an SQMC run, ``SMC(qmc=True, store_history=True)``) the history also keeps ``h_orders``: at each
    step t >= 1 ``save`` appends ``smc.h_order``, the Hilbert order of X[t-1] that the step resampled through, so that
    ``h_orders[t]`` orders X[t] for t = 0 .. T-2 ((N,) int64 CUDA tensors, 8 more bytes per particle per step);
    ``backward_sampling_qmc`` needs them."""

    def __init__(self, fk, qmc):
        self.X, self.A, self.wgts = [], [], []
        if qmc:
            self.h_orders = []
        self.fk = fk

    def save(self, smc):
        RollingParticleHistory.save(self, smc)
        if hasattr(self, "h_orders") and smc.t > 0:
            self.h_orders.append(smc.h_order)

    def extract_one_trajectory(self):
        traj, n = [], None
        for t in reversed(range(self.T)):
            if t == self.T - 1:
                n = int(rs.multinomial(self.wgts[-1].W, M=1)[0])
            else:
                n = int(self.A[t + 1][n])
            traj.append(self.X[t][n])
        return traj[::-1]

    # ------------------------------------------------------------------ FFBS
    # Extra keyword arguments of the samplers (optional, as SMC(seed=, noise=)): ``seed`` re-keys the device
    # generator first; ``noise`` is a dict of injected randomness for parity tests -- ``idx_T`` (M,) int, the
    # final-time indices, and per method:
    #   ON2     u (M, T-1): the uniform of the draw of trajectory m at time t;
    #   MCMC    prop (T-1, nsteps, M) int, lu (T-1, nsteps, M): proposals and log-uniforms of each step;
    #   reject  prop (T-1, M, max_trials) int, lu (T-1, M, max_trials): the trial-th proposal / log-uniform of
    #           trajectory m, and u_exact (T-1, M): the uniform of its exact fallback draw.
    def _init_backward_sampling(self, M, noise=None):
        """smoothing.py:278-281: idx (T, M) int64 on the device, idx[T-1] = multinomial(W_{T-1}, M)."""
        dev = self.X[-1].device
        idx = torch.empty((self.T, M), dtype=torch.int64, device=dev)
        if noise is not None and noise.get("idx_T") is not None:
            idx[-1] = as_device(noise["idx_T"], dtype=torch.int64, device=dev)
        else:
            idx[-1] = rs.multinomial(self.wgts[-1].W, M=M)
        return idx

    def _output_backward_sampling(self, paths):
        """smoothing.py:283-289: a list of T views of ONE (T, M[, d]) tensor; squeezed when M = 1."""
        if paths.shape[1] == 1:
            paths = paths[:, 0]
        return [paths[t] for t in range(self.T)]

    def backward_sampling_ON2(self, M, seed=None, noise=None):
        """O(N^2) FFBS, smoothing.py:291-311: paths[t][m] is component t of trajectory m."""
        return self._backward(_lib.SMOOTH_ON2, int(M), seed, noise)

    def backward_sampling_mcmc(self, M, nsteps=1, seed=None, noise=None):
        """MCMC backward sampling (independent Metropolis steps with multinomial proposals, started at the
        genealogy), smoothing.py:313-350; Dau & Chopin (2022)."""
        return self._backward(_lib.SMOOTH_MCMC, int(M), seed, noise, nsteps=int(nsteps))

    def backward_sampling_reject(self, M, max_trials=None, seed=None, noise=None):
        """Hybrid rejection backward sampling, smoothing.py:352-423: at most ``max_trials`` (default M) proposals
        per trajectory and time, then the exact O(N) draw.  Needs ``fk.upper_bound_trans``; sets ``acc_rate``,
        (T-1,) = (M - nrejected) / nprops per t."""
        M = int(M)
        max_trials = M if max_trials is None else int(max_trials)
        bounds = np.array([self.fk.upper_bound_trans(t + 1) for t in range(self.T - 1)], dtype=np.float64)
        return self._backward(_lib.SMOOTH_REJECT, M, seed, noise, max_trials=max_trials, bounds=bounds)

    def backward_sampling_qmc(self, M, seed=None, noise=None):
        """QMC forward-filtering backward-sampling of an SQMC history, smoothing.py:425-455.  One (M, T) point set u
        (scrambled Sobol', one dimension per time, so T <= rqmc.MAX_DIM = 4096): the final draw searches u[:, T-1] in
        the CDF of W_{T-1} taken in the Hilbert order of X[T-1]; at t < T-1 trajectory m searches u[m, t] in the CDF
        of lw_t + logpt(t + 1, X_t, x^m_{t+1}) taken in the order ``h_orders[t]``.  ``seed`` keys the points (as
        ``SMC(seed=)`` keys a run's), otherwise NumPy's global generator does, as ``rqmc.sobol``; ``noise={"u":
        (M, T)}`` injects the point set.  A history without Hilbert orders raises ``HilbertOrdersError``, a
        NotImplementedError and a ValueError."""
        from .rqmc import MAX_DIM
        if not hasattr(self, "h_orders"):
            raise HilbertOrdersError("QMC backward sampling needs a history that kept the Hilbert orders of its "
                                     "particles: run SMC(qmc=True, store_history=True)")
        if self.T > MAX_DIM:
            raise NotImplementedError(f"QMC backward sampling draws one Sobol' dimension per time step: T <= "
                                      f"{MAX_DIM} (got T = {self.T})")
        if len(self.h_orders) != self.T - 1:
            raise ValueError(f"QMC backward sampling: {len(self.h_orders)} Hilbert orders for T = {self.T}")
        return self._backward(_lib.SMOOTH_ON2, int(M), seed, noise, qmc=True)

    # ------------------------------------------------------------ two-filter
    def two_filter_smoothing(self, t, info, phi, loggamma, linear_cost=False, return_ess=False,
                             modif_forward=None, modif_info=None, seed=None, noise=None):
        """Two-filter estimate of the smoothing expectation of phi(X_t, X_{t+1}), smoothing.py:487-566.

        ``info`` is the information filter: an ``SMC`` run with ``store_history=True`` over the same T (usually the
        data in reverse), whose generation ti = T-2-t stands for X_{t+1}; ``loggamma`` is the log-density of its
        'prior' gamma_{t+1}.  One-dimensional states only (d > 1 raises NotImplementedError).

        Calling convention: ``phi(x, xf)`` and ``loggamma(x)`` receive CUDA fp64 tensors -- ``phi`` the two members
        of each pair as tensors of the same shape -- and return CUDA tensors or arrays of their length; in the O(N^2)
        method phi must give one value per pair, in the linear one a (K,) or (K, k) array.

        ``linear_cost=False`` (O(N^2)): sum_{n,m} omega_nm phi / sum_{n,m} omega_nm over all pairs, in blocks of at
        most 2^24 pairs (one kernel launch per block on a stock model's transition, ``fk.logpt`` on the pairs
        otherwise).  ``linear_cost=True`` (O(N), equal N in both filters): N pairs drawn by multinomial resampling
        (I from the information weights, then J from the forward ones, each optionally tilted by ``modif_info`` /
        ``modif_forward``), reweighted by the transition density.  ``return_ess`` also returns 1 / sum Om^2.

        Returns a CUDA fp64 0-d tensor (a (k,) tensor for a vector phi in the linear method); nothing is read back
        to the host.  ``seed`` re-keys the device generator first; ``noise={"I": ..., "J": ...}`` injects the
        draws of the linear method (parity tests)."""
        ti = self.T - 2 - t
        if t < 0 or t >= self.T - 1:
            raise ValueError("two-filter smoothing: t must be in range 0,...,T-2")
        if any(x.ndim > 1 and x.shape[1] != 1 for x in (self.X[t], self.X[t + 1])):
            raise NotImplementedError("two-filter smoothing is not built for d > 1 (one-dimensional states only)")
        ih = getattr(info, "hist", None)
        if not isinstance(ih, ParticleHistory) or ih.T != self.T:
            raise ValueError("two-filter smoothing: info must be an SMC run with store_history=True over the same "
                             f"T = {self.T}")
        x, xi = _flat(self.X[t]), _flat(ih.X[ti])
        lw = self.wgts[t].lw.contiguous()
        lwinfo = ih.wgts[ti].lw - as_device(loggamma(xi)).reshape(-1)
        from .state_space_models import transition_spec
        spec = transition_spec(self.fk)
        if linear_cost:
            return self._two_filter_ON(t, x, xi, lw, lwinfo, phi, spec, return_ess, modif_forward, modif_info,
                                       seed, noise)
        return self._two_filter_ON2(t, x, xi, lw, lwinfo, phi, spec)

    def _tf_desc(self, method, spec, t, x_fwd, x_info, **kw):
        d = _lib.TwoFilterDesc()
        d.method, d.model, d.dim, d.n_params = method, spec["model"], spec["dim"], len(spec["params"])
        for i, v in enumerate(spec["params"]):
            d.params[i] = float(v)
        sc = spec.get("step_consts")
        d.step_const = float(sc[t + 1]) if sc is not None else 0.0
        d.t, d.N, d.Ninfo = t, x_fwd.shape[0], x_info.shape[0]
        d.X, d.Xinfo = x_fwd.data_ptr(), x_info.data_ptr()
        d.x_stride, d.xi_stride = x_fwd.stride(0), x_info.stride(0)
        for k, v in kw.items():
            setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        ctx = context(x_fwd.device)
        _lib.check(ctx.lib.smcb_two_filter(ctx.handle, C.byref(d)))

    def _two_filter_ON2(self, t, x, xi, lw, lwinfo, phi, spec):
        """smoothing.py:527-547 by rows m of the information filter: L[m] = log sum_n exp(lw_t[n] + logpt(t+1,
        X_t[n], Xinfo[m])), S[m] the omega-weighted mean of phi over row m; then exp_and_normalise(lwinfo + L) . S.
        A row with no positive pair weight contributes exactly 0; no positive weight at all gives NaN (0 / 0)."""
        from .collectors import _ON2_PAIRS, _repeat_rows, _tile_rows
        N, Ni = x.shape[0], xi.shape[0]
        dev = x.device
        R = max(1, min(Ni, _ON2_PAIRS // N))
        L = torch.empty(Ni, dtype=torch.float64, device=dev)
        S = torch.empty(Ni, dtype=torch.float64, device=dev)
        for r0 in range(0, Ni, R):
            rows = min(R, Ni - r0)
            xa, xb = _tile_rows(x, rows), _repeat_rows(xi[r0:r0 + rows], N)      # pair [r, n] = (X_t[n], Xinfo[m])
            psi = as_device(phi(xa, xb))
            if psi.numel() != rows * N:
                raise ValueError("two-filter smoothing (O(N^2)): phi must return one value per pair, got shape "
                                 f"{tuple(psi.shape)} for {rows * N} pairs")
            psi = psi.reshape(rows, N).contiguous()
            if spec is not None:
                self._tf_desc(_lib.TF_ON2_ROWS, spec, t, x, xi, row0=r0, rows=rows, lw=lw, psi=psi, L=L, S=S)
            else:                  # fk.logpt on the device tensors of the pairs
                v = lw[None, :] + as_device(self.fk.logpt(t + 1, xa, xb)).reshape(rows, N)
                Lb = torch.logsumexp(v, dim=1)
                L[r0:r0 + rows] = Lb
                S[r0:r0 + rows] = torch.where(Lb > -np.inf, (torch.softmax(v, dim=1) * psi).sum(1), 0.0)
        W = rs.exp_and_normalise(lwinfo + L)
        return (W * S).sum()

    def _two_filter_ON(self, t, x, xi, lw, lwinfo, phi, spec, return_ess, modif_forward, modif_info, seed, noise):
        """smoothing.py:549-566."""
        N = x.shape[0]
        if xi.shape[0] != N:
            raise ValueError(f"two-filter smoothing (O(N)): the filters must have the same N, got {N} and "
                             f"{xi.shape[0]}")
        dev = x.device
        if seed is not None:
            context(dev).seed(seed)
        nz = noise or {}
        mf = None if modif_forward is None else as_device(modif_forward).reshape(-1).contiguous()
        mi = None if modif_info is None else as_device(modif_info).reshape(-1).contiguous()
        if nz.get("I") is not None:
            I = as_device(nz["I"], dtype=torch.int64, device=dev).reshape(-1)
        else:
            I = rs.multinomial(rs.exp_and_normalise(lwinfo if mi is None else lwinfo + mi))
        if nz.get("J") is not None:
            J = as_device(nz["J"], dtype=torch.int64, device=dev).reshape(-1)
        else:
            J = rs.multinomial(self.wgts[t].W if mf is None else rs.exp_and_normalise(lw + mf))
        if spec is not None:
            log_omega, xf, xg = (torch.empty(N, dtype=torch.float64, device=dev) for _ in range(3))
            self._tf_desc(_lib.TF_ON_LOGW, spec, t, x, xi, M=N, I=I, J=J, mf=0 if mf is None else mf,
                          mi=0 if mi is None else mi,
                          log_omega=log_omega, xf=xf, xi=xg)
        else:
            xf, xg = x[J], xi[I]
            log_omega = as_device(self.fk.logpt(t + 1, xf, xg)).reshape(-1)
            if mf is not None:
                log_omega = log_omega - mf[J]
            if mi is not None:
                log_omega = log_omega - mi[I]
        Om = rs.exp_and_normalise(log_omega)
        v = as_device(phi(xf, xg))
        if v.ndim == 0 or v.shape[0] != N or v.ndim > 2:
            raise ValueError(f"two-filter smoothing (O(N)): phi must return (N,) or (N, k) with N = {N}, got "
                             f"{tuple(v.shape)}")
        w = Om if v.ndim == 1 else Om[:, None]
        est = (w * v).sum(0) / Om.sum()                      # np.average(phi, axis=0, weights=Om)
        if return_ess:
            return est, 1.0 / (Om ** 2).sum()
        return est

    # -------------------------------------------------------------- plumbing
    def _history_desc(self, method, M):
        """Descriptor with the per-t pointer tables of the history, and the tensors it points into."""
        Xs = [as_device(x) if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float64) else x
              for x in self.X]
        shape = tuple(Xs[0].shape)
        if any(tuple(x.shape) != shape for x in Xs):
            raise ValueError("backward sampling: the particle arrays differ in shape over time")
        strides = {tuple(x.stride()) for x in Xs}
        if len(strides) != 1:
            Xs = [x.contiguous() for x in Xs]
        d = _lib.SmoothDesc()
        d.method, d.T, d.N, d.M = method, self.T, shape[0], M
        d.dim = 1 if len(shape) == 1 else shape[1]
        st = Xs[0].stride()
        d.x_stride_n, d.x_stride_c = st[0], (st[1] if len(shape) > 1 else 0)
        dev = Xs[0].device
        lws = [w.lw.contiguous() for w in self.wgts]
        As = list(self.A)
        keep = {"X": Xs, "lw": lws, "A": As,
                "tX": torch.tensor([x.data_ptr() for x in Xs], dtype=torch.int64, device=dev),
                "tlw": torch.tensor([w.data_ptr() for w in lws], dtype=torch.int64, device=dev),
                "tA": torch.tensor([0 if a is None else a.data_ptr() for a in As], dtype=torch.int64, device=dev)}
        d.X, d.lw, d.A = keep["tX"].data_ptr(), keep["tlw"].data_ptr(), keep["tA"].data_ptr()
        return d, keep, Xs

    def _cdfs(self, N, dev):
        """(T-1, N) inclusive prefix sums of W_t (the one fp64 scratch of the MCMC / reject samplers); rows padded to
        an even length so that each is 16-byte aligned for smcb_cumsum."""
        ctx = context(dev)
        cdf = torch.empty((max(self.T - 1, 1), N + (N & 1)), dtype=torch.float64, device=dev)
        W = torch.empty(N, dtype=torch.float64, device=dev)
        for t in range(self.T - 1):
            w = self.wgts[t]
            _lib.check(ctx.lib.smcb_weights_from_stats(ctx.handle, ptr(w.lw), N, ptr(w._stats), ptr(W)))
            _lib.check(ctx.lib.smcb_cumsum(ctx.handle, ptr(W), N, ptr(cdf[t])))
        return cdf

    def _init_qmc(self, M, seed, noise):
        """smoothing.py:443-450: the (M, T) points and idx (T, M) with the final draw idx[T-1] = hT[searchsorted(
        cumsum(W_{T-1}[hT]), u[:, T-1])], hT the Hilbert order of X[T-1]; the search runs on the sorted column."""
        from .hilbert import hilbert_order, hilbert_sort
        from .rqmc import sobol_points
        T, dev = self.T, self.X[-1].device
        ctx = context(dev)
        if noise is not None and noise.get("u") is not None:
            u = as_device(noise["u"], device=dev).reshape(M, T)
        else:
            key = int(np.random.randint(0, 2 ** 62, dtype=np.int64)) if seed is None else int(seed)
            u = sobol_points(M, T, key).t()
        orders = [as_device(h, dtype=torch.int64, device=dev).reshape(-1) for h in self.h_orders]
        hT = hilbert_sort(self.X[-1])
        cdf = rs.cumsum(self.wgts[-1].W[hT])
        uT = u[:, T - 1].contiguous()
        tau = hilbert_order(uT)                                  # argsort: the search takes sorted queries
        found = torch.empty(M, dtype=torch.int64, device=dev)
        _lib.check(ctx.lib.smcb_searchsorted(ctx.handle, ptr(cdf), cdf.shape[0], ptr(uT[tau]), M, ptr(found)))
        idx = torch.empty((T, M), dtype=torch.int64, device=dev)
        idx[-1, tau] = hT[found]
        return u, orders, idx

    def _backward(self, method, M, seed, noise, nsteps=1, max_trials=0, bounds=None, qmc=False):
        if M < 1:
            raise ValueError("backward sampling: M must be >= 1")
        from .state_space_models import transition_spec
        ctx = context(self.X[-1].device)
        if seed is not None:
            ctx.seed(seed)
        spec = transition_spec(self.fk)
        orders = None
        if qmc:
            u, orders, idx = self._init_qmc(M, seed, noise)
            noise = {"u": u[:, :self.T - 1]}
        else:
            idx = self._init_backward_sampling(M, noise)
        if spec is None:
            idx = self._plugin(method, M, idx, noise, nsteps, max_trials, bounds, orders)
        d, keep, Xs = self._history_desc(method if spec is not None else _lib.SMOOTH_GATHER, M)
        dev = Xs[0].device
        T, N, D = self.T, d.N, d.dim
        paths = torch.empty((T, M) + ((D,) if Xs[0].ndim > 1 else ()), dtype=torch.float64, device=dev)
        d.idx, d.paths = idx.data_ptr(), paths.data_ptr()
        if spec is not None:
            d.model, d.n_params = spec["model"], len(spec["params"])
            for i, v in enumerate(spec["params"]):
                d.params[i] = float(v)
            if spec["step_consts"] is not None:
                keep["sc"] = as_device(spec["step_consts"], device=dev)
                d.step_consts = keep["sc"].data_ptr()
            d.idx_T = idx[-1].data_ptr()           # read, then rewritten unchanged, by the same thread
            d.nsteps, d.max_trials = nsteps, max_trials
            nz = noise or {}
            if method == _lib.SMOOTH_ON2 and nz.get("u") is not None:
                keep["u"] = as_device(nz["u"], device=dev).reshape(M, T - 1).contiguous()
                d.u = keep["u"].data_ptr()
            if orders and T > 1:
                keep["orders"] = orders
                keep["tord"] = torch.tensor([o.data_ptr() for o in orders], dtype=torch.int64, device=dev)
                d.order = keep["tord"].data_ptr()
            if method != _lib.SMOOTH_ON2:
                if nz.get("prop") is not None:
                    shape = (T - 1, nsteps, M) if method == _lib.SMOOTH_MCMC else (T - 1, M, max_trials)
                    keep["prop"] = as_device(np.asarray(nz["prop"]).reshape(shape), dtype=torch.int64, device=dev)
                    keep["lu"] = as_device(np.asarray(nz["lu"]).reshape(shape), device=dev)
                    d.prop, d.lu = keep["prop"].data_ptr(), keep["lu"].data_ptr()
                elif T > 1:
                    keep["cdf"] = self._cdfs(N, dev)
                    d.cdf, d.cdf_ld = keep["cdf"].data_ptr(), keep["cdf"].shape[1]
            if method == _lib.SMOOTH_REJECT:
                if nz.get("u_exact") is not None:
                    keep["u_exact"] = as_device(np.asarray(nz["u_exact"]).reshape(T - 1, M), device=dev)
                    d.u_exact = keep["u_exact"].data_ptr()
                keep["bounds"] = as_device(bounds if T > 1 else np.zeros(1), device=dev)
                keep["counts"] = torch.zeros((max(T - 1, 1), 2), dtype=torch.int64, device=dev)
                d.log_bound, d.counts = keep["bounds"].data_ptr(), keep["counts"].data_ptr()
        _lib.check(ctx.lib.smcb_backward_sample(ctx.handle, C.byref(d)))
        if spec is not None and method == _lib.SMOOTH_REJECT:
            cnt = keep["counts"].cpu().numpy()[: T - 1].astype(np.float64)
            with np.errstate(divide="ignore", invalid="ignore"):
                self.acc_rate = cnt[:, 0] / cnt[:, 1]
        # the pointer tables and scratch may be freed now: the caching allocator hands their memory only to work
        # enqueued later on this stream.  The (T, M) indices of the last pass stay inspectable.
        self._bs_idx = idx
        return self._output_backward_sampling(paths)

    # ----------------------------------------------------------- plugin path
    def _exact_draw(self, t, xn, u, out, order=None):
        """smoothing.py:310 / 418-421 for one trajectory: searchsorted(cumsum(exp_and_normalise(lw_t +
        logpt(t + 1, X_t, xn))), u) written into the device int64 scalar ``out``.  With ``order`` (QMC, smoothing.py:
        449-452) the CDF runs over the weights in that order and the position found maps back through it."""
        ctx = context(out.device)
        W = rs.exp_and_normalise(self.wgts[t].lw + as_device(self.fk.logpt(t + 1, self.X[t], xn)))
        cdf = rs.cumsum(W if order is None else W[order])
        su = rs._uniforms(1, W) if u is None else torch.full((1,), float(u), dtype=torch.float64, device=W.device)
        _lib.check(ctx.lib.smcb_searchsorted(ctx.handle, ptr(cdf), W.shape[0], ptr(su), 1, C.c_void_p(out.data_ptr())))
        out.masked_fill_(~(W.sum() > 0), 0)      # no positive weight (a NaN row): 0, as the kernels' exact draws
        if order is not None:
            out.copy_(order[out])

    def _plugin(self, method, M, idx, noise, nsteps, max_trials, bounds, orders=None):
        """The reference's loops with ``fk.logpt`` on CUDA tensors (vectorised over M for MCMC / reject, over N per
        (t, m) for ON2); indices stay on the device."""
        nz = noise or {}
        T = self.T
        dev = idx.device
        X = self.X
        if method == _lib.SMOOTH_ON2:
            u = None if nz.get("u") is None else _np(nz["u"]).reshape(M, T - 1)
            for m in range(M):
                for t in reversed(range(T - 1)):
                    xn = X[t + 1][idx[t + 1, m]]
                    self._exact_draw(t, xn, None if u is None else u[m, t], idx[t, m],
                                     None if orders is None else orders[t])
            return idx
        if method == _lib.SMOOTH_MCMC:
            prop_in = None if nz.get("prop") is None else as_device(np.asarray(nz["prop"]).reshape(T - 1, nsteps, M),
                                                                     dtype=torch.int64, device=dev)
            lu_in = None if nz.get("lu") is None else as_device(np.asarray(nz["lu"]).reshape(T - 1, nsteps, M),
                                                                 device=dev)
            for t in reversed(range(T - 1)):
                xn = X[t + 1][idx[t + 1]]
                idx[t] = self.A[t + 1][idx[t + 1]]
                for i in range(nsteps):
                    prop = rs.multinomial_iid(self.wgts[t].W, M=M) if prop_in is None else prop_in[t, i]
                    lpr = (as_device(self.fk.logpt(t + 1, X[t][prop], xn))
                           - as_device(self.fk.logpt(t + 1, X[t][idx[t]], xn)))
                    lu = torch.log(rs._uniforms(M, lpr)) if lu_in is None else lu_in[t, i]
                    idx[t] = torch.where(lu < lpr, prop, idx[t])
            return idx
        prop_in = None if nz.get("prop") is None else as_device(np.asarray(nz["prop"]).reshape(T - 1, M, max_trials),
                                                                 dtype=torch.int64, device=dev)
        lu_in = None if nz.get("lu") is None else as_device(np.asarray(nz["lu"]).reshape(T - 1, M, max_trials),
                                                             device=dev)
        u_exact = None if nz.get("u_exact") is None else np.asarray(nz["u_exact"]).reshape(T - 1, M)
        self.acc_rate = np.zeros(T - 1)
        for t in reversed(range(T - 1)):
            where = torch.arange(M, device=dev)
            who = X[t + 1][idx[t + 1]]
            nprops, ntrials, nrej = 0, 0, M
            while nrej > 0 and ntrials < max_trials:
                nprops += nrej
                prop = rs.multinomial_iid(self.wgts[t].W, M=nrej) if prop_in is None else prop_in[t, where, ntrials]
                lpr = as_device(self.fk.logpt(t + 1, X[t][prop], who)) - float(bounds[t])
                lu = torch.log(rs._uniforms(nrej, lpr)) if lu_in is None else lu_in[t, where, ntrials]
                ntrials += 1
                acc = lu < lpr
                idx[t, where[acc]] = prop[acc]
                where, who = where[~acc], who[~acc]
                nrej = int(where.shape[0])
            for m in where.tolist():
                self._exact_draw(t, X[t + 1][idx[t + 1, m]], None if u_exact is None else u_exact[t, m], idx[t, m])
            self.acc_rate[t] = (M - nrej) / nprops if nprops else np.nan
        return idx


# ---------------------------------------------------------------------------
# smoothing_worker -- smoothing.py:569-677
# ---------------------------------------------------------------------------
_PURE_REJECT_TRIALS = (1 << 24) - 1     # the most proposals per draw the device samplers take (reference: N * 10^9)
WORKER_METHODS = ("FFBS_purereject", "FFBS_hybrid", "FFBS_MCMC", "FFBS_ON2", "FFBS_QMC",
                  "two-filter_ON", "two-filter_ON_prop", "two-filter_ON2")


def _norm_logpdf(x, loc, scale):
    """scipy.stats.norm.logpdf(x, loc, scale) on device tensors, in scipy's order of operations."""
    z = (x - loc) / scale
    return -z * z / 2.0 - 0.5 * np.log(2.0 * np.pi) - torch.log(scale)


def smoothing_worker(method=None, N=100, fk=None, fk_info=None, add_func=None, log_gamma=None):
    """Generic worker for the off-line smoothing algorithms, smoothing.py:569-677; usable with
    ``utils.multiplexer``.  Runs the forward filter (and, for the two-filter methods, the information filter
    ``fk_info``, by default the same model with the data in reverse), then estimates for every t in 0..T-2 the
    smoothing expectation of ``add_func(t, x, xf)`` (x = X_t, xf = X_{t+1}) with ``method``, one of
    ``WORKER_METHODS``.  ``add_func`` and ``log_gamma`` receive CUDA fp64 tensors, as ``two_filter_smoothing``'s
    ``phi`` and ``loggamma`` do.

    Returns {"est": (T-1,) array, "cpu": seconds}: the estimates stay on the device until one read at the end, and
    ``cpu`` is the wall time of the runs plus the smoothing, ending with that read.  'FFBS_purereject' is the
    hybrid sampler with 2^24 - 1 proposals per draw before the exact draw (the reference allows N * 10^9);
    'FFBS_QMC' raises NotImplementedError: it needs an SQMC forward pass, and the reference's worker calls
    ``particles.SQMC``, which the reference does not define, so there is no behaviour to follow; run
    ``SMC(qmc=True, store_history=True)`` and then ``hist.backward_sampling_qmc`` instead.  An unknown method raises
    ValueError."""
    import time

    from .core import SMC
    if method not in WORKER_METHODS:
        raise ValueError(f"smoothing_worker: no such method {method!r}; one of {WORKER_METHODS}")
    if method == "FFBS_QMC":
        raise NotImplementedError("smoothing_worker: FFBS_QMC needs an SQMC forward pass, which the reference's "
                                  "worker asks of particles.SQMC, a class it does not define; run SMC(qmc=True, "
                                  "store_history=True) and then hist.backward_sampling_qmc(M)")
    T = fk.T
    if fk_info is None:
        fk_info = fk.__class__(ssm=fk.ssm, data=fk.data[::-1])
    pf = SMC(fk=fk, N=N, store_history=True)
    tic = time.perf_counter()
    pf.run()
    h = pf.hist
    ests = []
    if method.startswith("FFBS"):
        sub = method.split("_")[-1]
        if sub == "ON2":
            z = h.backward_sampling_ON2(N)
        elif sub == "MCMC":
            z = h.backward_sampling_mcmc(N)
        elif sub == "hybrid":
            z = h.backward_sampling_reject(N)
        else:
            z = h.backward_sampling_reject(N, max_trials=_PURE_REJECT_TRIALS)
        for t in range(T - 1):
            ests.append(as_device(add_func(t, z[t], z[t + 1])).mean())
    else:
        infopf = SMC(fk=fk_info, N=N, store_history=True)
        infopf.run()
        ih = infopf.hist
        for t in range(T - 1):
            psi = lambda x, xf, t=t: add_func(t, x, xf)          # noqa: E731
            if method == "two-filter_ON2":
                ests.append(h.two_filter_smoothing(t, infopf, psi, log_gamma))
                continue
            mf = mi = None
            if method == "two-filter_ON_prop":
                ti = T - 2 - t
                a, b = _flat(ih.X[ti + 1]), _flat(h.X[t + 1])
                mf = _norm_logpdf(_flat(h.X[t]), a.mean(), a.std(correction=0))
                mi = _norm_logpdf(_flat(ih.X[ti]), b.mean(), b.std(correction=0))
            ests.append(h.two_filter_smoothing(t, infopf, psi, log_gamma, linear_cost=True, modif_forward=mf,
                                               modif_info=mi))
    est = torch.stack([e.reshape(()) for e in ests]).cpu().numpy() if ests else np.zeros(0)
    cpu_time = time.perf_counter() - tic
    return {"est": est, "cpu": cpu_time}
