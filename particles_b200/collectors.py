"""Per-step summaries -- the part of ``particles/collectors.py`` that sits on the
boundary of the hot path (SURVEY.md section 2 row 5, section 8b): the three default
collectors and ``Moments``.  A collector reads attributes of the running ``SMC``
object; on the fused path the three defaults are filled lazily from the (T, 4)
device table the kernels write, so they cost no per-step host sync.

The on-line smoothers of additive functionals (``Online_smooth_naive``, ``Online_smooth_ON2``, ``Paris``) keep
Phi on the device; their per-step work is csrc/smcb_online.cu plus the user's ``add_func``, and their summaries
are read from the device in one transfer per ``collect`` (per step) or per fused ``run()``.  The variance
collectors ``Var`` and ``Var_logLt`` (variance_estimators.py) share that row buffer.  ``Fixed_lag_smooth`` reads
the rolling history (``store_history=k``).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from . import resampling as rs
from .device import as_device, context


class Collector:
    """particles/collectors.py:234-271: subclass and define ``fetch(smc)``."""
    signature = {}

    @property
    def summary_name(self):
        cn = self.__class__.__name__
        return cn[0].lower() + cn[1:]          # Moments -> moments, LogLts -> logLts

    def __init__(self, **kwargs):
        self.summary = []
        for k, v in self.signature.items():
            setattr(self, k, v)
        for k, v in kwargs.items():
            if k in self.signature:
                setattr(self, k, v)
            else:
                raise ValueError(f"Collector {self.__class__.__name__}: unknown parameter {k}")
        self._kwargs = kwargs

    def __call__(self):
        # a collector instance is a template: calling it clones it (collectors.py:263-266)
        return self.__class__(**self._kwargs)

    def collect(self, smc):
        self.summary.append(self.fetch(smc))


class ESSs(Collector):      # collectors.py:278-282
    summary_name = "ESSs"

    def fetch(self, smc):
        return smc.wgts.ESS


class LogLts(Collector):    # collectors.py:285-287
    def fetch(self, smc):
        return smc.logLt


class Rs_flags(Collector):  # collectors.py:290-292
    def fetch(self, smc):
        return smc.rs_flag


default_collector_cls = [ESSs, LogLts, Rs_flags]


class Moments(Collector):
    """particles/collectors.py:301-317: ``mom_func(W, X)`` or the model's
    ``default_moments`` (weighted mean and variance, resampling.py:320-338)."""
    signature = {"mom_func": None}

    def fetch(self, smc):
        f = smc.fk.default_moments if self.mom_func is None else self.mom_func
        return f(smc.W, smc.X)


# ---------------------------------------------------------------------------
# on-line smoothing of additive functionals -- particles/collectors.py:345-449
# ---------------------------------------------------------------------------
_ON2_PAIRS = 1 << 24        # ON2: rows per block so that omega (rows, N) and psi stay within 2^24 pairs


class _Gen:
    """The generation a smoother reads at time t: X (N,) or (N, d), log-weights lw (N,) and, for t >= 1, the
    ancestors A (N,) of this step (the identity when the step did not resample).  All CUDA tensors."""
    __slots__ = ("t", "X", "lw", "A")

    def __init__(self, t, X, lw, A):
        self.t, self.X, self.lw, self.A = t, X, lw, A


def _gen_of(smc):
    """The current generation of a running ``SMC``, without a host sync on the fused path."""
    if smc.fused:
        return smc._engine_gen(smc._done - 1)
    return _Gen(smc.t, as_device(smc.X), as_device(smc.wgts.lw), smc.A)


class DeviceRowsMixin:
    """Collectors whose per-step work stays on the device: ``_step(smc, t)`` enqueues the work of step t and appends
    one device row to ``_rows`` (no host sync); ``_flush`` moves the rows into ``summary`` in one transfer -- per step
    in ``collect``, once per run in the fused ``SMC.run()``.  A row is a float summary, or a (k,) array when
    ``_vector``."""

    def collect(self, smc):
        self._step(smc, smc.t)
        self._flush()

    def _flush(self):
        """Move the rows enqueued since the last flush into ``summary`` (one device-to-host transfer)."""
        if not self._rows:
            return
        rows = torch.stack(self._rows).cpu().numpy()
        self._rows = []
        self.summary.extend(r.copy() if self._vector else float(r[0]) for r in rows)


class OnlineSmootherMixin(DeviceRowsMixin):
    """collectors.py:345-365: Phi_0 = add_func(0, None, X_0), then the class's ``update``; each step appends the
    weighted mean of Phi under W_t -- a float when Phi is (N,), a (k,) array when Phi is (N, k).

    Calling convention of ``add_func`` here: CUDA fp64 tensors ``xp`` and ``x`` of the same shape, (K,) or (K, d),
    returning (K,) or (K, k) (``xp`` is None at t = 0).  ON2 and PaRIS call it on flattened pairs."""

    def _step(self, smc, t):
        self._advance(smc.fk, smc._seed, smc._engine_gen(t) if smc.fused else _gen_of(smc))

    def _advance(self, fk, seed, g):
        """Enqueue the work of step g.t (no host sync)."""
        if g.t == 0 or not hasattr(self, "_Phi"):
            psi = fk.add_func(0, None, g.X)
            self._vector = _ndim(psi) > 1
            self._Phi = _as_phi(psi, g.X.shape[0]).clone()          # add_func may return its input
            self._rows, self._pending = [], []
        else:
            self._Phi = self.update(fk, seed, g)
        W = rs.exp_and_normalise(g.lw)
        self._rows.append((W[:, None] * self._Phi).sum(0) / W.sum())   # np.average(Phi, axis=0, weights=W)
        self._prev, self._prev_W = g, W

    def update(self, fk, seed, g):
        raise NotImplementedError

    def _psi(self, fk, t, xp, x):
        return _as_phi(fk.add_func(t, xp, x), x.shape[0])


def _ndim(v):
    return v.ndim if hasattr(v, "ndim") else np.ndim(v)


def _as_phi(v, K):
    """add_func's (K,) or (K, k) output -> (K, k) contiguous fp64 on the device."""
    v = as_device(v)
    if v.ndim == 0 or v.shape[0] != K or v.ndim > 2:
        raise ValueError(f"add_func must return an array of shape (K,) or (K, k) with K = {K}, got "
                         f"{tuple(v.shape)}")
    return (v.reshape(K, 1) if v.ndim == 1 else v).contiguous()


def _rows_of(X, idx):
    return X.index_select(0, idx)


def _repeat_rows(X, r):
    """Each row of X repeated r times, in place: (K, ...) -> (K * r, ...)."""
    return X.unsqueeze(1).expand(X.shape[0], r, *X.shape[1:]).reshape(X.shape[0] * r, *X.shape[1:])


def _tile_rows(X, r):
    """X stacked r times: (K, ...) -> (r * K, ...)."""
    return X.unsqueeze(0).expand(r, *X.shape).reshape(r * X.shape[0], *X.shape[1:])


def _online_desc(method, spec, g_prev, g, **kw):
    d = _lib.OnlineDesc()
    d.method, d.t, d.N = method, g.t, g.X.shape[0]
    if spec is not None:
        d.model, d.n_params, d.dim = spec["model"], len(spec["params"]), spec["dim"]
        for i, v in enumerate(spec["params"]):
            d.params[i] = float(v)
        sc = spec.get("step_consts")
        d.step_const = float(sc[g.t]) if sc is not None else 0.0
        Xp, X = g_prev.X, g.X
        if Xp.stride() != X.stride():
            raise ValueError("on-line smoothing: X_{t-1} and X_t differ in layout")
        d.X_prev, d.X = Xp.data_ptr(), X.data_ptr()
        d.x_stride_n, d.x_stride_c = X.stride(0), (X.stride(1) if X.ndim > 1 else 0)
        d.lw_prev = g_prev.lw.data_ptr()
    for k, v in kw.items():
        setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return d


def _run(d, like):
    ctx = context(like.device)
    _lib.check(ctx.lib.smcb_online_smooth(ctx.handle, C.byref(d)))


def _spec(fk):
    from .state_space_models import transition_spec
    return transition_spec(fk)


def _prepare(g):
    """Particles as the kernels read them: fp64 on the device, (N,) or (N, d) with element strides."""
    X = as_device(g.X) if not (isinstance(g.X, torch.Tensor) and g.X.is_cuda and g.X.dtype == torch.float64) else g.X
    return _Gen(g.t, X, g.lw.contiguous(), g.A)


class Online_smooth_naive(OnlineSmootherMixin, Collector):
    """collectors.py:368-370: Phi_t = Phi_{t-1}[A_t] + add_func(t, X_{t-1}[A_t], X_t) (genealogy tracking)."""

    def update(self, fk, seed, g):
        A = g.A
        return self._Phi.index_select(0, A) + self._psi(fk, g.t, _rows_of(self._prev.X, A), g.X)


class Online_smooth_ON2(OnlineSmootherMixin, Collector):
    """collectors.py:373-387: Phi_t[n] = sum_m omega[n, m] (Phi_{t-1}[m] + add_func(t, X_{t-1}[m], X_t[n])), with
    omega[n, :] = exp_and_normalise(lw_{t-1} + logpt(t, X_{t-1}, X_t[n])).  O(N^2): blocks of rows."""

    def update(self, fk, seed, g):
        gp, g = _prepare(self._prev), _prepare(g)
        N, K = g.X.shape[0], self._Phi.shape[1]
        spec = _spec(fk)
        R = max(1, min(N, _ON2_PAIRS // N))
        dev = g.X.device
        Phi = torch.empty((N, K), dtype=torch.float64, device=dev)
        omega = torch.empty((R, N), dtype=torch.float64, device=dev)
        for r0 in range(0, N, R):
            rows = min(R, N - r0)
            om = omega[:rows]
            xr = g.X[r0:r0 + rows]
            if spec is not None:
                _run(_online_desc(_lib.ONLINE_ON2_W, spec, gp, g, row0=r0, rows=rows, omega=om), om)
            else:                  # fk.logpt on the device tensors of the pairs
                lpt = as_device(fk.logpt(g.t, _tile_rows(gp.X, rows), _repeat_rows(xr, N))).reshape(rows, N)
                om.copy_(torch.softmax(gp.lw[None, :] + lpt, dim=1))
            psi = self._psi(fk, g.t, _tile_rows(gp.X, rows), _repeat_rows(xr, N))
            _run(_online_desc(_lib.ONLINE_PHI_ON2, None, gp, g, rows=rows, k=K, omega=om,
                              phi_prev=self._Phi, psi=psi, phi=Phi[r0:r0 + rows]), om)
        return Phi


class Paris(OnlineSmootherMixin, Collector):
    """collectors.py:390-449: hybrid PaRIS (Olsson & Westerborn 2017; Dau & Chopin 2022).  For each particle n,
    ``Nparis`` ancestors are drawn from the backward kernel by rejection (at most ``max_trials`` proposals from
    W_{t-1}, default N, accepted with probability p_t / C_t, C_t = ``ssm.upper_bound_log_pt(t)``), then exactly;
    Phi_t[n] is the mean over those draws of Phi_{t-1}[a] + add_func(t, X_{t-1}[a], X_t[n]).  ``nprop`` lists the
    proposals made at each step ([0.0] at t = 0).

    Optional keyword, as ``SMC(noise=)``: ``noise`` -- a callable ``t -> dict`` of injected randomness for step t
    (parity tests): ``prop`` (N, Nparis, L) int and ``lu`` (N, Nparis, L), the proposals and log-uniforms of each
    trial (L = max_trials), and ``u_exact`` (N, Nparis), the uniform of each exact draw."""

    signature = {"Nparis": 2, "max_trials": None, "noise": None}

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.nprop = [0.0]
        self._counts = []

    def _flush(self):
        DeviceRowsMixin._flush(self)
        if self._counts:
            c = torch.stack(self._counts).cpu().numpy()
            self._counts = []
            self.nprop.extend(int(v) for v in c[:, 1])
            self._acc = getattr(self, "_acc", []) + [int(v) for v in c[:, 0]]

    @property
    def acc_rate(self):
        """Accepted draws over proposals at each step t >= 1 (NaN where no proposal was made)."""
        acc, nprop = np.array(getattr(self, "_acc", []), dtype=float), np.array(self.nprop[1:], dtype=float)
        with np.errstate(divide="ignore", invalid="ignore"):
            return acc / nprop

    def update(self, fk, seed, g):
        gp, g = _prepare(self._prev), _prepare(g)
        N, Np = g.X.shape[0], int(self.Nparis)
        mt = N if self.max_trials is None else int(self.max_trials)
        bound = float(fk.ssm.upper_bound_log_pt(g.t))           # collectors.py:432
        nz = self.noise(g.t) if self.noise is not None else {}
        dev = g.X.device
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        B = torch.empty((N, Np), dtype=torch.int64, device=dev)
        keep = {}
        if nz.get("prop") is not None:
            keep["prop"] = as_device(np.asarray(nz["prop"]).reshape(N, Np, mt), dtype=torch.int64, device=dev)
            keep["lu"] = as_device(np.asarray(nz["lu"]).reshape(N, Np, mt), device=dev)
        if nz.get("u_exact") is not None:
            keep["u_exact"] = as_device(np.asarray(nz["u_exact"]).reshape(N, Np), device=dev)
        spec = _spec(fk)
        if spec is not None:
            kw = {k: v for k, v in keep.items()}
            if "prop" not in keep and mt > 0:
                kw["cdf"] = rs.cumsum(self._prev_W)
            _run(_online_desc(_lib.ONLINE_PARIS, spec, gp, g, Np=Np, max_trials=mt, seed=int(seed) & (2 ** 64 - 1),
                              log_bound=bound, B=B, counts=counts, **kw), B)
        else:
            self._plugin(fk, gp, g, B.view(-1), counts, bound, mt, keep)
        Bf = B.view(-1)
        psi = self._psi(fk, g.t, _rows_of(gp.X, Bf), _repeat_rows(g.X, Np))
        Phi = torch.empty_like(self._Phi)
        _run(_online_desc(_lib.ONLINE_PHI_PARIS, None, gp, g, Np=Np, k=self._Phi.shape[1], B=B,
                          phi_prev=self._Phi, psi=psi, phi=Phi), Phi)
        self._counts.append(counts)
        self._B = B                  # the ancestors of the last step (inspectable, like ParticleHistory._bs_idx)
        return Phi

    def _plugin(self, fk, gp, g, B, counts, bound, mt, keep):
        """The same draws with ``fk.logpt`` on CUDA tensors, vectorised over the draws still pending."""
        N = g.X.shape[0]
        Np = B.shape[0] // N
        dev = B.device
        where = torch.arange(B.shape[0], device=dev)
        who = _rows_of(g.X, where // Np)
        nprops, ntrials, nrej = 0, 0, B.shape[0]
        prop_in = None if "prop" not in keep else keep["prop"].view(-1, mt)
        lu_in = None if "lu" not in keep else keep["lu"].view(-1, mt)
        while nrej > 0 and ntrials < mt:
            nprops += nrej
            prop = rs.multinomial_iid(self._prev_W, M=nrej) if prop_in is None else prop_in[where, ntrials]
            lpr = as_device(fk.logpt(g.t, _rows_of(gp.X, prop), who)) - bound
            lu = torch.log(rs._uniforms(nrej, lpr)) if lu_in is None else lu_in[where, ntrials]
            ntrials += 1
            acc = lu < lpr
            B[where[acc]] = prop[acc]
            where, who = where[~acc], who[~acc]
            nrej = int(where.shape[0])
        ue = None if "u_exact" not in keep else keep["u_exact"].view(-1)
        for j in where.tolist():          # collectors.py:437-440
            lw = gp.lw + as_device(fk.logpt(g.t, gp.X, _repeat_rows(g.X[j // Np:j // Np + 1], N)))
            u = None if ue is None else float(ue[j])
            W = rs.exp_and_normalise(lw)
            a = rs.multinomial_once(W, u)
            B[j] = a if bool(W.sum() > 0) else 0      # no positive weight: 0, as the kernel's exact draw
        counts[0] = B.shape[0] - nrej
        counts[1] = nprops


def _lw_of(smc):
    """The log-weights of the current generation, on the device."""
    if smc.fused:
        return smc._engine.lw[smc._cur()]
    return as_device(smc.wgts.lw).contiguous()


class Fixed_lag_smooth(Collector):
    """collectors.py:324-342: with ``store_history=k``, the weighted mean under W_t of ``phi`` of the fixed-lag
    trajectories.  ``phi`` receives the list of the ``hist.T`` CUDA tensors X_s[B[s]] (B =
    ``hist.compute_trajectories()``) and returns (N,); the summary is a float.  Without ``phi`` it raises TypeError,
    as the reference's ``np.average`` of a list of arrays does."""
    signature = {"phi": None}

    def fetch(self, smc):
        if self.phi is None:
            raise TypeError("Fixed_lag_smooth: phi must map the list of fixed-lag particle arrays to an (N,) array")
        B = smc.hist.compute_trajectories()
        Xs = [as_device(X)[B[i]] for i, X in enumerate(smc.hist.X)]
        lw = _lw_of(smc)
        v = as_device(self.phi(Xs))
        if v.shape != lw.shape:
            raise ValueError(f"Fixed_lag_smooth: phi must return an array of shape {tuple(lw.shape)}, got "
                             f"{tuple(v.shape)}")
        W = rs.exp_and_normalise(lw)
        return float(((W * v).sum() / W.sum()).item())           # np.average(phi(Xs), weights=W)


_ONLINE = (Online_smooth_naive, Online_smooth_ON2, Paris)
_REF_COLLECTORS = {c.__name__: c for c in _ONLINE + (Fixed_lag_smooth,)}


def _ref_classes(module):
    if module == "particles.collectors":
        return _REF_COLLECTORS
    if module == "particles.variance_estimators":
        from . import variance_estimators as ve
        return {c.__name__: c for c in (ve.Var, ve.Var_logLt, ve.Lag_based_var)}
    return {}


def _native(col):
    """The reference's own on-line smoothing, fixed-lag and variance collectors (particles.collectors,
    particles.variance_estimators) -> ours, same keyword arguments."""
    cls = type(col)
    ours = _ref_classes(cls.__module__).get(cls.__name__)
    if ours is not None:
        return ours(**{k: getattr(col, k) for k in getattr(cls, "signature", {}) if k in ours.signature})
    return col()


class Summaries:
    """particles/collectors.py:215-231."""

    def __init__(self, cols):
        self._collectors = [cls() for cls in default_collector_cls]
        self._n_default = len(self._collectors)
        if cols is not None:
            self._collectors.extend(_native(col) for col in cols)
        for col in self._collectors:
            setattr(self, col.summary_name, col.summary)

    @property
    def only_defaults(self):
        return len(self._collectors) == self._n_default

    @property
    def online(self):
        """The on-line smoothers among the collectors."""
        return [c for c in self._collectors[self._n_default:] if isinstance(c, OnlineSmootherMixin)]

    @property
    def device_rows(self):
        """The collectors whose per-step work stays on the device (on-line smoothers, ``Var``, ``Var_logLt``)."""
        return [c for c in self._collectors[self._n_default:] if isinstance(c, DeviceRowsMixin)]

    def device_moments(self, fk):
        """True when every non-default collector other than the device-row collectors (on-line smoothers, ``Var``,
        ``Var_logLt``) is ``Moments()`` with the default ``mom_func`` and the model keeps
        ``FeynmanKac.default_moments`` (resampling.wmean_and_var): exactly what the fused step kernel accumulates."""
        extra = [c for c in self._collectors[self._n_default:] if not isinstance(c, DeviceRowsMixin)]
        if not extra or not all(type(c) is Moments and c.mom_func is None for c in extra):
            return False
        dm = getattr(type(fk), "default_moments", None)
        return getattr(dm, "__qualname__", "") == "FeynmanKac.default_moments"

    def collect(self, smc):
        for col in self._collectors:
            if type(col) is Moments and col.mom_func is None and getattr(smc, "_dev_moments", False):
                col.summary.append(_moments_row(smc._engine.mom[smc._done - 1].cpu().numpy(), smc._engine.dim))
            else:
                col.collect(smc)

    def _extend_moments(self, table, dim):
        """Bulk fill of every ``Moments`` collector from the (T, 8) device table (fused ``run()``)."""
        rows = [_moments_row(r, dim) for r in table]
        for col in self._collectors[self._n_default:]:
            if type(col) is Moments:
                col.summary.extend(dict(r) for r in rows)

    def _extend_defaults(self, ess, loglt, rs):
        """Bulk fill of the default collectors, e.g. with ``default_summaries`` of a device table."""
        self.ESSs.extend(ess)
        self.logLts.extend(loglt)
        self.rs_flags.extend(rs)


def default_summaries(table):
    """Rows of a (T, 4) summary table (ESS, logLt, rs_flag, log_mean_w) -> what the default collectors hold for
    them: the ESSs and logLts as floats, the rs_flags as bools."""
    return [float(v) for v in table[:, 0]], [float(v) for v in table[:, 1]], [bool(v) for v in table[:, 2]]


def _moments_row(r, dim):
    """One row of the device table -> what resampling.wmean_and_var returns (resampling.py:320-338)."""
    if dim == 1:
        return {"mean": float(r[0]), "var": float(r[4])}
    return {"mean": r[:dim].copy(), "var": r[4:4 + dim].copy()}


def default_moments(W, X):
    return rs.wmean_and_var(W, X)
