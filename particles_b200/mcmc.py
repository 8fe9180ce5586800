"""Particle MCMC (particles/mcmc.py): PMMH over the device filter bank, conditional SMC and Particle Gibbs on the
conditional-filter kernel (csrc/smcb_pmcmc.cu, DESIGN.md section 5.9).

Both samplers take ``nchains`` (default 1): K independent chains advanced together, one launch per iteration for
all of them.  With ``nchains=1`` the chain has the reference's layout: ``chain.theta`` / ``chain.lpost`` (niter,);
with K > 1 they are (niter, K).

Two deliberate deviations from the reference:

* the pinned particle of ``CSMC`` is weighted by logG(t, x*[t-1], x*[t]).  The reference's ``CSMC.resample_move``
  resets ``X[0]`` and ``A[0]`` but not ``Xp[0]``, so its weight uses the discarded resampled ancestor; that changes
  the result of every Guided kind and of StochVolLeverage, whose PY depends on xp;
* ``GenericGibbs.step`` draws x_n given theta_n.  The reference passes theta_{n-1} to ``update_states`` right after
  drawing theta_n, a simultaneous update that does not leave the joint posterior invariant.
"""
import ctypes as C

import numpy as np
import torch
from scipy.linalg import LinAlgError, cholesky

from . import _lib
from .device import as_device, context, empty, ptr


def msjd(theta):
    """Mean squared jumping distance of a structured array of draws (mcmc.py:105-118)."""
    s = 0.0
    for p in theta.dtype.names:
        s += np.sum(np.diff(theta[p], axis=0) ** 2)
    return s


class _Chain:
    """The chain's fields (``theta``, ``lpost``, ``x``): host arrays, the reference's ``ThetaParticles`` layout."""

    def __init__(self, **fields):
        self.__dict__.update(fields)

    @property
    def N(self):
        return self.theta.shape[0]


class MCMC:
    """MCMC base class (mcmc.py:121-182): subclasses define ``step0()`` and ``step(n)``."""

    def __init__(self, niter=10, verbose=0):
        self.niter = niter
        self.verbose = verbose

    def step0(self):
        raise NotImplementedError

    def step(self, n):
        raise NotImplementedError

    def mean_sq_jump_dist(self, discard_frac=0.1):
        discard = int(self.niter * discard_frac)
        return msjd(self.chain.theta[discard:])

    def print_progress(self, n):
        params = self.chain.theta.dtype.fields.keys()
        msg = "Iteration %i" % n
        if hasattr(self, "nacc") and n > 0:
            msg += ", acc. rate=%s" % np.round(np.asarray(self.nacc) / n, 3)
        for p in params:
            msg += f", {p}={self.chain.theta[p][n]}"
        print(msg)

    def run(self):
        for n in range(self.niter):
            if n == 0:
                self.step0()
            else:
                self.step(n)
            if self.verbose > 0 and (n * self.verbose) % self.niter == 0:
                self.print_progress(n)


class VanishCovTracker:
    r"""Running mean and covariance of the points t^(-alpha) X_t (mcmc.py:188-220)."""

    def __init__(self, alpha=0.6, dim=1, mu0=None, Sigma0=None):
        self.alpha = alpha
        self.t = 0
        self.mu = np.zeros(dim) if mu0 is None else mu0
        if Sigma0 is None:
            self.Sigma = np.eye(dim)
            self.L0 = np.eye(dim)
        else:
            self.Sigma = Sigma0
            self.L0 = cholesky(Sigma0, lower=True)
        self.L = self.L0.copy()

    def gamma(self):
        return (self.t + 1) ** (-self.alpha)

    def update(self, v):
        self.t += 1
        g = self.gamma()
        self.mu = (1.0 - g) * self.mu + g * v
        mv = v - self.mu
        self.Sigma = (1.0 - g) * self.Sigma + g * np.dot(mv[:, np.newaxis], mv[np.newaxis, :])
        try:
            self.L = cholesky(self.Sigma, lower=True)
        except LinAlgError:
            self.L = self.L0


def _names(prior):
    """The prior's fields, in the order of its structured draws."""
    dt = getattr(prior, "dtype", None)
    return list(np.dtype(dt).names if dt is not None else prior.rvs(size=1).dtype.names)


def _struct(rows, names):
    out = np.empty(rows.shape[0], dtype=[(k, float) for k in names])
    for i, k in enumerate(names):
        out[k] = rows[:, i]
    return out


def _rows(theta, names):
    theta = np.atleast_1d(theta)
    return np.stack([np.asarray(theta[k], dtype=np.float64).reshape(-1) for k in names], axis=1)


def _starting_rows(prior, theta0, K, names):
    th = prior.rvs(size=K) if theta0 is None else np.atleast_1d(theta0)
    rows = _rows(th, names)
    return np.ascontiguousarray(np.broadcast_to(rows, (K, len(names))))


def _device_seed():
    """64 bits from the device generator (``SMC(seed=s)`` / ``device.seed`` fix them)."""
    ctx = context()
    u = empty(2)
    _lib.check(ctx.lib.smcb_uniform(ctx.handle, ptr(u), 2))
    hi, lo = (int(v * 2.0 ** 32) for v in u.cpu().numpy())
    return (hi << 32) | lo


class GenericRWHM(MCMC):
    """Random-walk Hastings-Metropolis over K independent chains (mcmc.py:223-301); the subclass provides ``prior``
    and ``compute_post``.

    ``noise``: None, or a dict ``{'z': (niter, K, d), 'u': (niter, K)}`` of the proposal normals and the acceptance
    uniforms of every iteration (entry n is used at step n).  Without it both are drawn from the device generator
    when the chain starts, so ``seed`` fixes every bit; ``seed`` re-seeds the package's device generator
    (``device.seed``) for that draw, as ``SMC(seed=...)`` does, which changes the stream every later user of it
    sees."""

    def __init__(self, niter=10, verbose=0, theta0=None, adaptive=True, scale=1.0, rw_cov=None, nchains=1,
                 seed=None, noise=None):
        self.niter, self.verbose, self.theta0, self.adaptive = niter, verbose, theta0, adaptive
        self.K, self.seed, self.noise = int(nchains), seed, noise
        self.names = _names(self.prior)
        self.dim = len(self.names)
        shape = (niter,) if self.K == 1 else (niter, self.K)
        self.chain = _Chain(theta=np.empty(shape, dtype=[(k, float) for k in self.names]), lpost=np.empty(shape))
        self.arr = np.empty((niter, self.K, self.dim))
        self.lpost = np.empty((niter, self.K))
        self._nacc = np.zeros(self.K, dtype=np.int64)
        if self.adaptive:
            self.scale = scale * 2.38 / np.sqrt(self.dim)
            self.cov_tracker = [VanishCovTracker(dim=self.dim, Sigma0=rw_cov) for _ in range(self.K)]
            self.L = [self.scale * c.L for c in self.cov_tracker]
        else:
            L = np.eye(self.dim) if rw_cov is None else cholesky(rw_cov, lower=True)
            self.L = [L] * self.K

    @property
    def nacc(self):
        return int(self._nacc[0]) if self.K == 1 else self._nacc

    def _draws(self):
        if self.noise is not None:
            z = np.asarray(self.noise["z"], dtype=np.float64).reshape(self.niter, self.K, self.dim)
            u = np.asarray(self.noise["u"], dtype=np.float64).reshape(self.niter, self.K)
            return z, u
        from . import device
        if self.seed is not None:
            device.seed(self.seed)
        ctx = context()
        nz, nu = self.niter * self.K * self.dim, self.niter * self.K
        buf = empty(nz + nu)
        _lib.check(ctx.lib.smcb_standard_normal(ctx.handle, ptr(buf), nz))
        _lib.check(ctx.lib.smcb_uniform(ctx.handle, ptr(buf[nz:]), nu))
        h = buf.cpu().numpy()
        return h[:nz].reshape(self.niter, self.K, self.dim), h[nz:].reshape(self.niter, self.K)

    def _record(self, n):
        th = _struct(self.arr[n], self.names)
        if self.K == 1:
            self.chain.theta[n] = th[0]
            self.chain.lpost[n] = self.lpost[n, 0]
        else:
            self.chain.theta[n] = th
            self.chain.lpost[n] = self.lpost[n]

    def compute_post(self, rows):
        """log-posterior (K,) at the parameter rows (K, d)."""
        raise NotImplementedError

    def step0(self):
        self._z, self._u = self._draws()
        self.arr[0] = _starting_rows(self.prior, self.theta0, self.K, self.names)
        self.lpost[0] = self.compute_post(self.arr[0])
        self._record(0)

    def step(self, n):
        prop = np.empty((self.K, self.dim))
        for k in range(self.K):
            prop[k] = self.arr[n - 1, k] + np.dot(self.L[k], self._z[n, k])
        lp = self.compute_post(prop)
        acc = np.log(self._u[n]) < lp - self.lpost[n - 1]
        self.arr[n] = np.where(acc[:, None], prop, self.arr[n - 1])
        self.lpost[n] = np.where(acc, lp, self.lpost[n - 1])
        self._nacc += acc
        if self.adaptive:
            for k in range(self.K):
                self.cov_tracker[k].update(self.arr[n, k])
                self.L[k] = self.scale * self.cov_tracker[k].L
        self._record(n)

    @property
    def acc_rate(self):
        return self.nacc / (self.niter - 1)


def _check_fk(fk_cls, tmap, who):
    from .state_space_models import _FK_KINDS
    kind = dict(_FK_KINDS).get(getattr(fk_cls, "__name__", None))
    if kind not in (_lib.FK_BOOTSTRAP, _lib.FK_GUIDED) or (kind == _lib.FK_GUIDED and not tmap.proposal):
        raise NotImplementedError("%s: Feynman-Kac class %r is not built for %s on the device" % (who, fk_cls, tmap.name))
    return kind


class PMMH(GenericRWHM):
    """Particle marginal Metropolis-Hastings (mcmc.py:342-439): the log-likelihood of each proposal is the estimate
    of a particle filter of Nx particles.  The proposals of one iteration (one per chain) are the rows of one
    ``bank.FilterBank``, re-run from step 0 in one launch (those with a finite prior only) with fresh keys.

    ``ssm_cls`` must be a stock 1-D model (``bank.SUPPORTED``) and ``fk_cls`` Bootstrap or GuidedPF;
    ``smc_options`` passes ``resampling`` (one of the fused schemes) and ``ESSrmin``; ``qmc`` and an ``smc_cls``
    other than this package's or the reference's ``SMC`` raise NotImplementedError.  ``prior`` is duck-typed and
    evaluated on the host.  ``loglik`` is the one method to override to replace the filter."""

    def __init__(self, niter=10, verbose=0, ssm_cls=None, smc_cls=None, prior=None, data=None, smc_options=None,
                 fk_cls=None, Nx=100, theta0=None, adaptive=True, scale=1.0, rw_cov=None, nchains=1, seed=None,
                 noise=None):
        from .bank import ThetaMap
        from .state_space_models import Bootstrap, _flat_data
        if smc_cls is not None and not (getattr(smc_cls, "__name__", None) == "SMC" and getattr(
                smc_cls, "__module__", None) in ("particles.core", "particles_b200.core")):
            raise NotImplementedError("PMMH on the device runs the package's (or the reference's) SMC, not %r"
                                      % (smc_cls,))
        self.smc_options = {"collect": "off"}
        if smc_options is not None:
            self.smc_options.update(smc_options)
        if self.smc_options.get("qmc"):
            raise NotImplementedError("PMMH over SQMC filters (qmc=True) is not built")
        self.resampling = self.smc_options.get("resampling", "systematic")
        if self.resampling not in _lib.FUSED_SCHEMES:
            raise NotImplementedError("PMMH: the filters resample with one of %s" % (_lib.FUSED_SCHEMES,))
        self.ESSrmin = float(self.smc_options.get("ESSrmin", 0.5))
        self.ssm_cls, self.smc_cls, self.prior, self.data, self.Nx = ssm_cls, smc_cls, prior, data, int(Nx)
        self.fk_cls = Bootstrap if fk_cls is None else fk_cls
        GenericRWHM.__init__(self, niter=niter, verbose=verbose, theta0=theta0, adaptive=adaptive, scale=scale,
                             rw_cov=rw_cov, nchains=nchains, seed=seed, noise=noise)
        self._map = ThetaMap(ssm_cls, self.names, _flat_data(data, 1).reshape(-1))
        self.fk_kind = _check_fk(self.fk_cls, self._map, "PMMH")
        self._bank = None
        self.timer = None          # None, or a list that receives (start, end) CUDA events around each bank launch

    def compute_post(self, rows):
        lp = np.array(np.broadcast_to(np.asarray(self.prior.logpdf(_struct(rows, self.names)), dtype=np.float64),
                                      (rows.shape[0],)))
        ok = np.flatnonzero(np.isfinite(lp))
        if ok.size:
            lp[ok] += self.loglik(_struct(rows[ok], self.names))
        return lp

    def loglik(self, theta):
        """log-likelihood estimates (m,) at the structured array theta (m,) of proposals with a finite prior: one
        bank launch."""
        from .bank import FilterBank
        from .smc_samplers import _KeyCounter
        m = self._map
        if self._bank is None:
            if self.seed is None:
                self.seed = _device_seed()
            self._keys = _KeyCounter(self.seed)
            self._bank = FilterBank(m.model, self.fk_kind, self.resampling, self.Nx, self.K, as_device(m.data),
                                    m.n_params, self.ESSrmin,
                                    shared_sc=None if m.shared_sc is None else as_device(m.shared_sc),
                                    per_filter_sc=m.name == "Gordon_etal")
        b = self._bank
        b.timer = self.timer
        rows = _rows(theta, self.names)
        n = rows.shape[0]
        params = np.zeros((self.K, m.n_params))
        params[:n] = m.params(rows)
        sc = None
        if b.sc is not None:
            sc = np.zeros((self.K, m.T))
            sc[:n] = m.step_consts(rows)
        b.set_rows(params, sc)
        b.fresh_keys(self._keys.seed, self._keys.take(self.K))
        b.advance(m.T, idx=torch.arange(n, dtype=torch.int64, device=b.data.device), restart=True)
        return b.logLt[:n].cpu().numpy()


# ---------------------------------------------------------------------------------------------- conditional SMC
class _CsmcRuns:
    """Device rows of R conditional filters (X, lw, A (R, T, ld), trajectories, logLt) and the one launch that runs
    them all (smcb_csmc_run)."""

    def __init__(self, tmap, fk_kind, N, R, essrmin, draw):
        self.map, self.fk, self.N, self.R, self.essrmin = tmap, fk_kind, int(N), int(R), float(essrmin)
        self.T = tmap.T
        self.ld = self.N + (self.N & 1)
        self.draw = _lib.CSMC_BACKWARD if draw == "backward" else _lib.CSMC_GENEALOGY
        self.data = as_device(tmap.data)
        dev = self.data.device
        f64 = dict(dtype=torch.float64, device=dev)
        R, T, ld = self.R, self.T, self.ld
        self.X = torch.empty((R, T, ld), **f64)
        self.lw = torch.empty((R, T, ld), **f64)
        self.A = torch.empty((R, T, ld), dtype=torch.int64, device=dev)
        self.traj = torch.empty((R, T), **f64)
        self.xstar = torch.zeros((R, T), **f64)
        self.logLt = torch.empty(R, **f64)
        self.key = torch.empty(R, dtype=torch.int64, device=dev)
        self.params = torch.empty((R, tmap.n_params), **f64)
        self.sc = None if tmap.name != "Gordon_etal" else torch.empty((R, T), **f64)
        self.shared_sc = None if tmap.shared_sc is None else as_device(tmap.shared_sc)
        self.timer = None
        self.plan()

    def desc(self, pin=False, noise=None, summaries=None):
        d = _lib.CsmcDesc()
        d.model, d.fk, d.n_params, d.draw, d.pin = self.map.model, self.fk, self.map.n_params, self.draw, int(pin)
        d.N, d.T, d.R, d.essrmin = self.N, self.T, self.R, self.essrmin
        d.key, d.params = ptr(self.key), ptr(self.params)
        d.data, d.data_ld = ptr(self.data), (self.T if self.data.dim() == 2 else 0)
        if self.sc is not None:
            d.step_consts, d.sc_ld = ptr(self.sc), self.T
        elif self.shared_sc is not None:
            d.step_consts, d.sc_ld = ptr(self.shared_sc), 0
        d.xstar, d.X, d.lw, d.A = ptr(self.xstar), ptr(self.X), ptr(self.lw), ptr(self.A)
        d.traj, d.logLt, d.summaries = ptr(self.traj), ptr(self.logLt), ptr(summaries)
        if noise is not None:
            d.z_in, d.u_in, d.ud_in = (ptr(noise.get(k)) for k in ("z", "u", "ud"))
        return d

    def plan(self):
        """(the largest N this device holds, grid); NotImplementedError above the bound."""
        out = (C.c_int64 * 2)()
        ctx = context()
        _lib.check(ctx.lib.smcb_csmc_plan(ctx.handle, C.byref(self.desc()), out))
        return int(out[0]), int(out[1])

    def set_rows(self, rows, keys):
        """Model constants of the parameter rows (R, d) and the keys number keys.take(R) under the counter's seed."""
        self.params.copy_(torch.from_numpy(self.map.params(rows)))
        if self.sc is not None:
            self.sc.copy_(torch.from_numpy(self.map.step_consts(rows)))
        ctx = context()
        _lib.check(ctx.lib.smcb_bank_keys(ctx.handle, ptr(self.key), self.R, keys.seed, keys.take(self.R)))

    def run(self, pin, noise=None, summaries=None):
        ctx = context()
        ctx.bind_stream()
        ev = None
        if self.timer is not None:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        _lib.check(ctx.lib.smcb_csmc_run(ctx.handle, C.byref(self.desc(pin, noise, summaries))))
        if ev is not None:
            ev[1].record()
            self.timer.append(ev)


def _model_of(fk):
    """(ThetaMap, kind, parameter row) of a Feynman-Kac object built on a stock 1-D model."""
    from .bank import ThetaMap
    from .state_space_models import _flat_data
    ssm = fk.ssm
    cls = type(ssm)
    tmap0 = ThetaMap(cls, [], _flat_data(fk.data, 1).reshape(-1))
    names = [k for k in tmap0.defaults if getattr(ssm, k, None) is not None]
    tmap = ThetaMap(cls, names, tmap0.data)
    row = np.array([[float(getattr(ssm, k)) for k in names]])
    return tmap, _check_fk(type(fk), tmap, "CSMC"), row


class CSMC:
    """Conditional SMC (mcmc.py:453-475) on the device: multinomial resampling when ESS < ESSrmin N, the whole
    history kept, slot 0 pinned to ``xstar`` (an unconditional run when it is None).  ``fk``: Bootstrap or GuidedPF
    of a stock 1-D model (``bank.SUPPORTED``).  The pinned particle is weighted by logG(t, x*[t-1], x*[t]) (see the
    module docstring).  ``run()`` sets ``logLt``, ``hist`` (a ``smoothing.ParticleHistory`` on the device rows, so
    ``hist.extract_one_trajectory()`` and ``hist.backward_sampling_ON2(M)`` work) and ``traj``, the trajectory the
    kernel drew by tracing ancestors.  N is bounded by shared memory (about 1e4): above it, NotImplementedError."""

    def __init__(self, fk=None, N=100, ESSrmin=0.5, xstar=None, seed=None):
        self.fk, self.N, self.ESSrmin, self.xstar, self.seed = fk, int(N), ESSrmin, xstar, seed
        self._map, self._kind, self._row = _model_of(fk)
        self.T = self._map.T

    def run(self):
        from . import resampling as rs
        from .smc_samplers import _KeyCounter
        from .smoothing import ParticleHistory
        runs = _CsmcRuns(self._map, self._kind, self.N, 1, self.ESSrmin, "genealogy")
        seed = _device_seed() if self.seed is None else self.seed
        runs.set_rows(self._row, _KeyCounter(seed))
        pin = self.xstar is not None
        if pin:
            runs.xstar[0] = as_device(np.asarray([float(v) for v in self.xstar]))
        runs.run(pin)
        self.logLt = float(runs.logLt[0])
        self.traj = list(runs.traj[0].cpu().numpy())
        h = ParticleHistory(self.fk, False)
        N = self.N
        for t in range(self.T):
            h.X.append(runs.X[0, t, :N])
            h.A.append(runs.A[0, t, :N])
            h.wgts.append(rs.Weights(lw=runs.lw[0, t, :N]))
        self.hist = h
        self.X, self.A, self.wgts = h.X[-1], h.A[-1], h.wgts[-1]


# ---------------------------------------------------------------------------------------------- Gibbs samplers
class GenericGibbs(MCMC):
    """Gibbs sampler for a state-space model (mcmc.py:481-529) over K chains: x_n is drawn given theta_n (see the
    module docstring).  Subclasses define ``update_theta(theta, x)`` (one chain) and ``update_states``."""

    def __init__(self, niter=10, verbose=10, theta0=None, ssm_cls=None, prior=None, data=None, store_x=False,
                 nchains=1):
        self.ssm_cls, self.prior, self.data, self.theta0 = ssm_cls, prior, data, theta0
        self.niter, self.store_x, self.verbose, self.K = niter, store_x, verbose, int(nchains)
        self.names = _names(self.prior)
        shape = (niter,) if self.K == 1 else (niter, self.K)
        theta = np.empty(shape, dtype=[(k, float) for k in self.names])
        fields = dict(theta=theta)
        if store_x:
            fields["x"] = np.empty(shape + (len(data),))
        self.chain = _Chain(**fields)

    def _theta_of(self, n, k):
        return self.chain.theta[n] if self.K == 1 else self.chain.theta[n, k]

    def update_states(self, n):
        """Draw the states of every chain given chain.theta[n] (x of iteration n - 1 as the reference path)."""
        raise NotImplementedError

    def update_theta(self, theta, x):
        raise NotImplementedError

    def step0(self):
        if getattr(self, "seed", None) is not None:     # the prior draw and the re-simulated data come from it
            from . import device
            device.seed(self.seed)
        th = _starting_rows(self.prior, self.theta0, self.K, self.names)
        self.chain.theta[0] = _struct(th, self.names)[0] if self.K == 1 else _struct(th, self.names)
        self.x = self.update_states(0)
        self._store(0)

    def step(self, n):
        for k in range(self.K):
            new = self.update_theta(self._theta_of(n - 1, k), list(self.x[k]))
            if self.K == 1:
                self.chain.theta[n] = new
            else:
                self.chain.theta[n, k] = new
        self.x = self.update_states(n)
        self._store(n)

    def _store(self, n):
        if self.store_x:
            self.chain.x[n] = self.x[0] if self.K == 1 else self.x


class ParticleGibbs(GenericGibbs):
    """Particle Gibbs (mcmc.py:532-609) on the device: the states of all K chains are drawn by ONE conditional-SMC
    launch per iteration (the pin off at iteration 0), which also draws the new trajectories -- by tracing ancestors,
    or with ``backward_step`` one backward draw per step -- followed by one copy of the (K, T) trajectories to the
    host.  ``update_theta(theta, x)`` stays user code: it is called once per chain with the chain's record and x, a
    list of T NumPy float64 scalars.  ``regenerate_data`` re-simulates each chain's data given its new trajectory,
    one vectorised draw of the model's PY per t (this package's models draw from the device generator, the
    reference's from NumPy's global stream); it is refused for DiscreteCox, whose step constants log(y!) are computed
    once from the data.  ``seed`` fixes the filters' keys and re-seeds the package's device generator
    (``device.seed``) when the chain starts, so the prior draw and the re-simulated data follow it too; like
    ``SMC(seed=...)``, this changes the stream every later user of the device generator sees.  By default the keys
    come from the device generator."""

    def __init__(self, niter=10, verbose=0, ssm_cls=None, prior=None, data=None, theta0=None, Nx=100, fk_cls=None,
                 regenerate_data=False, backward_step=False, store_x=False, nchains=1, seed=None):
        from .bank import ThetaMap
        from .state_space_models import Bootstrap, _flat_data
        GenericGibbs.__init__(self, niter=niter, verbose=verbose, ssm_cls=ssm_cls, prior=prior, data=data,
                              theta0=theta0, store_x=store_x, nchains=nchains)
        self.Nx = int(Nx)
        self.fk_cls = Bootstrap if fk_cls is None else fk_cls
        self.regenerate_data, self.backward_step, self.seed = regenerate_data, backward_step, seed
        self._map = ThetaMap(ssm_cls, self.names, _flat_data(data, 1).reshape(-1))
        self.fk_kind = _check_fk(self.fk_cls, self._map, "ParticleGibbs")
        if regenerate_data and self._map.shared_sc is not None:
            raise NotImplementedError("ParticleGibbs: regenerate_data is not built for %s (its step constants are "
                                      "computed once from the data)" % self._map.name)
        self._runs = None
        self.timer = None

    def update_states(self, n):
        from .smc_samplers import _KeyCounter
        if self._runs is None:
            self._runs = _CsmcRuns(self._map, self.fk_kind, self.Nx, self.K, 0.5,
                                   "backward" if self.backward_step else "genealogy")
            if self.seed is None:
                self.seed = _device_seed()
            self._keys = _KeyCounter(self.seed)
            if self.regenerate_data:
                self._runs.data = as_device(np.broadcast_to(self._map.data, (self.K, self._map.T)).copy())
        r = self._runs
        r.timer = self.timer
        th = self.chain.theta[n]
        rows = _rows(th, self.names)
        r.set_rows(rows, self._keys)
        if n > 0:
            r.xstar.copy_(torch.from_numpy(np.ascontiguousarray(self.x)))
        r.run(pin=n > 0)
        x = r.traj.cpu().numpy()
        if self.regenerate_data:
            r.data.copy_(torch.from_numpy(self._simulate_given_x(rows, x)))
        return x

    def _simulate_given_x(self, rows, x):
        """(K, T) data: y_t ~ PY(t, x_{t-1}, x_t) of each chain's model, one draw over the chains per t
        (StateSpaceModel.simulate_given_x); this package's models take the states as a CUDA tensor."""
        ssm = self.ssm_cls(**{k: rows[:, i] for i, k in enumerate(self.names)})
        native = getattr(self.ssm_cls, "__module__", "").startswith("particles_b200")
        xs = as_device(x) if native else x
        T = x.shape[1]
        y = np.empty((self.K, T))
        for t in range(T):
            v = ssm.PY(t, None if t == 0 else xs[:, t - 1], xs[:, t]).rvs(size=self.K)
            y[:, t] = (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)).reshape(self.K)
        return y
