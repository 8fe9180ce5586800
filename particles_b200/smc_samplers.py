"""SMC samplers on the device: tempering / adaptive tempering and IBIS with standard or waste-free MCMC
moves -- the part of ``particles/smc_samplers.py`` that BASELINE config 5 exercises (file:line
cited per class).  They are Feynman-Kac models for ``particles_b200.SMC`` (plugin path):

    model = LogisticRegression(data=flipped_predictors, prior_scale=5.)
    fk = AdaptiveTempering(model=model, wastefree=True, len_chain=100)
    pf = particles_b200.SMC(fk=fk, N=10_000, ESSrmin=1.)      # N * len_chain particles
    pf.run();  pf.logLt;  pf.X.theta;  pf.X.shared["exponents"]

Particles are a ``ThetaParticles`` of CUDA tensors; the per-particle work (tempered target of
the model, random-walk proposal, Metropolis accept/copy, resampling, weights) runs in libsmcb
kernels; the O(d^2) calibration of the proposal (weighted covariance + Cholesky) and the scalar
root-find for the next exponent (scipy.optimize.brentq, as in the reference) run on the host.
"""
import ctypes as C

import numpy as np
import torch
from scipy import optimize

from . import _lib
from . import resampling as rs
from .binary_smc import BinaryMetropolis
from .core import FeynmanKac
from .device import as_device, context, empty, ptr


class ThetaParticles:
    """smc_samplers.py:401-500: N particles packed as named CUDA tensors (``theta`` (N, d),
    ``lprior``, ``llik``, ``lpost`` (N,)) plus a ``shared`` dict; fancy indexing by an int64
    ancestor tensor returns a new object (gather kernels), as the reference's class does."""

    def __init__(self, shared=None, **fields):
        self.shared = {} if shared is None else shared
        self.__dict__.update(fields)

    @property
    def dict_fields(self):
        return {k: v for k, v in self.__dict__.items() if k != "shared"}

    @property
    def N(self):
        return len(next(iter(self.dict_fields.values())))

    def __getitem__(self, key):
        if not (isinstance(key, torch.Tensor) and key.dtype == torch.int64):
            return self.__class__(shared=self.shared.copy(),
                                  **{k: v[key] for k, v in self.dict_fields.items()})
        ctx = context(key.device)
        out = {}
        for k, v in self.dict_fields.items():
            if v.dtype != torch.float64:          # e.g. the (N, p) bool theta of binary_smc: a plain row copy
                out[k] = v.index_select(0, key)
                continue
            d = 1 if v.ndim == 1 else v.shape[1]
            o = torch.empty((key.shape[0],) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
            _lib.check(ctx.lib.smcb_gather_rows(ctx.handle, ptr(v), v.shape[0], ptr(key), key.shape[0], d,
                                                ptr(o)))
            out[k] = o
        return self.__class__(shared=self.shared.copy(), **out)

    def copy(self):
        return self.__class__(shared=self.shared.copy(),
                              **{k: v.clone() for k, v in self.dict_fields.items()})

    @classmethod
    def concatenate(cls, *xs):
        fields = {k: torch.cat([getattr(x, k) for x in xs]) for k in xs[0].dict_fields}
        return cls(shared=xs[0].shared.copy(), **fields)


class LogisticRegression:
    """Bayesian logistic regression static model (book/smc_samplers/logistic_reg.py:60-67):
    ``data`` = (n_data, d) predictors with the response sign folded in (datasets.py:286-292),
    prior beta ~ MvNormal(scale=prior_scale, cov=I_d).  ``target(x, epn)`` fills
    ``x.lprior / x.llik / x.lpost`` (Tempering.current_target, smc_samplers.py:836-845)."""

    def __init__(self, data=None, prior_scale=5.0):
        self.data_host = np.ascontiguousarray(np.asarray(data, dtype=np.float64))
        self.data = as_device(self.data_host)
        self.prior_scale = float(prior_scale)
        self.d = self.data_host.shape[1]

    @property
    def T(self):
        return self.data_host.shape[0]

    def prior_rvs(self, size):
        ctx = context()
        z = empty(size * self.d)
        _lib.check(ctx.lib.smcb_standard_normal(ctx.handle, ptr(z), size * self.d))
        return (self.prior_scale * z).reshape(size, self.d)     # loc + scale * (z @ I)

    def _rows(self, n_rows, epn):
        """(rows, exponent) of the kernels' call for the posterior given the first ``n_rows`` data rows (None: all of
        them).  No rows is the prior alone: one row at exponent 0, whose log-likelihood the caller then zeroes."""
        rows = self.T if n_rows is None else int(n_rows)
        return (1, 0.0) if rows == 0 else (rows, float(epn))

    def wf_move(self, x, epn, P, noise=None, n_rows=None, lmin=None):
        """Fused waste-free move (smcb_logistic_wf_move): x = the M resampled particles with their
        lprior / llik / lpost at exponent ``epn`` and ``shared['chol_cov']``; returns P*M particles.
        ``n_rows``: target the posterior given the first n_rows data rows only (IBIS).  ``lmin``: target the prior
        truncated to llik >= lmin instead (nested sampling SMC, smcb_logistic_ns_move; ``epn`` is then unused)."""
        ctx = context()
        M, d = x.theta.shape
        rows, epn = self._rows(n_rows, epn)
        out = x.__class__(shared=x.shared.copy(), theta=empty((P * M, d)), lprior=empty(P * M),
                          llik=empty(P * M), lpost=empty(P * M))
        pb = empty((P - 1, M))
        z = u = None
        if noise is not None:
            z, u = as_device(noise[0]), as_device(noise[1])
        move = ctx.lib.smcb_logistic_wf_move if lmin is None else ctx.lib.smcb_logistic_ns_move
        _lib.check(move(
            ctx.handle, M, d, P, ptr(x.theta), ptr(x.lprior), ptr(x.llik), ptr(x.lpost), ptr(self.data), rows,
            self.prior_scale, epn if lmin is None else float(lmin), ptr(x.shared["chol_cov"]), ptr(z), ptr(u),
            ptr(out.theta), ptr(out.lprior), ptr(out.llik), ptr(out.lpost), ptr(pb)))
        if n_rows == 0:
            out.llik.zero_()
        out.shared["acc_rates"] = x.shared.get("acc_rates", []) + [pb.mean(dim=1)]
        return out

    def target(self, x, epn, n_rows=None, lmin=None):
        """lprior / llik / lpost of x at exponent ``epn`` (smcb_logistic_target); ``n_rows``: the posterior given
        the first n_rows data rows only (IBIS.current_target, n_rows = t + 1); ``lmin``: lpost = lprior where
        llik >= lmin, -inf elsewhere instead (NestedSamplingSMC.current_target, smcb_logistic_ns_target)."""
        ctx = context()
        n = x.theta.shape[0]
        rows, epn = self._rows(n_rows, epn)
        x.lprior, x.llik, x.lpost = empty(n), empty(n), empty(n)
        target = ctx.lib.smcb_logistic_target if lmin is None else ctx.lib.smcb_logistic_ns_target
        _lib.check(target(ctx.handle, ptr(x.theta), n, self.d, ptr(self.data), rows, self.prior_scale,
                          epn if lmin is None else float(lmin), ptr(x.lprior), ptr(x.llik), ptr(x.lpost)))
        if n_rows == 0:
            x.llik.zero_()

    def logpyt_rows(self, theta, r0, K, lw, lpost=None, llik=None, scratch=None):
        """IBIS reweighting over the data rows [r0, r0 + K) (smcb_logistic_logpyt), one row at a time in row order:
        with ``scratch`` (K, n), row k receives lw + the rows r0 .. r0 + k and nothing else is written (scan);
        without it, lw and -- when given -- lpost and llik are incremented in place (commit)."""
        ctx = context()
        n = theta.shape[0]
        _lib.check(ctx.lib.smcb_logistic_logpyt(ctx.handle, ptr(theta), n, self.d, ptr(self.data), self.T, int(r0),
                                                int(K), int(scratch is None), ptr(lw), ptr(lpost), ptr(llik),
                                                ptr(scratch)))

    def logpyt(self, theta, t):
        """log p(y_t | theta) for the (N, d) CUDA tensor theta (StaticModel.logpyt): a one-row commit into zeros."""
        lpyt = torch.zeros(theta.shape[0], dtype=torch.float64, device=theta.device)
        self.logpyt_rows(theta, t, 1, lpyt)
        return lpyt


class ArrayRandomWalk:
    """Gaussian random-walk Metropolis, smc_samplers.py:596-629."""

    def calibrate(self, W, x):
        """smc_samplers.py:617-622: L = 2.38 / sqrt(d) * chol(wcov(W, theta)) -- weighted mean, covariance and the
        Cholesky factor all on the device (smcb_rw_calibrate), nothing comes back to the host."""
        theta = x.theta
        n, d = theta.shape
        ctx = context()
        L = empty(d * d).reshape(d, d)
        _lib.check(ctx.lib.smcb_rw_calibrate(ctx.handle, ptr(as_device(W)), ptr(theta), n, d, 2.38 / np.sqrt(d), ptr(L)))
        x.shared["chol_cov"] = L

    def step(self, x, target, noise=None):
        """ArrayMetropolis.step (601-611); returns the mean acceptance probability (device scalar)."""
        ctx = context()
        n, d = x.theta.shape
        xprop = x.__class__(theta=torch.empty_like(x.theta))
        z = None if noise is None else as_device(noise[0])
        _lib.check(ctx.lib.smcb_rw_propose(ctx.handle, ptr(x.theta), n, d, ptr(x.shared["chol_cov"]), ptr(z),
                                           ptr(xprop.theta)))
        target(xprop)
        u = None if noise is None else as_device(noise[1])
        acc = empty(1)
        _lib.check(ctx.lib.smcb_mh_accept(ctx.handle, n, d, ptr(x.theta), ptr(x.lprior), ptr(x.llik),
                                          ptr(x.lpost), ptr(xprop.theta), ptr(xprop.lprior), ptr(xprop.llik),
                                          ptr(xprop.lpost), ptr(u), ptr(acc)))
        return acc


class MCMCSequence:
    """smc_samplers.py:651-663."""

    def __init__(self, mcmc=None, len_chain=10):
        self.mcmc = ArrayRandomWalk() if mcmc is None else mcmc
        self.nsteps = len_chain - 1

    def calibrate(self, W, x):
        self.mcmc.calibrate(W, x)


class MCMCSequenceWF(MCMCSequence):
    """Waste-free: keep every intermediate state, smc_samplers.py:669-683."""

    def __call__(self, x, target, noise=None):
        fused = getattr(target, "fused_wf", None)
        if fused is not None and isinstance(self.mcmc, (ArrayRandomWalk, BinaryMetropolis)) and self.nsteps >= 1:
            return fused(x, self.nsteps + 1, noise)     # all chains, all steps: one kernel launch
        xs, ars = [x], []
        for _ in range(self.nsteps):
            x = x.copy()
            ars.append(self.mcmc.step(x, target))
            xs.append(x)
        xout = x.concatenate(*xs)
        xout.shared["acc_rates"] = x.shared.get("acc_rates", []) + [ars]
        return xout


class AdaptiveMCMCSequence(MCMCSequence):
    """Standard SMC sampler move: keep only the final states, smc_samplers.py:686-709
    (fixed number of steps; the adaptive stopping rule of the reference is not implemented)."""

    def __call__(self, x, target):
        xout, ars = x.copy(), []
        for _ in range(self.nsteps):
            ars.append(self.mcmc.step(xout, target))
        xout.shared["acc_rates"] = x.shared.get("acc_rates", []) + [ars]
        return xout


class FKSMCsampler(FeynmanKac):
    """smc_samplers.py:714-769."""

    def __init__(self, model=None, wastefree=True, len_chain=10, move=None):
        self.model, self.wastefree, self.len_chain = model, wastefree, len_chain
        if move is None:
            move = MCMCSequenceWF(len_chain=len_chain) if wastefree else AdaptiveMCMCSequence(len_chain=len_chain)
        self.move = move

    @property
    def T(self):
        return self.model.T

    def default_moments(self, W, x):
        return rs.wmean_and_var(W, x.theta)

    def summary_format(self, smc):
        return "t=%i, ESS=%.2f" % (smc.t, smc.wgts.ESS)

    def time_to_resample(self, smc):
        rs_flag = smc.aux.ESS < smc.X.N * smc.ESSrmin
        smc.X.shared["rs_flag"] = rs_flag
        if rs_flag:
            self.move.calibrate(smc.W, smc.X)
        return rs_flag

    def M0(self, N):
        return self._M0(N * self.len_chain if self.wastefree else N)


class Tempering(FKSMCsampler):
    """smc_samplers.py:797-874."""

    def __init__(self, model=None, wastefree=True, len_chain=10, move=None, exponents=None):
        super().__init__(model=model, wastefree=wastefree, len_chain=len_chain, move=move)
        self.exponents = exponents
        self.deltas = None if exponents is None else np.diff(exponents, prepend=0.0)

    @property
    def T(self):
        return len(self.exponents)

    def logG_tempering(self, x, delta):
        dl = delta * x.llik
        x.lpost = x.lpost + dl
        return dl

    def logG(self, t, xp, x):
        x.shared["exponents"].append(self.exponents[t])
        return self.logG_tempering(x, self.deltas[t])

    def current_target(self, epn):
        def func(x):
            self.model.target(x, epn)
        if hasattr(self.model, "wf_move"):      # lets MCMCSequenceWF run the whole move in one kernel
            func.fused_wf = lambda x, P, noise=None: self.model.wf_move(x, epn, P, noise)
        return func

    def _M0(self, N):
        x0 = ThetaParticles(theta=self.model.prior_rvs(N))
        x0.shared["exponents"] = [0.0]
        self.current_target(0.0)(x0)
        return x0

    def _M(self, t, xp, epn):
        return self.move(xp, self.current_target(epn))

    def M(self, t, xp):
        if xp.shared["rs_flag"]:
            return self._M(t, xp, self.exponents[t - 1])
        return xp


def next_annealing_epn(epn, alpha, lw):
    """smc_samplers.py:876-895: the exponent at which ESS(e * lw) = alpha * N.  The whole bracketing root-find runs on
    the device (smcb_next_annealing_epn: 16 candidate exponents per pass, 11 passes, bracket < 1e-13); the host reads
    the one resulting scalar, because the reference keeps the exponents as Python floats in ``shared``."""
    lw = as_device(lw)
    ctx = context()
    out = empty(1)
    _lib.check(ctx.lib.smcb_next_annealing_epn(ctx.handle, ptr(lw), lw.shape[0], float(epn), float(alpha), ptr(out)))
    return float(out.item())


def next_annealing_epn_host(epn, alpha, lw):
    """The reference's own formulation (brentq on the host, essl on the device): kept for the parity test."""
    N = lw.shape[0]

    def f(e):
        ess = rs.essl(e * lw) if e > 0.0 else N
        return ess - alpha * N

    if f(1.0 - epn) < 0.0:
        return epn + optimize.brentq(f, 0.0, 1.0 - epn)
    return 1.0


class AdaptiveTempering(Tempering):
    """smc_samplers.py:897-936."""

    def __init__(self, model=None, wastefree=True, len_chain=10, move=None, ESSrmin=0.5, max_iter=1000):
        FKSMCsampler.__init__(self, model=model, wastefree=wastefree, len_chain=len_chain, move=move)
        self.ESSrmin, self.max_iter = ESSrmin, max_iter

    @property
    def T(self):
        return self.max_iter

    def time_to_resample(self, smc):
        self.move.calibrate(smc.W, smc.X)
        return True

    def done(self, smc):
        if smc.t >= self.max_iter:
            return True
        if smc.X is None:
            return False
        return smc.X.shared["exponents"][-1] >= 1.0

    def logG(self, t, xp, x):
        epn = x.shared["exponents"][-1]
        new_epn = next_annealing_epn(epn, self.ESSrmin, x.llik)
        x.shared["exponents"].append(new_epn)
        return self.logG_tempering(x, new_epn - epn)

    def M(self, t, xp):
        xp.shared["rs_flag"] = True
        return self._M(t, xp, xp.shared["exponents"][-1])


# ----------------------------------------------------------------------------------------------------------- IBIS
def _layout(prior):
    """[(name, column slice)] of the (N, p) theta tensor, from the fields of the prior's structured dtype."""
    out, j = [], 0
    dt = np.dtype(prior.dtype)
    for name in dt.names:
        k = int(np.prod(dt[name].shape)) if dt[name].shape else 1
        out.append((name, slice(j, j + k) if dt[name].shape else j))
        j += k
    return out


class StaticModel:
    """smc_samplers.py:216-301: a static model given by its data and a ``StructDist`` prior; sub-classes define
    ``logpyt(theta, t)``.  User code runs on CUDA tensors: ``theta`` is a mapping from field name to a column view
    of the particles' (N, p) tensor (a (N,) column for a scalar field, (N, dim) for a vector field) and NumPy
    ``data`` is copied to the device once (``self.data``; the host copy is ``self.data_host``)."""

    def __init__(self, data=None, prior=None):
        self.data_host = data
        self.data = as_device(np.asarray(data, dtype=np.float64)) if isinstance(data, np.ndarray) else data
        self.prior = prior

    @property
    def T(self):
        return 0 if self.data is None else len(self.data)

    @property
    def dim(self):
        return sum(1 if isinstance(c, int) else c.stop - c.start for _, c in _layout(self.prior))

    def fields(self, theta):
        """{name: column view} of the (N, p) CUDA tensor theta."""
        return {name: theta[:, c] for name, c in _layout(self.prior)}

    def logpyt(self, theta, t):
        raise NotImplementedError("StaticModel: logpyt not implemented")

    def loglik(self, theta, t=None):
        """Sum of logpyt over the rows 0..t in row order (all rows if t is None), NaN mapped to -inf."""
        if t is None:
            t = self.T - 1
        ll = torch.zeros(theta.shape[0], dtype=torch.float64, device=theta.device)
        f = self.fields(theta)
        for s in range(t + 1):
            ll = ll + as_device(self.logpyt(f, s))
        return torch.nan_to_num(ll, nan=-float("inf"), posinf=float("inf"), neginf=-float("inf"))

    def logprior(self, theta):
        """The prior's log-density at the rows of the (N, p) tensor theta, as a CUDA tensor."""
        return as_device(np.asarray(self.prior.logpdf(self.to_struct(theta)), dtype=np.float64))

    def logpost(self, theta, t=None):
        return self.logprior(theta) + self.loglik(theta, t)

    def to_struct(self, theta):
        """(N, p) tensor -> NumPy structured array with the prior's fields."""
        th = theta.detach().cpu().numpy()
        out = np.empty(th.shape[0], dtype=self.prior.dtype)
        for name, c in _layout(self.prior):
            out[name] = th[:, c]
        return out

    def prior_rvs(self, size):
        """Prior draws as the (N, p) CUDA tensor of the particles."""
        th = self.prior.rvs(size=size)
        cols = [np.asarray(th[name], dtype=np.float64).reshape(size, -1) for name, _ in _layout(self.prior)]
        return as_device(np.ascontiguousarray(np.concatenate(cols, axis=1)))


def _device_likelihood(model):
    return hasattr(model, "logpyt_rows")


class IBIS(FKSMCsampler):
    """smc_samplers.py:772-794: data tempering -- the target at step t is the posterior given y_0..y_t.

    ``model`` is a ``StaticModel`` with a user ``logpyt`` (evaluated on CUDA tensors, one call per particle set and
    data row) or a model with a device likelihood (``LogisticRegression``: reweighting, targets and the waste-free
    move in libsmcb kernels, no per-row Python).  ``X.theta`` is the (N, d) CUDA tensor.  With a device likelihood,
    ``SMC.run()`` adds the data rows of a stretch of non-resampling steps with one host read (DESIGN.md 5.10).
    The adaptive stopping rule of ``AdaptiveMCMCSequence`` is not built; nor is d > 20 (the calibration's bound)."""

    def __init__(self, model=None, wastefree=True, len_chain=10, move=None):
        super().__init__(model=model, wastefree=wastefree, len_chain=len_chain, move=move)
        if not _device_likelihood(model) and getattr(type(model), "logpyt", None) in (None, StaticModel.logpyt):
            raise NotImplementedError("IBIS: model %r has neither a device likelihood nor a logpyt method"
                                      % type(model).__name__)
        d = model.d if _device_likelihood(model) else model.dim
        if d > 20:
            raise NotImplementedError("IBIS: d = %d parameters; the random-walk calibration is built for d <= 20" % d)

    def logG(self, t, xp, x):
        if _device_likelihood(self.model):        # a one-row commit: lpost and llik in place, lpyt into zeros
            lpyt = torch.zeros(x.N, dtype=torch.float64, device=x.theta.device)
            self.model.logpyt_rows(x.theta, t, 1, lpyt, x.lpost, x.llik)
            return lpyt
        lpyt = as_device(self.model.logpyt(self.model.fields(x.theta), t))
        x.lpost = x.lpost + lpyt
        x.llik = x.llik + lpyt
        return lpyt

    def current_target(self, t):
        model = self.model
        if _device_likelihood(model):
            def func(x):
                model.target(x, 1.0, n_rows=t + 1)
            func.fused_wf = lambda x, P, noise=None: model.wf_move(x, 1.0, P, noise, n_rows=t + 1)
            return func

        def func(x):
            x.lprior = model.logprior(x.theta)
            x.llik = model.loglik(x.theta, t)
            x.lpost = x.lprior + x.llik
        return func

    def _M0(self, N):
        x0 = ThetaParticles(theta=self.model.prior_rvs(N))
        self.current_target(-1)(x0)
        return x0

    def M(self, t, xp):
        if xp.shared["rs_flag"]:
            return self.move(xp, self.current_target(t - 1))      # the target at time t - 1: given y_0..y_{t-1}
        return xp


# ---------------------------------------------------------------------------------------------------------- SMC^2
def _as_struct(arr, names):
    """(n, p) host array -> structured array with one float field per column."""
    out = np.empty(arr.shape[0], dtype=[(k, float) for k in names])
    for i, k in enumerate(names):
        out[k] = arr[:, i]
    return out


class SMC2Particles(ThetaParticles):
    """The particles of ``SMC2``: ``theta_dev`` (n, p) fp64 CUDA tensor of the parameters (columns ``names``, the
    prior's fields), ``lprior``, ``llik`` (each filter's logLt), ``lpost`` (n,) and ``bank``, the n inner filters
    (``bank.FilterBank``) in place of the reference's list ``pfs``.  ``theta`` is the NumPy structured array of the
    reference's particles, materialised from the device on each access (``X.theta['sigma']``).  Indexing by an
    int64 tensor gathers the fields and the bank; the bank copies of a repeated ancestor after the first draw new keys
    from the sampler's key counter ``keys``."""

    _META = ("shared", "names", "bank", "keys")

    def __init__(self, shared=None, names=(), bank=None, keys=None, **fields):
        super().__init__(shared=shared, **fields)
        self.names, self.bank, self.keys = tuple(names), bank, keys

    @property
    def dict_fields(self):
        return {k: v for k, v in self.__dict__.items() if k not in self._META}

    @property
    def theta(self):
        return _as_struct(self.theta_dev.cpu().numpy(), self.names)

    @property
    def Nx(self):
        return self.bank.N

    def _like(self, fields, bank):
        return self.__class__(shared=self.shared.copy(), names=self.names, bank=bank, keys=self.keys, **fields)

    def __getitem__(self, key):
        if not (isinstance(key, torch.Tensor) and key.dtype == torch.int64):
            key = torch.as_tensor(np.arange(self.N)[key], dtype=torch.int64, device=self.theta_dev.device)
        x = ThetaParticles.__getitem__(ThetaParticles(**self.dict_fields), key)
        bank = self.bank.gather(key, self.keys.seed, self.keys.take(key.shape[0]))
        return self._like(x.dict_fields, bank)

    def copy(self):
        """A copy whose filters continue independently of the originals (the reference deep-copies its filters, whose
        futures then draw different numbers from the global stream): the rows are copied, the keys are fresh."""
        b = self.bank.empty_like()
        for name in ("X", "lw", "state", "params") + (("sc",) if b.sc is not None else ()):
            getattr(b, name).copy_(getattr(self.bank, name))
        b.fresh_keys(self.keys.seed, self.keys.take(b.R))
        b.timer = self.bank.timer
        return self._like({k: v.clone() for k, v in self.dict_fields.items()}, b)

    @classmethod
    def concatenate(cls, *xs):
        from .bank import FilterBank
        fields = {k: torch.cat([getattr(x, k) for x in xs]) for k in xs[0].dict_fields}
        return xs[0]._like(fields, FilterBank.concatenate(*[x.bank for x in xs]))


class _KeyCounter:
    """The sampler's seed and the number of inner-filter keys drawn so far: key number c is
    fmix64(fmix64(seed) + c) (smcb_bank_keys), so no two filters of a run ever share a key."""

    def __init__(self, seed):
        self.seed, self.count = int(seed) & (2 ** 64 - 1), 0

    def take(self, n):
        c = self.count
        self.count += int(n)
        return c


class BankRandomWalk(ArrayRandomWalk):
    """Gaussian random-walk Metropolis on ``theta_dev`` whose target re-runs the proposals' filters: the accepted
    proposals' filters replace the current ones (smcb_mh_accept_flags + smcb_bank_merge)."""

    def calibrate(self, W, x):
        n, d = x.theta_dev.shape
        ctx = context()
        L = empty(d * d).reshape(d, d)
        _lib.check(ctx.lib.smcb_rw_calibrate(ctx.handle, ptr(as_device(W)), ptr(x.theta_dev), n, d,
                                             2.38 / np.sqrt(d), ptr(L)))
        x.shared["chol_cov"] = L

    def step(self, x, target):
        ctx = context()
        n, d = x.theta_dev.shape
        xprop = x._like({"theta_dev": torch.empty_like(x.theta_dev)}, None)
        _lib.check(ctx.lib.smcb_rw_propose(ctx.handle, ptr(x.theta_dev), n, d, ptr(x.shared["chol_cov"]), None,
                                           ptr(xprop.theta_dev)))
        target(xprop)
        acc = empty(1)
        flags = torch.empty(n, dtype=torch.uint8, device=x.theta_dev.device)
        _lib.check(ctx.lib.smcb_mh_accept_flags(
            ctx.handle, n, d, ptr(x.theta_dev), ptr(x.lprior), ptr(x.llik), ptr(x.lpost), ptr(xprop.theta_dev),
            ptr(xprop.lprior), ptr(xprop.llik), ptr(xprop.lpost), None, ptr(acc), ptr(flags)))
        x.bank.merge(xprop.bank, flags)
        return acc


class SMC2(FKSMCsampler):
    """SMC^2 (smc_samplers.py:1038-1167): an SMC sampler over theta whose likelihood factors are estimated by one
    particle filter per theta-particle.  Same constructor as the reference; the inner filters are one
    ``bank.FilterBank`` on the device, advanced one step for every theta-particle in ONE launch per SMC^2 step, and
    re-run from step 0 for all proposals of an MCMC step (or all particles of an exchange step) in one launch.

    ``ssm_cls`` must be one of the stock 1-D models (``bank.SUPPORTED``), of this package or the reference;
    ``fk_cls`` one of the stock Feynman-Kac kinds (Bootstrap by default).  ``smc_options`` passes ``resampling``
    and ``ESSrmin`` to the inner filters (``qmc=True`` is not built).  ``prior`` is duck-typed: ``rvs(size)`` returns a
    structured array of scalar fields, ``logpdf(theta)`` their joint log-density, evaluated on the host
    (``distributions.StructDist``, or the reference's own).  ``seed``: the key of the inner filters' streams;
    by default it is drawn from the device generator when the sampler starts, so ``SMC(seed=s)`` fixes it."""

    def __init__(self, ssm_cls=None, prior=None, data=None, smc_options=None, fk_cls=None, init_Nx=100,
                 ar_to_increase_Nx=-1.0, wastefree=True, len_chain=10, move=None, seed=None, tier="auto"):
        if move is None:
            seq = MCMCSequenceWF if wastefree else AdaptiveMCMCSequence
            move = seq(mcmc=BankRandomWalk(), len_chain=len_chain)
        super().__init__(model=None, wastefree=wastefree, len_chain=len_chain, move=move)
        self.smc_options = {"collect": "off"}
        if smc_options is not None:
            self.smc_options.update(smc_options)
        if "model" in self.smc_options or "data" in self.smc_options:
            raise ValueError("SMC2: options model and data are not allowed in smc_options")
        if self.smc_options.get("qmc"):
            raise NotImplementedError("SMC2 over SQMC inner filters (qmc=True) is not built")
        self.resampling = self.smc_options.get("resampling", "systematic")
        if self.resampling not in _lib.FUSED_SCHEMES:
            raise NotImplementedError("SMC2: the inner filters resample with one of %s" % (_lib.FUSED_SCHEMES,))
        self.ESSrmin_inner = float(self.smc_options.get("ESSrmin", 0.5))
        from .state_space_models import _FK_KINDS, Bootstrap
        self.fk_cls = Bootstrap if fk_cls is None else fk_cls
        self.fk_kind = dict(_FK_KINDS).get(getattr(self.fk_cls, "__name__", None))
        self.ssm_cls, self.prior, self.data = ssm_cls, prior, data
        self.init_Nx, self.ar_to_increase_Nx = int(init_Nx), ar_to_increase_Nx
        self.seed, self.tier = seed, tier
        self._map = None
        if data is not None:
            self._setup()

    def _setup(self):
        from .bank import ThetaMap
        from .state_space_models import _flat_data
        flat = _flat_data(self.data, 1).reshape(-1)
        names = list(getattr(self.prior, "laws", {}).keys()) or list(self.prior.rvs(size=1).dtype.names)
        self._map = ThetaMap(self.ssm_cls, names, flat)
        if self.fk_kind is None or (self.fk_kind != _lib.FK_BOOTSTRAP and not self._map.proposal) or (
                self.fk_kind == _lib.FK_GUIDED and self._map.name == "ThetaLogistic"):
            raise NotImplementedError("SMC2: Feynman-Kac class %r is not built for %s on the device"
                                      % (self.fk_cls, self._map.name))
        self._data_dev = self._sc_dev = None      # uploaded with the first bank
        self.timer = None          # None, or a list that receives the CUDA events of every bank launch

    @property
    def T(self):
        return 0 if self.data is None else len(self.data)

    # ------------------------------------------------------------------ theta -> filters
    def _bank(self, theta_dev, Nx, keys):
        from .bank import FilterBank
        m = self._map
        n = theta_dev.shape[0]
        if self._data_dev is None:
            self._data_dev = as_device(m.data)
            self._sc_dev = None if m.shared_sc is None else as_device(m.shared_sc)
        b = FilterBank(m.model, self.fk_kind, self.resampling, Nx, n, self._data_dev, m.n_params, self.ESSrmin_inner,
                       shared_sc=self._sc_dev, per_filter_sc=m.name == "Gordon_etal", tier=self.tier)
        th = theta_dev.cpu().numpy()
        b.set_rows(m.params(th), m.step_consts(th))
        b.fresh_keys(keys.seed, keys.take(n))
        b.timer = self.timer
        return b

    def current_target(self, t, Nx):
        """smc_samplers.py:1129-1143: new filters for every particle, prior, and -- for t >= 0 -- the filters of the
        particles with a finite prior re-run over steps 0..t in one launch; lpost = lprior + logLt."""
        def func(x):
            x.bank = self._bank(x.theta_dev, Nx, x.keys)
            lp = np.asarray(self.prior.logpdf(x.theta), dtype=np.float64)
            lp = np.array(np.broadcast_to(lp, (x.theta_dev.shape[0],)))
            x.lprior = as_device(lp)
            if t >= 0:
                idx = np.flatnonzero(np.isfinite(lp))
                if idx.size:
                    x.bank.advance(t + 1, idx=as_device(idx, dtype=torch.int64), restart=True)
            x.llik = x.bank.logLt.clone()
            x.lpost = x.lprior + x.llik
        return func

    def _M0(self, N):
        if self._map is None:
            self._setup()
        seed = self.seed
        if seed is None:                       # from the device generator: SMC(seed=s) fixes the inner keys
            ctx = context()
            u = empty(2)
            _lib.check(ctx.lib.smcb_uniform(ctx.handle, ptr(u), 2))
            hi, lo = (int(v * 2.0 ** 32) for v in u.cpu().numpy())
            seed = (hi << 32) | lo
        th = self.prior.rvs(size=N)
        names = self._map.names = list(th.dtype.names)
        cols = np.stack([np.asarray(th[k], dtype=np.float64).reshape(N) for k in names], axis=1)
        x0 = SMC2Particles(shared={"Nxs": [self.init_Nx]}, names=names, keys=_KeyCounter(seed),
                           theta_dev=as_device(cols))
        self.current_target(-1, self.init_Nx)(x0)
        return x0

    def logG(self, t, xp, x):
        """smc_samplers.py:1099-1120: exchange step if the last move accepted too little, then every filter advances
        by step t (one launch); the increments loglt are the log-weights."""
        we_increase_Nx = False
        if x.shared.get("rs_flag", False) and x.shared.get("acc_rates"):
            ars = x.shared["acc_rates"][-1]          # the last move's list of mean acceptance rates (device scalars)
            ar = float(torch.cat([a.reshape(1) for a in ars]).mean())
            we_increase_Nx = ar < self.ar_to_increase_Nx
        liw_Nx = None
        if we_increase_Nx:
            liw_Nx = self.exchange_step(x, t, 2 * x.bank.N)
        x.bank.advance(t + 1)
        lpyt = x.bank.loglt.clone()
        x.lpost = x.lpost + lpyt
        x.llik = x.bank.logLt.clone()
        if t > 0:
            x.shared["Nxs"].append(x.bank.N)
        return lpyt + liw_Nx if we_increase_Nx else lpyt

    def M(self, t, xp):
        if xp.shared["rs_flag"]:
            return self.move(xp, self.current_target(t - 1, xp.bank.N))
        return xp

    def exchange_step(self, x, t, new_Nx):
        """smc_samplers.py:1159-1163: every filter re-run over steps 0..t-1 at new_Nx particles."""
        old_lpost = x.lpost.clone()
        self.current_target(t - 1, new_Nx)(x)
        return x.lpost - old_lpost

    def default_moments(self, W, x):
        """Weighted mean and variance of every parameter, as structured arrays (the reference's
        wmean_and_var_str_array)."""
        m = rs.wmean_and_var(W, x.theta_dev)
        mean, var = np.atleast_1d(m["mean"]), np.atleast_1d(m["var"])
        return {"mean": _as_struct(mean[None, :], x.names), "var": _as_struct(var[None, :], x.names)}

    def summary_format(self, smc):
        return super().summary_format(smc) + ", Nx=%i" % smc.X.bank.N


def from_reference_smc2(fk):
    """``SMC2`` for the reference's own ``particles.smc_samplers.SMC2`` object when its ``ssm_cls`` is a stock 1-D
    model (recognised by class name and module, as ``state_space_models.fused_spec`` does), else None: that object
    then keeps its own path.  The sampler takes the reference object's model, prior, data, options, Feynman-Kac
    class, Nx schedule and chain length; the move is this package's (random walk over the filter bank)."""
    cls = type(fk)
    if cls.__name__ != "SMC2" or cls.__module__ != "particles.smc_samplers":
        return None
    move = getattr(fk, "move", None)
    len_chain = getattr(move, "nsteps", getattr(fk, "len_chain", 10) - 1) + 1
    try:
        return SMC2(ssm_cls=fk.ssm_cls, prior=fk.prior, data=fk.data, smc_options=dict(fk.smc_options),
                    fk_cls=fk.fk_cls, init_Nx=fk.init_Nx, ar_to_increase_Nx=fk.ar_to_increase_Nx,
                    wastefree=fk.wastefree, len_chain=len_chain)
    except NotImplementedError:
        return None
