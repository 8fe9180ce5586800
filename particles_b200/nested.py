"""Nested sampling SMC on the device: ``NestedSamplingSMC`` (particles/nested.py:281-373; Salomone, South, Drovandi and
Kroese 2018, arXiv 1805.03924), a Feynman-Kac model for ``particles_b200.SMC`` (plugin path):

    model = smc_samplers.LogisticRegression(data=flipped_predictors, prior_scale=5.)
    fk = NestedSamplingSMC(model=model, len_chain=100, ESSrmin=0.5)
    pf = particles_b200.SMC(fk=fk, N=1000)
    pf.run();  pf.X.shared["log_evid"][-1];  pf.X.shared["lts"]

The target at generation t is the prior truncated to ``llik >= lts[-1]``.  Every generation resamples and moves
with the random-walk Metropolis of the tempering samplers; the next level ``lt`` is the ``100 (1 - ESSrmin)``
percentile of the particles' log-likelihoods.  The whole threshold step (order statistics, evidence update, stopping
rule, new log-weights) is one library call (``smcb_ns_threshold``) followed by one read of three doubles: the
reference keeps ``lts`` and ``log_evid`` as Python floats and stops when ``lts[-1] == inf``.

Two kinds of model run: ``smc_samplers.LogisticRegression``, whose targets and waste-free move are libsmcb kernels
(one launch per waste-free generation), and a ``smc_samplers.StaticModel`` with a user ``logpyt`` on CUDA tensors.
"""
import numpy as np
import torch

from . import _lib
from . import smc_samplers as ssps
from .device import as_device, context, empty, ptr


def percentile_rule(n, ESSrmin):
    """(k0, k1, gamma) such that ``lerp(v[k0], v[k1], gamma)`` over the sorted values ``v`` of an array of length
    ``n`` is ``np.percentile(v, 100 * (1 - ESSrmin))``: NumPy's "linear" method (virtual index (n - 1) q; past the
    last index both statistics are the last one and NumPy's gamma is measured from index -1)."""
    if not 0.0 < ESSrmin <= 1.0:
        raise ValueError("NestedSamplingSMC: ESSrmin must be in (0, 1] (got %r)" % (ESSrmin,))
    q = (100.0 * (1.0 - ESSrmin)) / 100.0
    v = (n - 1) * q
    if v >= n - 1:
        return n - 1, n - 1, v + 1.0
    k0 = int(np.floor(v))
    return k0, k0 + 1, v - float(k0)


def lerp(a, b, gamma):
    """numpy's ``_lerp`` on scalars: a + (b - a) gamma, or b - (b - a)(1 - gamma) where gamma >= 0.5."""
    diff = b - a
    return b - diff * (1.0 - gamma) if gamma >= 0.5 else a + diff * gamma


def threshold(llik, ESSrmin, t, log_evid, eps):
    """NestedSamplingSMC.logG (nested.py:330-351) without its bookkeeping: (lw, lt, new_evid, stop) for the (n,)
    CUDA tensor llik.  One smcb_ns_threshold call and one read of three doubles."""
    llik = as_device(llik)
    n = llik.shape[0]
    k0, k1, gamma = percentile_rule(n, ESSrmin)
    ctx = context(llik.device)
    lw, out = empty(n), empty(3)
    _lib.check(ctx.lib.smcb_ns_threshold(ctx.handle, ptr(llik), n, k0, k1, gamma, int(t), float(np.log(ESSrmin)),
                                         float(log_evid), float(eps), ptr(lw), ptr(out)))
    lt, new_evid, stop = out.cpu().numpy().tolist()
    return lw, lt, new_evid, bool(stop)


class NestedSamplingSMC(ssps.FKSMCsampler):
    """Feynman-Kac model of nested sampling SMC (nested.py:281-373), same constructor and defaults as the reference.
    ``ESSrmin``: the next level ``lt`` leaves a fraction ESSrmin of the particles above it; ``eps``: the run stops
    when the last log-evidence estimate changes by less than eps if lt is taken as +inf.  The successive estimates
    are ``X.shared['log_evid']`` and the levels ``X.shared['lts']``.

    ``model`` is ``smc_samplers.LogisticRegression`` (device likelihood) or a ``smc_samplers.StaticModel`` whose
    ``logpyt`` runs on CUDA tensors.  As for ``IBIS``, a model with neither, or with d > 20 parameters (the bound of
    the random-walk calibration), raises NotImplementedError.  The adaptive stopping rule of ``AdaptiveMCMCSequence`` is
    not built: the standard move has a fixed length."""

    def __init__(self, model=None, wastefree=True, len_chain=10, move=None, ESSrmin=0.1, eps=0.01):
        super().__init__(model=model, wastefree=wastefree, len_chain=len_chain, move=move)
        device = ssps._device_likelihood(model)
        if not device and getattr(type(model), "logpyt", None) in (None, ssps.StaticModel.logpyt):
            raise NotImplementedError("NestedSamplingSMC: model %r has neither a device likelihood nor a logpyt method"
                                      % type(model).__name__)
        d = model.d if device else model.dim
        if d > 20:
            raise NotImplementedError("NestedSamplingSMC: d = %d parameters; the random-walk calibration is built "
                                      "for d <= 20" % d)
        self.ESSrmin = ESSrmin
        self.eps = eps

    def time_to_resample(self, smc):
        self.move.calibrate(smc.W, smc.X)
        return True                       # always resample

    def done(self, smc):
        try:
            lt = smc.X.shared["lts"][-1]
        except (AttributeError, KeyError, IndexError):
            lt = 0.0
        return lt == np.inf

    def summary_format(self, smc):
        return "{}, loglik={:f}".format(super().summary_format(smc), smc.X.shared["lts"][-1])

    def logG(self, t, xp, x):
        lw, lt, new_evid, _ = threshold(x.llik, self.ESSrmin, t, x.shared["log_evid"][-1], self.eps)
        x.shared["lts"].append(lt)
        x.shared["log_evid"].append(new_evid)
        return lw

    def current_target(self, lt):
        model = self.model
        if ssps._device_likelihood(model):
            def func(x):
                model.target(x, 0.0, lmin=lt)
            func.fused_wf = lambda x, P, noise=None: model.wf_move(x, 0.0, P, noise, lmin=lt)
            return func

        def func(x):
            x.lprior = model.logprior(x.theta)
            x.llik = model.loglik(x.theta)
            if lt == -np.inf:
                x.lpost = x.lprior.clone()
            else:
                x.lpost = torch.where(x.llik >= lt, x.lprior, torch.full_like(x.lprior, -np.inf))
        return func

    def _M0(self, N):
        x0 = ssps.ThetaParticles(theta=self.model.prior_rvs(N))
        x0.shared["lts"] = [-np.inf]
        x0.shared["log_evid"] = [-np.inf]
        self.current_target(-np.inf)(x0)
        return x0

    def M(self, t, xp):
        return self.move(xp, self.current_target(xp.shared["lts"][-1]))
