"""SMC samplers on binary spaces {0, 1}^p on the device -- ``particles/binary_smc.py`` (Schäfer & Chopin 2013, with
the waste-free moves of Dau & Chopin 2022), file:line cited per name:

    prior = distributions.IID(Bernoulli(0.5), p)
    model = BayesianVS(data=(X, y), prior=prior)
    move = MCMCSequenceWF(mcmc=BinaryMetropolis(), len_chain=P)
    pf = particles_b200.SMC(fk=AdaptiveTempering(model, len_chain=P, move=move), N=M)

Particles are a ``ThetaParticles`` whose ``theta`` is an (N, p) ``torch.bool`` CUDA tensor.  The batched Cholesky of
every particle's X^T X[gamma, gamma] (``chol_and_friends``), the nested-logistic proposal and the whole waste-free
move (one launch per tempering step) run in libsmcb kernels (csrc/smcb_binary.cu).  ``NestedLogistic.fit`` runs on
the host with scikit-learn, as in the reference, so the proposal has the reference's coefficients; it reads the
particles once per calibration and uploads the coefficients once.  p <= 128 (the kernels' shared-memory bound), and
the prior must be ``IID(Bernoulli(q), p)``, whose log-density the kernels compute in closed form.
"""
import ctypes as C

import numpy as np
import torch
from scipy.special import logit

from . import _lib
from .device import as_device, context, empty, ptr
from .distributions import IID, ProbDist

MAX_P = 128


def _check_p(p):
    if p > MAX_P:
        raise NotImplementedError("binary_smc: p = %d predictors; the device kernels are built for p <= %d "
                                  "(one packed Cholesky triangle per warp in shared memory)" % (p, MAX_P))


def all_binary_words(p):
    """binary_smc.py:54-59."""
    out = np.zeros((2 ** p, p), dtype=bool)
    ns = np.arange(2 ** p)
    for i in range(p):
        out[:, i] = (ns % 2 ** (i + 1)) // 2 ** i
    return out


def log_no_warn(x):
    """binary_smc.py:62-64."""
    return np.log(np.clip(x, 1e-300, None))


def _bool_device(x):
    if isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.bool:
        return x.contiguous()
    if isinstance(x, torch.Tensor):
        return x.to(device="cuda", dtype=torch.bool).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=bool))).cuda()


class Bernoulli(ProbDist):
    """binary_smc.py:67-80, with a scalar probability p.  ``rvs`` returns a (size,) bool CUDA tensor."""
    dtype = bool

    def __init__(self, p):
        self.p = p

    def _iid(self, k):
        """IID(Bernoulli(p), k) is the nested logistic law whose coordinates are all edgy with probability p."""
        return NestedLogistic(np.diag(np.full(k, float(self.p))), np.ones(k, dtype=bool))

    def rvs(self, size=None):
        return self._iid(1).rvs(size=1 if size is None else size)[:, 0]

    def logpdf(self, x):
        return self._iid(1).logpdf(_bool_device(x).reshape(-1, 1))


def _bernoulli_q(prior, p):
    """q of a prior IID(Bernoulli(q), p); NotImplementedError for any other prior."""
    if not (isinstance(prior, IID) and isinstance(prior.law, Bernoulli) and prior.dim == p
            and np.ndim(prior.law.p) == 0):
        raise NotImplementedError("binary_smc: the prior must be distributions.IID(Bernoulli(q), p) with p = %d "
                                  "and a scalar q (the kernels compute its log-density in closed form); got %r"
                                  % (p, prior))
    return float(prior.law.p)


class NestedLogistic(ProbDist):
    """binary_smc.py:83-143: coordinate i is Bernoulli(coeffs[i, i]) if edgy[i], else a logistic regression on the
    coordinates before it.  ``coeffs`` / ``edgy`` are host arrays; they go to the device once."""
    dtype = "bool"

    def __init__(self, coeffs, edgy):
        self.coeffs = np.ascontiguousarray(np.asarray(coeffs, dtype=np.float64))
        self.edgy = np.asarray(edgy, dtype=bool)
        self.dim = len(self.edgy)
        _check_p(self.dim)
        self._dev = None

    def _device(self):
        """(coeffs, edgy) on the device, uploaded on first use."""
        if self._dev is None:
            self._dev = (as_device(self.coeffs), torch.from_numpy(self.edgy.astype(np.uint8)).cuda())
        return self._dev

    def predict_prob(self, x, i):
        """binary_smc.py:98-106 for the (N, p) bool CUDA tensor x: a scalar if edgy[i], else an (N,) tensor."""
        if self.edgy[i]:
            return self.coeffs[i, i]
        x = _bool_device(x)
        lin = 0.0
        if i > 0:
            lin = torch.sum(self._device()[0][i, :i] * x[:, :i], dim=1)
        return torch.special.expit(self.coeffs[i, i] + lin)

    def _call(self, n, x, draw, u=None):
        ctx = context()
        lp = empty(n)
        coeffs, edgy = self._device()
        _lib.check(ctx.lib.smcb_nested_logistic(ctx.handle, self.dim, ptr(coeffs), ptr(edgy), n,
                                                int(draw), ptr(x), ptr(None if u is None else as_device(u)), ptr(lp)))
        return lp

    def rvs(self, size=1, u=None):
        """binary_smc.py:108-112; ``u``: injected (p, size) uniforms, in the reference's order of draws."""
        x = torch.empty((size, self.dim), dtype=torch.bool, device="cuda")
        self._call(size, x, True, u)
        return x

    def rvs_and_logpdf(self, size=1, u=None):
        x = torch.empty((size, self.dim), dtype=torch.bool, device="cuda")
        return x, self._call(size, x, True, u)

    def logpdf(self, x):
        """binary_smc.py:114-118."""
        x = _bool_device(x)
        return self._call(x.shape[0], x, False)

    @classmethod
    def fit(cls, W, x, probs_thresh=0.02, corr_thresh=0.075):
        """binary_smc.py:120-143, on the host with scikit-learn as in the reference: W and x are read once."""
        from sklearn.linear_model import LogisticRegression as SkLogisticRegression
        W = W.detach().cpu().numpy() if isinstance(W, torch.Tensor) else np.asarray(W)
        x = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=bool)
        N, dim = x.shape
        coeffs = np.zeros((dim, dim))
        ph = np.average(x, weights=W, axis=0)
        edgy = (ph < probs_thresh) | (ph > 1.0 - probs_thresh)
        for i in range(dim):
            if edgy[i]:
                coeffs[i, i] = ph[i]
            else:
                preds = []
                for j in range(i):
                    pij = np.average(x[:, i] & x[:, j], weights=W, axis=0)
                    corr = corr_bin(ph[i], ph[j], pij)
                    if np.abs(corr) > corr_thresh:
                        preds.append(j)
                if preds:
                    reg = SkLogisticRegression(penalty=None)
                    reg.fit(x[:, preds], x[:, i], sample_weight=W)
                    coeffs[i, i] = reg.intercept_[0]
                    coeffs[i, preds] = reg.coef_
                else:
                    coeffs[i, i] = logit(ph[i])
        return cls(coeffs, edgy)


def corr_bin(pi, pj, pij):
    """binary_smc.py:146-151."""
    varij = pi * (1.0 - pi) * pj * (1.0 - pj)
    if varij <= 0:
        return 0.0
    return (pij - pi * pj) / np.sqrt(varij)


class BinaryMetropolis:
    """binary_smc.py:154-162: independent Metropolis with a NestedLogistic proposal fitted to the weighted sample.
    Plugs into ``MCMCSequenceWF`` (fused: one launch per move when the target offers it) and
    ``AdaptiveMCMCSequence`` (one proposal, target and accept launch per step)."""

    def calibrate(self, W, x):
        x.shared["proposal"] = NestedLogistic.fit(W, x.theta)

    def proposal(self, x, xprop, u=None):
        prop_dist = x.shared["proposal"]
        xprop.theta, lq_prop = prop_dist.rvs_and_logpdf(size=x.N, u=u)
        return prop_dist.logpdf(x.theta) - lq_prop

    def step(self, x, target, noise=None):
        """ArrayMetropolis.step (smc_samplers.py:601-611); returns the mean acceptance probability (device scalar).
        ``noise``: injected (proposal uniforms (p, N), acceptance uniforms (N,)).  smcb_mh_accept_flags takes the
        decision on lpost' + delta_lp against lpost (the reference sums lpost' - lpost + delta_lp: the same up to
        rounding) and copies the fp64 scores of accepted proposals; the bool rows follow its flags."""
        ctx = context()
        xprop = x.__class__()
        delta_lp = self.proposal(x, xprop, None if noise is None else noise[0])
        target(xprop)
        lpost_p = xprop.lpost
        shifted = lpost_p + delta_lp
        u = None if noise is None else as_device(noise[1])
        acc = empty(1)
        flags = torch.empty(x.N, dtype=torch.uint8, device=x.theta.device)
        _lib.check(ctx.lib.smcb_mh_accept_flags(ctx.handle, x.N, 1, ptr(x.llik), ptr(x.lprior), ptr(x.llik),
                                                ptr(x.lpost), ptr(xprop.llik), ptr(xprop.lprior), ptr(xprop.llik),
                                                ptr(shifted), ptr(u), ptr(acc), ptr(flags)))
        keep = flags.bool()
        x.theta = torch.where(keep[:, None], xprop.theta, x.theta)
        x.lpost = torch.where(keep, lpost_p, x.lpost)
        return acc


class VariableSelection:
    """binary_smc.py:183-213: a (pseudo-)posterior over the indicators gamma of the predictors to include.
    ``data`` = (X (n, p), y (n,)); X^T X, y^T y and X^T y are formed on the host as in the reference and uploaded
    once.  ``target`` / ``wf_move`` give ``Tempering`` and ``AdaptiveTempering`` the device target and the fused
    waste-free move, as ``smc_samplers.LogisticRegression`` does."""

    use_ldet = 0

    def __init__(self, data=None):
        self.x, self.y = data
        self.n, self.p = self.x.shape
        _check_p(self.p)
        self.xtx = self.x.T @ self.x
        self.yty = np.sum(self.y ** 2)
        self.xty = self.x.T @ self.y
        self._xtx_dev = as_device(self.xtx)
        self._xty_dev = as_device(self.xty)

    @property
    def T(self):
        return 0

    @property
    def d(self):
        return self.p

    def _gw(self):
        return 1.0

    def _desc(self):
        q = _bernoulli_q(self.prior, self.p) if getattr(self, "prior", None) is not None else 0.5
        return _vs_desc(self._xtx_dev, self._xty_dev, self.use_ldet, self.iv2, self.coef_len, self.coef_log,
                        self.coef_in_log, self._gw(), q)

    def complete_enum(self):
        """binary_smc.py:202-205, for p <= 20: all 2^p gammas and their log-posterior (CUDA tensor)."""
        if self.p > 20:
            raise NotImplementedError("complete_enum: p = %d; enumeration is built for p <= 20" % self.p)
        gammas = all_binary_words(self.p)
        return gammas, self.logpost(gammas)

    def chol_intermediate(self, gamma):
        out = _vs_call(self._desc(), gamma, self.iv2, ("len_gam", "ldet", "wtw"))
        return out["len_gam"], out["ldet"], out["wtw"]

    def sig2_full(self):
        """binary_smc.py:210-213 (the full model's factorisation on the device)."""
        gamma_full = np.ones((1, self.p), dtype=bool)
        btb = _vs_call(_vs_desc(self._xtx_dev, self._xty_dev), gamma_full, 0.0, ("wtw",))["wtw"]
        return (self.yty - float(btb[0])) / self.n

    def loglik(self, gamma, t=None):
        return _vs_call(self._desc(), gamma, self.iv2, ("llik",))["llik"]

    def logprior(self, gamma):
        _bernoulli_q(self.prior, self.p)
        return self.prior.logpdf(gamma)

    def logpost(self, gamma, t=None):
        return _vs_call(self._desc(), gamma, self.iv2, ("lprior", "llik", "lpost"), epn=1.0)["lpost"]

    # -------------------------------------------------------------- sampler interface (as LogisticRegression's)
    def prior_rvs(self, size):
        _bernoulli_q(self.prior, self.p)
        return self.prior.rvs(size=size)

    def target(self, x, epn):
        """Tempering.current_target (smc_samplers.py:836-845): lprior, llik and lpost = lprior + epn llik."""
        _bernoulli_q(self.prior, self.p)
        out = _vs_call(self._desc(), x.theta, self.iv2, ("lprior", "llik", "lpost"), epn=epn)
        x.lprior, x.llik, x.lpost = out["lprior"], out["llik"], out["lpost"]

    def wf_move(self, x, epn, P, noise=None):
        """The fused waste-free move (smcb_binary_wf_move): x = the M resampled particles with their scores at
        exponent ``epn`` and ``shared['proposal']``; returns P*M particles.  ``noise`` = (proposal uniforms
        (P-1, p, M), acceptance uniforms (P-1, M)) in the reference's order of draws, or None."""
        _bernoulli_q(self.prior, self.p)
        ctx = context()
        M = x.theta.shape[0]
        coeffs, edgy = x.shared["proposal"]._device()
        out = x.__class__(shared=x.shared.copy(), theta=torch.empty((P * M, self.p), dtype=torch.bool, device="cuda"),
                          lprior=empty(P * M), llik=empty(P * M), lpost=empty(P * M))
        pb = empty((P - 1, M))
        up = ua = None
        if noise is not None:
            up, ua = as_device(noise[0]), as_device(noise[1])
        desc = self._desc()
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        _lib.check(ctx.lib.smcb_binary_wf_move(
            ctx.handle, C.byref(desc), ptr(coeffs), ptr(edgy), M, P, float(epn),
            ptr(_bool_device(x.theta)), ptr(x.lprior), ptr(x.llik), ptr(x.lpost), ptr(up), ptr(ua), ptr(out.theta),
            ptr(out.lprior), ptr(out.llik), ptr(out.lpost), ptr(pb), ptr(err)))
        _raise_on(err)
        out.shared["acc_rates"] = x.shared.get("acc_rates", []) + [pb.mean(dim=1)]
        return out


def _raise_on(err):
    e = int(err.item())
    if e & 1:
        raise np.linalg.LinAlgError("binary_smc: X^T X[gamma, gamma] + iv2 I is not positive definite for some "
                                    "gamma (scipy.linalg.cholesky raises here too)")
    if e & 2:
        raise ValueError("smcb_vs_loglik: a row has more selected predictors than kmax")


def _vs_desc(xtx_dev, xty_dev, use_ldet=0, vm2=0.0, coef_len=0.0, coef_log=0.0, coef_in_log=1.0, gw=1.0, q=0.5):
    return _lib.VsDesc(xtx_dev.shape[0], int(use_ldet), xtx_dev.data_ptr(), xty_dev.data_ptr(), float(vm2),
                       float(coef_len), float(coef_log), float(coef_in_log), float(gw), float(log_no_warn(q)),
                       float(log_no_warn(1.0 - q)))


def _vs_call(desc, gamma, vm2, outputs, epn=0.0):
    """smcb_vs_loglik for the (N, p) gamma: {name: (N,) CUDA tensor} for the requested outputs (len_gam, ldet, wtw,
    lprior, llik, lpost).  The launch is sized from the batch's largest |gamma| (one read)."""
    gamma = _bool_device(gamma)
    n = gamma.shape[0]
    kmax = int(gamma.sum(dim=1).max().item())
    err = torch.zeros(1, dtype=torch.int32, device=gamma.device)
    out = {k: empty(n) for k in outputs}
    ctx = context()
    _lib.check(ctx.lib.smcb_vs_loglik(ctx.handle, C.byref(desc), ptr(gamma), n, kmax, float(vm2), float(epn),
                                      *[ptr(out.get(k)) for k in ("len_gam", "ldet", "wtw", "lprior", "llik",
                                                                  "lpost")], ptr(err)))
    _raise_on(err)
    return out


def chol_and_friends(gamma, xtx, xty, vm2):
    """binary_smc.py:165-180 on the device: (len_gam, ldet, wtw) as CUDA tensors for the (N, p) gamma.  A matrix
    that is not positive definite raises numpy.linalg.LinAlgError (scipy.linalg.LinAlgError), as in the reference."""
    xtx, xty = as_device(xtx), as_device(xty)
    _check_p(xtx.shape[0])
    out = _vs_call(_vs_desc(xtx, xty), gamma, vm2, ("len_gam", "ldet", "wtw"))
    return out["len_gam"], out["ldet"], out["wtw"]


class BIC(VariableSelection):
    """binary_smc.py:216-230: likelihood exp(-lambda BIC(gamma)).  As in the reference, the constructor takes no
    prior: set ``model.prior = IID(Bernoulli(q), p)`` before sampling."""

    def __init__(self, data=None, lamb=10.0):
        super().__init__(data=data)
        self.lamb = lamb
        self.coef_len = np.log(self.n) * self.lamb
        self.coef_log = self.n * self.lamb
        self.coef_in_log = self.yty
        self.iv2 = 0.0


class BayesianVS(VariableSelection):
    """binary_smc.py:233-265: marginal likelihood of Y = X beta + noise, sigma^2 ~ IG(nu / 2, lambda nu / 2),
    beta | sigma^2 ~ N(0, v2 sigma^2 I); iv2 = 1 / v2."""

    use_ldet = 1

    def __init__(self, data=None, prior=None, nu=4.0, lamb=None, iv2=None):
        super().__init__(data=data)
        self.prior = prior
        if prior is not None:
            _bernoulli_q(prior, self.p)
        self.nu = nu
        self.lamb = self.sig2_full() if lamb is None else lamb
        self.iv2 = float(self.lamb / 10.0) if iv2 is None else iv2
        self.set_constants()

    def set_constants(self):
        self.coef_len = -0.5 * np.log(self.iv2)
        self.coef_log = 0.5 * (self.nu + self.n)
        self.coef_in_log = self.nu * self.lamb + self.yty


class BayesianVS_gprior(BayesianVS):
    """binary_smc.py:268-293: beta | sigma^2 ~ N(0, g sigma^2 (X^T X)^-1)."""

    use_ldet = 0

    def __init__(self, data=None, prior=None, nu=4.0, lamb=None, g=None):
        self.g = g
        super().__init__(data=data, prior=prior, nu=nu, lamb=lamb, iv2=0.0)

    def set_constants(self):
        if self.g is None:
            self.g = self.n
        self.coef_len = 0.5 * np.log(1 + self.g)
        self.coef_log = 0.5 * (self.n + self.nu)
        self.coef_in_log = self.nu * self.lamb + self.yty
        self.gogp1 = self.g / (self.g + 1.0)

    def _gw(self):
        return self.gogp1
