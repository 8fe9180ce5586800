"""State-space models and their Feynman-Kac adaptors: the user-facing surface the
north-star keeps (``particles/state_space_models.py``), re-stated over device arrays.

* ``StateSpaceModel`` subclasses define ``PX0 / PX / PY`` (optionally ``proposal0 /
  proposal / logeta``) returning ``particles_b200.distributions`` objects; their
  closures receive CUDA tensors, so user models keep the reference's style.
* ``Bootstrap / GuidedPF / AuxiliaryPF / AuxiliaryBootstrap`` expose ``M0 / M / logG /
  logeta`` to ``core.SMC`` exactly as state_space_models.py:299-438 does.
* Stock models additionally carry ``fused_spec()``: the constants of the fused
  sm_90a step kernel (csrc/smcb_models.cuh), so ``SMC`` never calls their Python
  closures on the hot path.  The same recogniser accepts the reference's own model
  objects (``particles.state_space_models.StochVol`` ...) by class name + module.
"""
import numpy as np
import torch

from . import _lib
from . import distributions as dists
from .core import FeynmanKac


err_msg_missing_cst = """
    State-space model %s is missing method upper_bound_log_pt, which provides
    log of constant C_t, such that
    p(x_t|x_{t-1}) <= C_t
    This is required for smoothing algorithms based on rejection
    """


class StateSpaceModel:
    """particles/state_space_models.py:172-296."""

    def __init__(self, **kwargs):
        if hasattr(self, "default_params"):
            self.__dict__.update(self.default_params)
        self.__dict__.update(kwargs)

    def _error_msg(self, method):
        return "method " + method + " not implemented in class%s" % self.__class__.__name__

    def PX0(self):
        raise NotImplementedError(self._error_msg("PX0"))

    def PX(self, t, xp):
        raise NotImplementedError(self._error_msg("PX"))

    def PY(self, t, xp, x):
        raise NotImplementedError(self._error_msg("PY"))

    def proposal0(self, data):
        raise NotImplementedError(self._error_msg("proposal0"))

    def proposal(self, t, xp, data):
        raise NotImplementedError(self._error_msg("proposal"))

    def upper_bound_log_pt(self, t):
        """state_space_models.py:261-266: log of a constant C_t >= p(x_t | x_{t-1}) (rejection smoothing)."""
        raise NotImplementedError(err_msg_missing_cst % self.__class__.__name__)

    def add_func(self, t, xp, x):
        """state_space_models.py:268-270: the additive function psi_t(x_{t-1}, x_t) of on-line smoothing."""
        raise NotImplementedError(self._error_msg("add_func"))

    def simulate_given_x(self, x):
        lag_x = [None] + x[:-1]
        return [self.PY(t, xp, xx).rvs(size=1) for t, (xp, xx) in enumerate(zip(lag_x, x))]

    def simulate(self, T):
        """state_space_models.py:272-296; returns two lists of length T of (1,) tensors."""
        x = []
        for t in range(T):
            law_x = self.PX0() if t == 0 else self.PX(t, x[-1])
            x.append(law_x.rvs(size=1))
        return x, self.simulate_given_x(x)


class Bootstrap(FeynmanKac):
    """state_space_models.py:299-349."""

    def __init__(self, ssm=None, data=None):
        self.ssm = ssm
        self.data = data

    @property
    def T(self):
        return 0 if self.data is None else len(self.data)

    def M0(self, N):
        return self.ssm.PX0().rvs(size=N)

    def M(self, t, xp):
        return self.ssm.PX(t, xp).rvs(size=xp.shape[0])

    @property
    def du(self):
        """Dimension of the uniforms of SQMC (state_space_models.py:320)."""
        return self.ssm.PX0().dim

    def Gamma0(self, u):
        return self.ssm.PX0().ppf(u)

    def Gamma(self, t, xp, u):
        return self.ssm.PX(t, xp).ppf(u)

    def logG(self, t, xp, x):
        return self.ssm.PY(t, xp, x).logpdf(self.data[t])

    def logpt(self, t, xp, x):
        return self.ssm.PX(t, xp).logpdf(x)

    def upper_bound_trans(self, t):
        """state_space_models.py:345-346."""
        return self.ssm.upper_bound_log_pt(t)

    def add_func(self, t, xp, x):
        """state_space_models.py:348-349."""
        return self.ssm.add_func(t, xp, x)


class GuidedPF(Bootstrap):
    """state_space_models.py:352-398."""

    def M0(self, N):
        return self.ssm.proposal0(self.data).rvs(size=N)

    def M(self, t, xp):
        return self.ssm.proposal(t, xp, self.data).rvs(size=xp.shape[0])

    def Gamma0(self, u):
        return self.ssm.proposal0(self.data).ppf(u)

    def Gamma(self, t, xp, u):
        return self.ssm.proposal(t, xp, self.data).ppf(u)

    def logG(self, t, xp, x):
        if t == 0:
            return (self.ssm.PX0().logpdf(x) + self.ssm.PY(0, xp, x).logpdf(self.data[0])
                    - self.ssm.proposal0(self.data).logpdf(x))
        return (self.ssm.PX(t, xp).logpdf(x) + self.ssm.PY(t, xp, x).logpdf(self.data[t])
                - self.ssm.proposal(t, xp, self.data).logpdf(x))


class APFMixin:
    """state_space_models.py:401-403."""

    def logeta(self, t, x):
        return self.ssm.logeta(t, x, self.data)


class AuxiliaryPF(GuidedPF, APFMixin):
    """state_space_models.py:406-428."""


class AuxiliaryBootstrap(Bootstrap, APFMixin):
    """state_space_models.py:431-438."""


# ---------------------------------------------------------------------------
# stock models
# ---------------------------------------------------------------------------
def _scalar(y):
    return float(np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y).reshape(-1)[0])


class StochVol(StateSpaceModel):
    """state_space_models.py:446-498."""
    default_params = {"mu": -1.02, "rho": 0.9702, "sigma": 0.178}

    def sig0(self):
        return self.sigma / np.sqrt(1.0 - self.rho ** 2)

    def PX0(self):
        return dists.Normal(loc=self.mu, scale=self.sig0())

    def EXt(self, xp):
        return (1.0 - self.rho) * self.mu + self.rho * xp

    def PX(self, t, xp):
        return dists.Normal(loc=self.EXt(xp), scale=self.sigma)

    def PY(self, t, xp, x):
        return dists.Normal(loc=0.0, scale=torch.exp(0.5 * x))

    def _xhat(self, xst, sig, yt):
        e = torch.exp(-xst) if isinstance(xst, torch.Tensor) else np.exp(-xst)
        return xst + 0.5 * sig ** 2 * (yt ** 2 * e - 1.0)

    def proposal0(self, data):
        return dists.Normal(loc=self._xhat(0.0, self.sig0(), _scalar(data[0])), scale=self.sig0())

    def proposal(self, t, xp, data):
        return dists.Normal(loc=self._xhat(self.EXt(xp), self.sigma, _scalar(data[t])),
                            scale=self.sigma)

    def logeta(self, t, x, data):
        y = _scalar(data[t + 1])
        xst = self.EXt(x)
        xstmmu = xst - self.mu
        xhat = self._xhat(xst, self.sigma, y)
        xhatmmu = xhat - self.mu
        return (0.5 / self.sigma ** 2 * (xhatmmu ** 2 - xstmmu ** 2)
                - 0.5 * y ** 2 * torch.exp(-xst) * (1.0 + xstmmu))


class StochVolLeverage(StochVol):
    """state_space_models.py:501-543."""
    default_params = {"mu": -1.02, "rho": 0.9702, "sigma": 0.178, "phi": 0.0}

    def PY(self, t, xp, x):
        if t == 0:
            u = (x - self.mu) / self.sig0()
        else:
            u = (x - self.EXt(xp)) / self.sigma
        std_x = torch.exp(0.5 * x)
        return dists.Normal(loc=std_x * self.phi * u, scale=std_x * np.sqrt(1.0 - self.phi ** 2))


class DiscreteCox(StateSpaceModel):
    """state_space_models.py:611-630."""
    default_params = {"mu": 0.0, "sigma": 1.0, "phi": 0.95}

    def PX0(self):
        return dists.Normal(loc=self.mu, scale=self.sigma / np.sqrt(1.0 - self.phi ** 2))

    def PX(self, t, xp):
        return dists.Normal(loc=self.mu + self.phi * (xp - self.mu), scale=self.sigma)

    def PY(self, t, xp, x):
        return dists.Poisson(rate=torch.exp(x))


class Gordon_etal(StateSpaceModel):
    """state_space_models.py:546-577."""
    default_params = {"a": 0.05, "b": 0.5, "c": 25.0, "d": 8.0, "e": 1.2, "sigmaX": 3.162278}

    def PX0(self):
        return dists.Normal(scale=2.0)

    def PX(self, t, xp):
        return dists.Normal(loc=self.b * xp + self.c * xp / (1.0 + xp ** 2)
                            + self.d * np.cos(self.e * (t - 1)), scale=self.sigmaX)

    def PY(self, t, xp, x):
        return dists.Normal(loc=self.a * x ** 2)


class ThetaLogistic(StateSpaceModel):
    """state_space_models.py:657-689 (PX0 / PX / PY)."""
    default_params = {"tau0": 0.15, "tau1": 0.12, "tau2": 0.1, "sigmaX": 0.47, "sigmaY": 0.39}

    def PX0(self):
        return dists.Normal(loc=0.0, scale=1.0)

    def PX(self, t, xp):
        return dists.Normal(loc=xp + self.tau0 - self.tau1 * torch.exp(self.tau2 * xp),
                            scale=self.sigmaX)

    def PY(self, t, xp, x):
        return dists.Normal(loc=x, scale=self.sigmaY)


class BearingsOnly(StateSpaceModel):
    """state_space_models.py:580-608."""
    default_params = {"sigmaX": 2.0e-4, "sigmaY": 1e-3, "x0": np.array([3e-3, -3e-3, 1.0, 1.0])}

    def PX0(self):
        return dists.IndepProd(dists.Normal(loc=self.x0[0], scale=self.sigmaX),
                               dists.Normal(loc=self.x0[1], scale=self.sigmaX),
                               dists.Dirac(loc=self.x0[2]), dists.Dirac(loc=self.x0[3]))

    def PX(self, t, xp):
        return dists.IndepProd(dists.Normal(loc=xp[:, 0].contiguous(), scale=self.sigmaX),
                               dists.Normal(loc=xp[:, 1].contiguous(), scale=self.sigmaX),
                               dists.Dirac(loc=xp[:, 0] + xp[:, 2]),
                               dists.Dirac(loc=xp[:, 1] + xp[:, 3]))

    def PY(self, t, xp, x):
        angle = torch.arctan(x[:, 3] / x[:, 2])
        angle = torch.where(x[:, 2] < 0.0, angle + np.pi, angle)
        return dists.Normal(loc=angle, scale=self.sigmaY)


class MVStochVol(StateSpaceModel):
    """state_space_models.py:633-654: X_0 ~ N(mu, covX), X_t - mu = F (X_{t-1} - mu) + U_t, Y_t(k) = exp(X_t(k) / 2)
    V_t(k), V_t ~ N(0, corY).  The reference ships it without default parameters (``None``): pass mu (d,), covX,
    corY, F (d, d).  Plugin path (MvNormal kernels with per-particle scale), d <= 32."""
    default_params = {"mu": 0.0, "covX": None, "corY": None, "F": None}

    def _dev(self, name):
        key = "_dev_" + name
        if key not in self.__dict__:
            self.__dict__[key] = dists.as_device(np.asarray(getattr(self, name), dtype=np.float64))
        return self.__dict__[key]

    def offset(self):
        return np.asarray(self.mu, dtype=np.float64) - np.dot(self.F, np.asarray(self.mu, dtype=np.float64))

    def PX0(self):
        return dists.MvNormal(loc=np.asarray(self.mu, dtype=np.float64), cov=self.covX)

    def PX(self, t, xp):
        if "_dev_off" not in self.__dict__:
            self.__dict__["_dev_off"] = dists.as_device(np.broadcast_to(self.offset(), (np.asarray(self.F).shape[0],)).copy())
        return dists.MvNormal(loc=xp @ self._dev("F").t() + self.__dict__["_dev_off"], cov=self.covX)

    def PY(self, t, xp, x):
        return dists.MvNormal(scale=torch.exp(0.5 * x), cov=self.corY)


# ---------------------------------------------------------------------------
# recogniser: Feynman-Kac object -> constants of the fused kernel
# ---------------------------------------------------------------------------
_FK_KINDS = [("AuxiliaryPF", _lib.FK_APF), ("AuxiliaryBootstrap", _lib.FK_AUXBOOT),
             ("GuidedPF", _lib.FK_GUIDED), ("Bootstrap", _lib.FK_BOOTSTRAP)]
_TRUSTED_MODULES = ("particles.state_space_models", "particles.kalman",
                    "particles_b200.state_space_models", "particles_b200.kalman")


def _flat_data(data, dy=1):
    rows = [np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y, dtype=np.float64).reshape(-1)
            for y in data]
    arr = np.array(rows, dtype=np.float64)
    if arr.ndim != 2 or arr.shape[1] != dy:
        raise ValueError(f"data must be a sequence of T observations of dimension {dy}")
    return np.ascontiguousarray(arr)


def spec_stochvol(m, T):
    sig0 = m.sigma / np.sqrt(1.0 - m.rho ** 2)
    p = [m.mu, m.rho, m.sigma, sig0, (1.0 - m.rho) * m.mu, np.log(m.sigma), np.log(sig0)]
    return {"model": _lib.MODEL_STOCHVOL, "params": p, "dim": 1, "proposal": True}


def spec_lingauss(m, T):
    sX, sY, s0, rho = float(m.sigmaX), float(m.sigmaY), float(m.sigma0), float(m.rho)
    s2p0 = 1.0 / (1.0 / s0 ** 2 + 1.0 / sY ** 2)
    s2p = 1.0 / (1.0 / sX ** 2 + 1.0 / sY ** 2)
    se = np.sqrt(sX ** 2 + sY ** 2)
    p = [rho, sX, sY, s0, np.log(sX), np.log(sY), np.log(s0),
         s2p0, np.sqrt(s2p0), np.log(np.sqrt(s2p0)), s2p, np.sqrt(s2p), np.log(np.sqrt(s2p)),
         se, np.log(se), sX ** 2, sY ** 2]
    return {"model": _lib.MODEL_LINGAUSS, "params": p, "dim": 1, "proposal": True}


def spec_gordon(m, T):
    p = [m.a, m.b, m.c, m.sigmaX, np.log(m.sigmaX)]
    sc = np.array([m.d * np.cos(m.e * (t - 1)) for t in range(T)], dtype=np.float64)
    return {"model": _lib.MODEL_GORDON, "params": p, "dim": 1, "proposal": False, "step_consts": sc}


def spec_thetalogistic(m, T):
    p = [m.tau0, m.tau1, m.tau2, m.sigmaX, m.sigmaY, np.log(m.sigmaX), np.log(m.sigmaY)]
    return {"model": _lib.MODEL_THETALOGISTIC, "params": p, "dim": 1, "proposal": False}


def spec_stochvollev(m, T):
    sp = spec_stochvol(m, T)
    sq = np.sqrt(1.0 - m.phi ** 2)
    sp.update(model=_lib.MODEL_STOCHVOLLEV, params=sp["params"] + [m.phi, sq, np.log(sq)], proposal=False)
    return sp


def spec_discretecox(m, T, data=None):
    from scipy.special import gammaln
    sig0 = m.sigma / np.sqrt(1.0 - m.phi ** 2)
    p = [m.mu, m.sigma, m.phi, sig0, np.log(m.sigma), np.log(sig0)]
    y = _flat_data(data, 1).reshape(-1)
    return {"model": _lib.MODEL_DISCRETECOX, "params": p, "dim": 1, "proposal": False,
            "step_consts": gammaln(y + 1.0)}


def spec_bearings(m, T):
    x0 = np.asarray(m.x0, dtype=np.float64).reshape(4)
    p = [m.sigmaX, m.sigmaY, np.log(m.sigmaY)] + list(x0) + [np.log(m.sigmaX)]
    return {"model": _lib.MODEL_BEARINGS, "params": p, "dim": 4, "dy": 1, "n_noise": 2, "proposal": False}


def _pad(M, rows, cols):
    out = np.zeros((rows, cols))
    M = np.atleast_2d(np.asarray(M, dtype=np.float64))
    out[: M.shape[0], : M.shape[1]] = M
    return out


def spec_mvlingauss(m, T, data=None):
    """kalman.py:296-361: all matrices of the fused kernel (csrc/smcb_models.cuh, MvLinGaussM) are
    computed here with NumPy exactly as the reference's closures compute them per step."""
    dx, dy = int(m.dx), int(m.dy)
    if not (2 <= dx <= 4 and 1 <= dy <= 4):
        return None
    F, G = np.asarray(m.F, float), np.asarray(m.G, float)
    covX, covY, cov0, mu0 = (np.asarray(v, float) for v in (m.covX, m.covY, m.cov0, m.mu0))

    def chol(c):
        L = np.linalg.cholesky(c)
        return L, float(np.sum(np.log(np.diag(L))))

    def update(pred_cov):                      # filter_step, kalman.py:196-229
        dpc = G @ pred_cov @ G.T + covY
        gain = np.linalg.solve(dpc, (pred_cov @ G.T).T).T
        return dpc, gain, pred_cov - gain @ G @ pred_cov

    dpc, K, fcov = update(covX)
    dpc0, K0, fcov0 = update(cov0)
    LX, hX = chol(covX); LY, hY = chol(covY); LP, hP = chol(fcov); LE, hE = chol(dpc)
    L0, h0 = chol(cov0); LP0, hP0 = chol(fcov0)
    y0 = np.zeros(dy) if data is None else np.asarray(data[0], float).reshape(-1)
    loc0p = mu0 + (y0 - mu0 @ G.T) @ K0.T       # proposal0 (kalman.py:351-354)
    p = [float(dy)]
    p += list(F.reshape(-1)) + list(_pad(G, 4, dx).reshape(-1)) + list(LX.reshape(-1)) + [hX]
    p += list(_pad(LY, 4, 4).reshape(-1)) + [hY] + list(_pad(K, dx, 4).reshape(-1))
    p += list(LP.reshape(-1)) + [hP] + list(_pad(LE, 4, 4).reshape(-1)) + [hE]
    p += list(mu0.reshape(-1)) + list(L0.reshape(-1)) + [h0] + list(loc0p.reshape(-1))
    p += list(LP0.reshape(-1)) + [hP0]
    return {"model": _lib.MODEL_MVLINGAUSS, "params": p, "dim": dx, "dy": dy, "n_noise": dx,
            "proposal": True}


_SPECS = {"StochVol": spec_stochvol, "LinearGauss": spec_lingauss, "Gordon_etal": spec_gordon,
          "ThetaLogistic": spec_thetalogistic, "BearingsOnly": spec_bearings,
          "MVLinearGauss": spec_mvlingauss, "MVLinearGauss_Guarniero_etal": spec_mvlingauss,
          "StochVolLeverage": spec_stochvollev, "DiscreteCox": spec_discretecox}


_SMOOTHING_HOOKS = {"add_func", "upper_bound_log_pt", "upper_bound_trans"}
_INERT = {"__module__", "__qualname__", "__doc__", "__dict__", "__weakref__", "__firstlineno__",
          "__static_attributes__"}


def _hooks_base(cls):
    """``cls``, or -- when it adds nothing to its single base but the smoothing hooks, which the filter never
    calls -- that base, recursively."""
    while len(cls.__bases__) == 1 and not (set(cls.__dict__) - _SMOOTHING_HOOKS - _INERT):
        cls = cls.__bases__[0]
    return cls


def fused_spec(fk, smoothing_hooks=False):
    """Return the fused-kernel description of ``fk`` or None if it is not a stock
    (Feynman-Kac kind, model) pair.  Only exact stock classes are recognised: a user
    subclass that overrides a closure has another class name or module and takes the
    generic plugin path instead.  With ``smoothing_hooks`` (the run smooths on-line), a
    subclass that adds only ``add_func``, ``upper_bound_log_pt`` or ``upper_bound_trans``
    to a stock class counts as that class."""
    base = _hooks_base if smoothing_hooks else (lambda c: c)
    fk_cls = base(type(fk))
    names = [c.__name__ for c in fk_cls.__mro__]
    kind = next((code for nm, code in _FK_KINDS if nm in names), None)
    if kind is None or fk_cls.__name__ not in [k for k, _ in _FK_KINDS]:
        return None
    ssm = getattr(fk, "ssm", None)
    ssm_cls = None if ssm is None else base(type(ssm))
    if ssm is None or ssm_cls.__module__ not in _TRUSTED_MODULES:
        return None
    make = _SPECS.get(ssm_cls.__name__)
    if make is None:
        return None
    if getattr(ssm, "batch", None) is not None:
        raise ValueError(f"fused_spec: a batch of B = {ssm.batch} {ssm_cls.__name__} models runs in kalman.Kalman only")
    spec = make(ssm, fk.T, fk.data) if make in (spec_mvlingauss, spec_discretecox) else make(ssm, fk.T)
    if spec is None:
        return None
    if kind != _lib.FK_BOOTSTRAP and not spec["proposal"]:
        return None
    if kind == _lib.FK_GUIDED and type(ssm).__name__ == "ThetaLogistic":
        return None
    spec["fk"] = kind
    spec["data"] = _flat_data(fk.data, spec.get("dy", 1))
    return spec


def _defining_class(cls, name):
    return next((c for c in cls.__mro__ if name in c.__dict__), None)


def transition_spec(fk):
    """Return the device description of ``fk.logpt(t, xp, x) = PX(t, xp).logpdf(x)`` (backward sampling,
    csrc/smcb_smooth.cu) or None if the density must be evaluated by calling ``fk.logpt``.

    Wider than ``fused_spec``: smoothing users subclass a stock model to add ``upper_bound_log_pt`` or
    ``add_func`` (the reference's book scripts do), so the model is accepted when the class that DEFINES ``PX`` in
    its MRO is a stock class, and the Feynman-Kac object's ``logpt`` is ``Bootstrap.logpt`` (ours or the
    reference's, inherited by every Feynman-Kac kind).  Keys: model, params, dim, step_consts (or None)."""
    owner = _defining_class(type(fk), "logpt")
    if owner is None or owner.__name__ != "Bootstrap" or owner.__module__ not in _TRUSTED_MODULES:
        return None
    ssm = getattr(fk, "ssm", None)
    px = None if ssm is None else _defining_class(type(ssm), "PX")
    if px is None or px.__module__ not in _TRUSTED_MODULES:
        return None
    make = _SPECS.get(px.__name__)
    if make is None:
        return None
    data = getattr(fk, "data", None)
    T = 0 if data is None else len(data)
    if make is spec_discretecox:        # its step constants describe the observations, not PX: none needed here
        spec = make(ssm, T, [np.zeros(1)] * max(T, 1))
    elif make is spec_mvlingauss:
        spec = make(ssm, T, None)
    else:
        spec = make(ssm, T)
    if spec is None:
        return None
    return {"model": spec["model"], "params": list(spec["params"]), "dim": int(spec.get("dim", 1)),
            "step_consts": spec.get("step_consts") if make is spec_gordon else None}
