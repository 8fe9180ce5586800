"""A bank of resumable particle filters on the device: the inner filters of SMC^2 (``smc_samplers.SMC2``).

``FilterBank`` owns the device rows of R filters of one 1-D stock model, Feynman-Kac kind, resampling scheme, N and
data (csrc/smcb_bank.cu, DESIGN.md section 5.8): the last two generations X (R, 2, ld), the log-weights lw (R, ld),
the recursion's scalars ``state`` (R, 8), the model constants ``params`` (R, p), the per-filter step constants (or one
shared row) and the Philox key of each filter.  ``advance`` runs every selected filter up to a common step in one
launch; ``gather`` and ``merge`` are the outer sampler's X[A] and Metropolis copy-where on the rows.

``ThetaMap`` turns the rows of a parameter matrix into those model constants with the expressions of the scalar
``spec_*`` functions of ``state_space_models``, vectorised over the rows.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .device import context, ptr

STATE_T, STATE_LOGLT, STATE_LOGLT_STEP = 0, 1, 7      # columns of the state row (include/smcb.h SMCB_BANK_STATE)


# ---------------------------------------------------------------------------------------------- theta -> params
def _stochvol(p):
    mu, rho, sigma = p["mu"], p["rho"], p["sigma"]
    sig0 = sigma / np.sqrt(1.0 - rho ** 2)
    return [mu, rho, sigma, sig0, (1.0 - rho) * mu, np.log(sigma), np.log(sig0)]


def _stochvollev(p):
    sq = np.sqrt(1.0 - p["phi"] ** 2)
    return _stochvol(p) + [p["phi"], sq, np.log(sq)]


def _pysq(v):
    """v ** 2 of Python floats (libm pow), as spec_lingauss squares them: NumPy's array power is a product, which
    may round differently by one ulp."""
    return np.array([float(a) ** 2 for a in v], dtype=np.float64)


def _lingauss(p):
    sX, sY, rho = p["sigmaX"], p["sigmaY"], p["rho"]
    s0 = p["sigma0"]
    sX2, sY2 = _pysq(sX), _pysq(sY)
    s2p0 = 1.0 / (1.0 / _pysq(s0) + 1.0 / sY2)
    s2p = 1.0 / (1.0 / sX2 + 1.0 / sY2)
    se = np.sqrt(sX2 + sY2)
    return [rho, sX, sY, s0, np.log(sX), np.log(sY), np.log(s0),
            s2p0, np.sqrt(s2p0), np.log(np.sqrt(s2p0)), s2p, np.sqrt(s2p), np.log(np.sqrt(s2p)),
            se, np.log(se), sX2, sY2]


def _gordon(p):
    return [p["a"], p["b"], p["c"], p["sigmaX"], np.log(p["sigmaX"])]


def _thetalogistic(p):
    return [p["tau0"], p["tau1"], p["tau2"], p["sigmaX"], p["sigmaY"], np.log(p["sigmaX"]), np.log(p["sigmaY"])]


def _discretecox(p):
    sig0 = p["sigma"] / np.sqrt(1.0 - p["phi"] ** 2)
    return [p["mu"], p["sigma"], p["phi"], sig0, np.log(p["sigma"]), np.log(sig0)]


# class name -> (model id, constants, the kinds with a proposal are built, default parameters)
_MAPS = {
    "StochVol": (_lib.MODEL_STOCHVOL, _stochvol, True, {"mu": -1.02, "rho": 0.9702, "sigma": 0.178}),
    "StochVolLeverage": (_lib.MODEL_STOCHVOLLEV, _stochvollev, False,
                         {"mu": -1.02, "rho": 0.9702, "sigma": 0.178, "phi": 0.0}),
    "LinearGauss": (_lib.MODEL_LINGAUSS, _lingauss, True, {"sigmaY": 0.2, "rho": 0.9, "sigmaX": 1.0, "sigma0": None}),
    "Gordon_etal": (_lib.MODEL_GORDON, _gordon, False,
                    {"a": 0.05, "b": 0.5, "c": 25.0, "d": 8.0, "e": 1.2, "sigmaX": 3.162278}),
    "ThetaLogistic": (_lib.MODEL_THETALOGISTIC, _thetalogistic, False,
                      {"tau0": 0.15, "tau1": 0.12, "tau2": 0.1, "sigmaX": 0.47, "sigmaY": 0.39}),
    "DiscreteCox": (_lib.MODEL_DISCRETECOX, _discretecox, False, {"mu": 0.0, "sigma": 1.0, "phi": 0.95}),
}
SUPPORTED = tuple(_MAPS)


class ThetaMap:
    """Rows of theta (named columns) -> the (n, p) model constants and step constants of the bank's kernel.

    Parameters the columns do not name take the class's ``default_params``, as ``ssm_cls(**theta)`` does
    (LinearGauss: sigma0 = sigmaX / sqrt(1 - rho^2) when neither names it)."""

    def __init__(self, ssm_cls, names, data):
        from .state_space_models import _TRUSTED_MODULES
        name = getattr(ssm_cls, "__name__", None)
        if name not in _MAPS or getattr(ssm_cls, "__module__", None) not in _TRUSTED_MODULES:
            raise NotImplementedError(
                "SMC2 on the device runs the stock 1-D models %s (of particles or particles_b200); %r is not one of "
                "them" % (", ".join(SUPPORTED), ssm_cls))
        self.model, self._fn, self.proposal, defaults = _MAPS[name]
        self.defaults = dict(defaults)
        self.defaults.update(getattr(ssm_cls, "default_params", None) or {})
        self.names = list(names)
        self.data = np.asarray(data, dtype=np.float64).reshape(-1)
        self.T = self.data.shape[0]
        self.name = name
        # step constants that do not depend on theta: one shared row
        self.shared_sc = None
        if name == "DiscreteCox":
            from scipy.special import gammaln
            self.shared_sc = gammaln(self.data + 1.0)
        self.n_params = self.params(np.empty((0, len(self.names)))).shape[1]

    def columns(self, theta):
        """theta (n, p) host array whose columns follow ``names`` -> {parameter: (n,) array} with the defaults."""
        theta = np.asarray(theta, dtype=np.float64)
        n = theta.shape[0]
        cols = {k: theta[:, i].copy() for i, k in enumerate(self.names)}
        for k, v in self.defaults.items():
            if k not in cols and v is not None:
                cols[k] = np.full(n, float(v))
        if self.name == "LinearGauss" and "sigma0" not in cols:
            cols["sigma0"] = cols["sigmaX"] / np.sqrt(1.0 - cols["rho"] ** 2)
        return cols

    def params(self, theta):
        """(n, p) model constants, column j = the j-th constant of spec_*(ssm_cls(**theta_i))."""
        cols = self.columns(theta)
        n = np.asarray(theta).shape[0]
        with np.errstate(invalid="ignore", divide="ignore"):     # proposals outside the model's domain: NaN rows,
            rows = self._fn(cols)                                # never run (their prior density is 0)
        return np.ascontiguousarray(np.stack([np.broadcast_to(np.asarray(v, dtype=np.float64), (n,))
                                              for v in rows], axis=1))

    def step_consts(self, theta):
        """(n, T) per-filter step constants (Gordon_etal: d cos(e (t - 1))), or None."""
        if self.name != "Gordon_etal":
            return None
        c = self.columns(theta)
        t = np.arange(self.T)
        return np.ascontiguousarray(c["d"][:, None] * np.cos(c["e"][:, None] * (t[None, :] - 1)))


# ---------------------------------------------------------------------------------------------- the bank
class FilterBank:
    """R filters of N particles: device rows and the launches that work on them."""

    def __init__(self, model, fk, scheme, N, R, data_dev, n_params, essrmin, shared_sc=None, per_filter_sc=False,
                 tier="auto"):
        self.model, self.fk, self.scheme = int(model), int(fk), scheme
        self.N, self.R, self.T = int(N), int(R), int(data_dev.shape[0])
        self.ld = self.N + (self.N & 1)
        self.data, self.n_params, self.essrmin = data_dev, int(n_params), float(essrmin)
        self.tier = _lib.BATCH_TIERS[tier]
        self._tier_name = tier
        dev = data_dev.device
        f64 = dict(dtype=torch.float64, device=dev)
        R, ld, T = self.R, self.ld, self.T
        self.X = torch.zeros((R, 2, ld), **f64)
        self.lw = torch.zeros((R, ld), **f64)
        self.state = torch.zeros((R, _lib.BANK_STATE), **f64)
        self.params = torch.zeros((R, self.n_params), **f64)
        self.key = torch.zeros(R, dtype=torch.int64, device=dev)
        self.shared_sc = shared_sc
        self.sc = torch.zeros((R, T), **f64) if per_filter_sc else None
        self._scr = None
        self.timer = None          # None, or a list that receives (start, end) CUDA events around each advance

    def empty_like(self, R=None):
        return FilterBank(self.model, self.fk, self.scheme, self.N, self.R if R is None else R, self.data,
                          self.n_params, self.essrmin, self.shared_sc, self.sc is not None, self._tier_name)

    def desc(self):
        d = _lib.BankDesc()
        d.model, d.fk, d.scheme, d.tier = self.model, self.fk, _lib.RS_CODES[self.scheme], self.tier
        d.n_params, d.N, d.T, d.R = self.n_params, self.N, self.T, self.R
        d.essrmin = self.essrmin
        d.key, d.params, d.data = self.key.data_ptr(), self.params.data_ptr(), self.data.data_ptr()
        if self.sc is not None:
            d.step_consts, d.sc_ld = self.sc.data_ptr(), self.T
        elif self.shared_sc is not None:
            d.step_consts, d.sc_ld = self.shared_sc.data_ptr(), 0
        d.X, d.lw, d.state = self.X.data_ptr(), self.lw.data_ptr(), self.state.data_ptr()
        return d

    def plan(self):
        """(tier, grid) of an advance of every filter."""
        d = self.desc()
        out = (C.c_int64 * 2)()
        ctx = context()
        _lib.check(ctx.lib.smcb_bank_plan(ctx.handle, C.byref(d), out))
        return int(out[0]), int(out[1])

    def set_rows(self, params, sc=None):
        """Upload the model constants (n, p) (and step constants) of every filter."""
        self.params.copy_(torch.from_numpy(np.ascontiguousarray(params, dtype=np.float64)))
        if self.sc is not None:
            self.sc.copy_(torch.from_numpy(np.ascontiguousarray(sc, dtype=np.float64)))

    def fresh_keys(self, seed, counter, rows=None):
        """Keys number counter, counter + 1, ... under ``seed`` for every filter (or the first ``rows``)."""
        n = self.R if rows is None else int(rows)
        ctx = context()
        _lib.check(ctx.lib.smcb_bank_keys(ctx.handle, ptr(self.key), n, int(seed) & (2 ** 64 - 1),
                                          int(counter) & (2 ** 64 - 1)))

    def advance(self, t1, idx=None, restart=False, summaries=None, A=None):
        """Run every filter (or the filters ``idx``, an int64 CUDA tensor) from its step to step ``t1``; ``restart``
        starts them from M0.  ``summaries`` (R, T, 4) / ``A`` (R, ld): optional outputs."""
        d = self.desc()
        d.t1, d.restart = int(t1), int(bool(restart))
        if idx is not None:
            d.idx, d.n_idx = idx.data_ptr(), int(idx.shape[0])
        d.summaries = None if summaries is None else summaries.data_ptr()
        d.A = None if A is None else A.data_ptr()
        ctx = context()
        ctx.bind_stream()
        plan = (C.c_int64 * 2)()
        _lib.check(ctx.lib.smcb_bank_plan(ctx.handle, C.byref(d), plan))
        if plan[0] == _lib.BATCH_STREAMING:
            rows = int(plan[1])
            multi = self.scheme == "multinomial"
            if self._scr is None or self._scr[0].shape[0] < rows:
                f64 = dict(dtype=torch.float64, device=self.data.device)
                self._scr = (torch.empty((rows, self.ld), **f64),
                             torch.empty((rows, self.ld + 2), **f64) if multi else None)
            d.cdf = self._scr[0].data_ptr()
            d.scratch = None if self._scr[1] is None else self._scr[1].data_ptr()
            d.scratch_rows = self._scr[0].shape[0]
        ev = None
        if self.timer is not None:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        _lib.check(ctx.lib.smcb_bank_advance(ctx.handle, C.byref(d)))
        if ev is not None:
            ev[1].record()
            self.timer.append(ev)

    def gather(self, A, seed, counter):
        """A new bank with rows ``self[A[i]]``: the first copy of an ancestor keeps its key, further copies take the
        keys number ``counter + i`` under ``seed``."""
        out = self.empty_like(int(A.shape[0]))
        first = torch.empty(max(self.R, 1), dtype=torch.int64, device=self.data.device)
        ctx = context()
        s, d = self.desc(), out.desc()
        _lib.check(ctx.lib.smcb_bank_gather(ctx.handle, C.byref(s), ptr(A), int(A.shape[0]), C.byref(d),
                                            int(seed) & (2 ** 64 - 1), int(counter) & (2 ** 64 - 1), ptr(first)))
        out.timer = self.timer
        return out

    def merge(self, src, accepted):
        """Rows of ``src`` where ``accepted`` (uint8 CUDA tensor), in place."""
        ctx = context()
        d, s = self.desc(), src.desc()
        _lib.check(ctx.lib.smcb_bank_merge(ctx.handle, C.byref(d), C.byref(s), ptr(accepted)))

    @classmethod
    def concatenate(cls, *banks):
        out = banks[0].empty_like(sum(b.R for b in banks))
        for name in ("X", "lw", "state", "params", "key") + (("sc",) if banks[0].sc is not None else ()):
            torch.cat([getattr(b, name) for b in banks], out=getattr(out, name))
        out.timer = banks[0].timer
        return out

    @property
    def logLt(self):
        return self.state[:, STATE_LOGLT]

    @property
    def loglt(self):
        return self.state[:, STATE_LOGLT_STEP]
