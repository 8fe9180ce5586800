"""Probability distributions on the device -- the ``ProbDist`` subset that sits on the
SMC hot path (SURVEY.md section 8 rows a19-a21), same constructor arguments and
``rvs`` / ``logpdf`` semantics as ``particles/distributions.py``.

Parameters may be Python scalars or CUDA fp64 tensors of shape (N,) (resp. (N, d) /
(d,) for MvNormal); array-valued parameters make the object a Markov kernel, exactly
as in the reference (distributions.py:135-154).  Randomness comes from the context's
Philox stream (``particles_b200.seed``); ``rvs(size, z=...)`` accepts injected
standard normals for deterministic parity tests.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .device import as_device, context, empty, ptr

HALFLOG2PI = 0.5 * np.log(2.0 * np.pi)


def ndtri(u):
    """Phi^-1(u) on the device (csrc/smcb_sqmc.cuh; within 8 ulp of scipy.special.ndtri on the squeezed range)."""
    u = as_device(u)
    out = torch.empty_like(u)
    ctx = context()
    _lib.check(ctx.lib.smcb_ndtri(ctx.handle, ptr(u), ptr(out), u.numel()))
    return out


def _split(v):
    """scalar-or-array argument -> (device tensor or None, scalar).  A size-1 array or tensor is a scalar that
    broadcasts -- ``StateSpaceModel.simulate`` returns observations of shape (1,), and NumPy broadcasts
    ``data[t]`` against the (N,) particles (SURVEY.md section 9.10)."""
    if isinstance(v, (int, float)):                     # numpy.float64 too
        return None, float(v)
    if isinstance(v, torch.Tensor):
        if v.numel() == 1:
            return None, float(v.reshape(-1)[0].item())
        return as_device(v), 0.0
    if isinstance(v, np.ndarray) and v.ndim > 0 and v.size > 1:
        return as_device(v), 0.0
    return None, float(np.asarray(v).reshape(-1)[0])


class ProbDist:
    """particles/distributions.py:215-251."""
    dim = 1
    dtype = float

    def shape(self, size):
        if size is None:
            return None
        return (size,) if self.dim == 1 else (size, self.dim)

    def logpdf(self, x):
        raise NotImplementedError

    def rvs(self, size=None):
        raise NotImplementedError

    def ppf(self, u):
        raise NotImplementedError   # SQMC only: out of scope (SURVEY.md section 2 row 3)


class LocScaleDist(ProbDist):
    """particles/distributions.py:259-264."""

    def __init__(self, loc=0.0, scale=1.0):
        self.loc = loc
        self.scale = scale


def _common_length(size, *arrs):
    """Common length of the array arguments (scalars broadcast); mismatched lengths are an error, as NumPy's
    broadcasting would make them."""
    lens = {int(a.shape[0]) for a in arrs if a is not None}
    if len(lens) > 1:
        raise ValueError(f"operands could not be broadcast together with lengths {sorted(lens)}")
    if lens:
        return lens.pop()
    return 1 if size is None else int(size)


class _KernelLaw(ProbDist):
    """A law with a device log-density, law code ``_law`` of include/smcb.h, and, for codes 0-7, a device sampler.
    Its parameters, ``_params()``, are scalars or (N,) arrays / tensors: array parameters make it a Markov kernel,
    as in the reference (distributions.py:135-154)."""
    _law = None

    def _params(self):
        raise NotImplementedError

    def _args(self):
        """-> the four parameters' device arrays (None for a scalar) and the host array of their scalars"""
        arrays, scalars = [None] * 4, (C.c_double * 4)()
        for k, v in enumerate(self._params()):
            arrays[k], scalars[k] = _split(v)
        return arrays, scalars

    def logpdf(self, x):
        xa, x0 = _split(x)
        arrays, scalars = self._args()
        n = _common_length(None, xa, *arrays)
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_dist_logpdf(ctx.handle, self._law, ptr(xa), x0, *map(ptr, arrays), scalars,
                                            ptr(out), n))
        return out

    def rvs(self, size=None):
        arrays, scalars = self._args()
        n = _common_length(size, *arrays)
        if size is not None and int(size) != n:        # numpy.random's broadcast error
            raise ValueError(f"shape mismatch: {n} parameter values cannot be broadcast to size {int(size)}")
        ctx = context()
        out = empty(n, dtype=torch.int64 if self.dtype == np.int64 else torch.float64)
        _lib.check(ctx.lib.smcb_dist_rvs(ctx.handle, self._law, *map(ptr, arrays), scalars, ptr(out), n))
        return out


class Normal(LocScaleDist, _KernelLaw):
    """N(loc, scale^2) -- particles/distributions.py:267-285."""
    _law = _lib.LAW_NORMAL

    def _params(self):
        return self.loc, self.scale

    def rvs(self, size=None, z=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        zd = None if z is None else as_device(z)
        n = _common_length(size, la, sa, zd)
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_normal_rvs(ctx.handle, ptr(la), l0, ptr(sa), s0, ptr(zd), ptr(out), n))
        return out

    def ppf(self, u):
        """scipy.stats.norm.ppf(u, loc, scale) = loc + scale * Phi^-1(u), on the device."""
        return self.rvs(z=ndtri(u))

    def posterior(self, x, sigma=1.0):
        """particles/distributions.py:279-285: X_1..X_n ~ N(theta, sigma^2), theta ~ self (host arithmetic)."""
        x = _host(x)
        pr0 = 1.0 / _host(self.scale) ** 2
        prd = x.size / sigma ** 2
        varp = 1.0 / (pr0 + prd)
        mu = varp * (pr0 * _host(self.loc) + prd * x.mean())
        return Normal(loc=mu, scale=np.sqrt(varp))


class Student(_KernelLaw):
    """Student(df, loc, scale) -- particles/distributions.py:417-433 (scipy.stats.t.logpdf); ``df`` scalar."""
    _law = _lib.LAW_STUDENT

    def __init__(self, df=3.0, loc=0.0, scale=1.0):
        self.df, self.loc, self.scale = df, loc, scale

    def _params(self):
        from scipy.special import gammaln
        df = float(self.df)
        return df, self.loc, self.scale, gammaln(0.5 * (df + 1.0)) - gammaln(0.5 * df) - 0.5 * np.log(df * np.pi)

    def rvs(self, size=None):
        """loc + scale * z / sqrt(chi2_df / df): the normals from the context's Philox stream, the chi-square
        from torch's generator (the reference draws through scipy.stats.t.rvs)."""
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = _common_length(size, la, sa)
        z = Normal().rvs(size=n)
        g = torch.distributions.Chi2(torch.tensor(float(self.df), dtype=torch.float64, device=z.device)).sample((n,))
        t = z / torch.sqrt(g / float(self.df))
        return (la if la is not None else l0) + (sa if sa is not None else s0) * t


class Gamma(_KernelLaw):
    """Gamma(a, b), density prop. to x^(a-1) exp(-b x) -- particles/distributions.py:336-356; ``a`` scalar,
    ``b`` scalar or per-particle array."""
    _law = _lib.LAW_GAMMA

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = a, b
        self.scale = 1.0 / b

    def _params(self):
        from scipy.special import gammaln
        return float(self.a), self.b, -gammaln(float(self.a))

    def posterior(self, x):
        """particles/distributions.py:353-355: X_1..X_n ~ N(0, 1/theta), theta ~ self."""
        x = _host(x)
        return Gamma(a=self.a + 0.5 * x.size, b=self.b + 0.5 * np.sum(x ** 2))

    def rvs(self, size=None):
        b = as_device(self.b) if isinstance(self.b, (torch.Tensor, np.ndarray)) else \
            torch.full((1 if size is None else int(size),), float(self.b), dtype=torch.float64, device="cuda")
        a = torch.full_like(b, float(self.a))
        return torch.distributions.Gamma(a, b).sample()


class Laplace(LocScaleDist, _KernelLaw):
    """particles/distributions.py:301-314."""
    _law = _lib.LAW_LAPLACE

    def _params(self):
        return self.loc, self.scale

    def rvs(self, size=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = _common_length(size, la, sa)
        u = torch.rand(n, dtype=torch.float64, device="cuda") - 0.5
        return (la if la is not None else l0) - (sa if sa is not None else s0) * torch.sign(u) * torch.log1p(-2 * u.abs())


class Logistic(LocScaleDist, _KernelLaw):
    """particles/distributions.py:288-299."""
    _law = _lib.LAW_LOGISTIC

    def _params(self):
        return self.loc, self.scale

    def rvs(self, size=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = _common_length(size, la, sa)
        u = torch.rand(n, dtype=torch.float64, device="cuda")
        return (la if la is not None else l0) + (sa if sa is not None else s0) * (torch.log(u) - torch.log1p(-u))


def _host(v):
    """A log-density or draw (CUDA tensor, NumPy array or scalar) as a host fp64 array."""
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy().astype(np.float64)
    return np.asarray(v, dtype=np.float64)


class Uniform(ProbDist):
    """Uniform([a, b]) -- particles/distributions.py:399-414.  A law of static parameters: ``logpdf`` runs on the
    host (NumPy in, NumPy out, scipy.stats.uniform's closed support); ``rvs`` draws from the context's Philox
    stream."""

    def __init__(self, a=0.0, b=1.0):
        self.a, self.b = a, b
        self.scale = b - a

    def rvs(self, size=None):
        n = 1 if size is None else int(size)
        ctx = context()
        u = empty(n)
        _lib.check(ctx.lib.smcb_uniform(ctx.handle, ptr(u), n))
        return self.a + self.scale * u

    def logpdf(self, x):
        x = _host(x)
        return np.where((x >= self.a) & (x <= self.a + self.scale), -np.log(self.scale), -np.inf)


class Beta(ProbDist):
    """Beta(a, b) -- particles/distributions.py:319-333; ``logpdf`` on the host (scipy.stats.beta's formula),
    ``rvs`` from torch's generator as Gamma.rvs."""

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = a, b

    def rvs(self, size=None):
        n = 1 if size is None else int(size)
        a = torch.full((n,), float(self.a), dtype=torch.float64, device="cuda")
        return torch.distributions.Beta(a, torch.full_like(a, float(self.b))).sample()

    def logpdf(self, x):
        from scipy.special import betaln, xlog1py, xlogy
        x = _host(x)
        a, b = float(self.a), float(self.b)
        with np.errstate(divide="ignore", invalid="ignore"):
            lp = xlog1py(b - 1.0, -x) + xlogy(a - 1.0, x) - betaln(a, b)
        return np.where((x > 0.0) & (x < 1.0), lp, -np.inf)


class StructDist(ProbDist):
    """Independent laws of named parameters -- particles/distributions.py:1149-1214.  ``rvs(size)`` returns a
    NumPy structured array (fields in sorted order for a dict, as in the reference), ``logpdf(theta)`` the host
    array of the summed log-densities.  A law with ``dim > 1`` (``MvNormal``) gets a vector field
    ``(name, float, (dim,))``; every other law a scalar field.  The component laws may be this package's (device
    draws, copied to the host) or any object with the same two methods; a callable law (``Cond``) receives the
    structured array."""

    def __init__(self, laws):
        from collections import OrderedDict
        if isinstance(laws, OrderedDict):
            self.laws = laws
        elif isinstance(laws, dict):
            self.laws = OrderedDict([(k, laws[k]) for k in sorted(laws)])
        else:
            raise TypeError("recdist class requires a dict or an ordered dict to be instantiated")
        self.dtype = [(k, float) if getattr(law, "dim", 1) == 1 else (k, float, (law.dim,))
                      for k, law in self.laws.items()]

    def logpdf(self, theta):
        lp = 0.0
        for par, law in self.laws.items():
            cond = law(theta) if callable(law) else law
            lp = lp + _host(cond.logpdf(theta[par]))
        return lp

    def rvs(self, size=1):
        out = np.empty(size, dtype=self.dtype)
        for par, law in self.laws.items():
            cond = law(out) if callable(law) else law
            out[par] = _host(cond.rvs(size=size)).reshape(out[par].shape)
        return out


class DiscreteDist(ProbDist):
    """Base class of the discrete laws -- particles/distributions.py:513-516: ``rvs`` returns int64 CUDA tensors."""
    dtype = np.int64


class Categorical(DiscreteDist):
    """Categorical(p), p (k,) or (N, k) -- particles/distributions.py:598-628."""

    def __init__(self, p=None):
        if p is None:
            raise ValueError("Categorical: missing argument p")
        self.p = as_device(p)

    def logpdf(self, x):
        lp = torch.log(self.p)
        x = as_device(x, dtype=torch.int64)
        if lp.ndim == 1:
            return lp[x]
        return lp.gather(1, x.reshape(-1, 1).expand(lp.shape[0], 1)).reshape(-1)      # np.choose(x, columns)

    def rvs(self, size=None):
        from . import resampling as rs
        if self.p.ndim == 1:                                   # searchsorted(cumsum(p), u)
            n = 1 if size is None else int(size)
            u = torch.sort(torch.rand(n, dtype=torch.float64, device="cuda"))
            out = torch.empty(n, dtype=torch.int64, device="cuda")
            out[u.indices] = rs.inverse_cdf(u.values, self.p)
            return out
        n = self.p.shape[0] if size is None else int(size)
        u = torch.rand(n, 1, dtype=torch.float64, device="cuda")
        return (torch.cumsum(self.p[:n], 1) < u).sum(1).clamp_(max=self.p.shape[1] - 1)


class MixMissing(ProbDist):
    """Mixture of ``base_dist`` and 'missing' (NaN) -- particles/distributions.py:819-847."""

    def __init__(self, pmiss=0.10, base_dist=None):
        self.pmiss, self.base_dist = pmiss, base_dist

    def logpdf(self, x):
        xd = as_device(x)
        lp = self.base_dist.logpdf(torch.nan_to_num(xd, nan=0.0) if bool(torch.isnan(xd).any()) else xd)
        ina = torch.isnan(xd).reshape(-1)
        if ina.shape[0] == 1:
            ina = ina.expand(lp.shape[0])
        return torch.where(ina, torch.full_like(lp, float(np.log(self.pmiss))), lp + float(np.log(1.0 - self.pmiss)))

    def rvs(self, size=None):
        x = self.base_dist.rvs(size=size)
        miss = torch.rand(x.shape[0], dtype=torch.float64, device=x.device) < self.pmiss
        x[miss] = float("nan")
        return x


class Poisson(DiscreteDist):
    """Poisson(rate) -- particles/distributions.py:519-532 (logpdf on the device; ``rate`` a CUDA
    tensor or scalar, ``x`` the observed count).  scipy evaluates xlogy(k, mu) - gammaln(k+1) - mu."""

    def __init__(self, rate=1.0):
        self.rate = rate

    def rvs(self, size=None):
        r = as_device(self.rate) if isinstance(self.rate, (torch.Tensor, np.ndarray)) else \
            torch.full((1 if size is None else size,), float(self.rate), dtype=torch.float64, device="cuda")
        return torch.poisson(r)

    def logpdf(self, x):
        from scipy.special import gammaln
        k = float(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x).reshape(-1)[0])
        rate = as_device(self.rate) if isinstance(self.rate, (torch.Tensor, np.ndarray)) else \
            torch.full((1,), float(self.rate), dtype=torch.float64, device="cuda")
        xl = 0.0 if k == 0 else k * torch.log(rate)
        return xl - float(gammaln(k + 1.0)) - rate


class Dirac(ProbDist):
    """Dirac mass -- particles/distributions.py:454-472."""

    def __init__(self, loc=0.0):
        self.loc = loc

    def rvs(self, size=None, z=None):
        if isinstance(self.loc, torch.Tensor) and self.loc.ndim > 0:
            return self.loc.clone()
        n = 1 if size is None else size
        return torch.full((n,), float(self.loc), dtype=torch.float64, device="cuda")

    def ppf(self, u):
        return self.rvs(size=u.shape[0])                 # distributions.py:471-472

    def logpdf(self, x):
        x = as_device(x)
        loc = self.loc if isinstance(self.loc, torch.Tensor) else float(self.loc)
        zero = torch.zeros((), dtype=torch.float64, device=x.device)
        return torch.where(x == loc, zero, zero - float("inf"))


class IndepProd(ProbDist):
    """Product of independent univariate laws -- particles/distributions.py:1066-1109.
    Inputs / outputs are (N, d) tensors."""

    def __init__(self, *dists):
        self.dists = dists
        self.dim = len(dists)

    def logpdf(self, x):
        x = as_device(x)
        out = None
        for i, d in enumerate(self.dists):
            li = d.logpdf(x[..., i].contiguous())
            out = li if out is None else out + li
        return out

    def rvs(self, size=None, z=None):
        cols, k = [], 0
        for d in self.dists:
            if isinstance(d, Dirac) or z is None:
                cols.append(d.rvs(size=size))
            else:
                cols.append(d.rvs(size=size, z=as_device(z)[:, k].contiguous()))
                k += 1
        return torch.stack(cols, dim=1)

    def ppf(self, u):
        """Column i of u through law i's ppf (distributions.py:1108-1109)."""
        u = as_device(u)
        return torch.stack([d.ppf(u[..., i].contiguous()) for i, d in enumerate(self.dists)], dim=1)


class IID(IndepProd):
    """Joint law of k iid copies of ``law`` -- particles/distributions.py:1111-1121 (there IndepProd(*[law] * k));
    (N, k) inputs / outputs.  A law with a joint device kernel for its iid product (``binary_smc.Bernoulli``) is
    drawn and evaluated by that kernel, in the reference's order of draws and terms."""

    def __init__(self, law, k):
        super().__init__(*[law for _ in range(k)])
        self.law = law

    def rvs(self, size=None, z=None):
        joint = getattr(self.law, "_iid", None)
        if joint is not None:
            return joint(self.dim).rvs(size=1 if size is None else size)
        return super().rvs(size=size, z=z)

    def logpdf(self, x):
        joint = getattr(self.law, "_iid", None)
        if joint is not None:
            return joint(self.dim).logpdf(x)
        return super().logpdf(x)


class MvNormal(ProbDist):
    """Multivariate Normal -- particles/distributions.py:888-982 (d <= 32 on the device).
    ``loc``: (d,) or (N, d); ``scale``: scalar, (d,) or (N, d); ``cov``: (d, d) host array."""

    def __init__(self, loc=0.0, scale=1.0, cov=None):
        self.loc = loc
        self.scale = scale
        if cov is None:
            cov = np.eye(loc.shape[-1])
        self.cov = np.asarray(cov.cpu() if isinstance(cov, torch.Tensor) else cov, dtype=np.float64)
        err_msg = "MvNormal: argument cov must be a (d, d) pos. definite matrix"
        try:
            self.L = np.linalg.cholesky(self.cov)     # distributions.py:937
        except np.linalg.LinAlgError:
            raise ValueError(err_msg)
        assert self.cov.shape == (self.dim, self.dim), err_msg

    @property
    def dim(self):
        return self.cov.shape[-1]

    def _params(self, v, default):
        """-> (SoA device array (d, n) or None, host vector (d,))"""
        d = self.dim
        if isinstance(v, torch.Tensor):
            if v.ndim == 2:
                return v.t().contiguous(), None
            v = v.cpu().numpy()
        a = np.asarray(v, dtype=np.float64)
        if a.ndim == 2:
            return as_device(a).t().contiguous(), None
        return None, np.ascontiguousarray(np.broadcast_to(a, (d,)), dtype=np.float64)

    @staticmethod
    def _hp(a):
        return None if a is None else a.ctypes.data_as(C.c_void_p)

    def rvs(self, size=None, z=None):
        d = self.dim
        la, l0 = self._params(self.loc, 0.0)
        sa, s0 = self._params(self.scale, 1.0)
        zd = None if z is None else as_device(z).t().contiguous()
        n = la.shape[1] if la is not None else (sa.shape[1] if sa is not None else
                                                (zd.shape[1] if zd is not None else
                                                 (1 if size is None else int(size))))
        ctx = context()
        out = empty((d, n))
        L = np.ascontiguousarray(self.L)
        _lib.check(ctx.lib.smcb_mvnormal_rvs(ctx.handle, ptr(la), self._hp(l0), ptr(sa), self._hp(s0),
                                             self._hp(L), d, ptr(zd), ptr(out), n))
        return out.t().contiguous()

    def ppf(self, u):
        """Rosenblatt transform through the Cholesky factor, loc + scale * Phi^-1(u) @ L.T; when u has fewer than d
        columns the remaining ones of z are 0 (distributions.py:971-983)."""
        u = as_device(u)
        u = u.reshape(u.shape[0], -1)
        z = ndtri(u)
        if z.shape[1] < self.dim:
            z = torch.cat([z, torch.zeros((z.shape[0], self.dim - z.shape[1]), dtype=z.dtype, device=z.device)], 1)
        return self.rvs(z=z)

    def logpdf(self, x):
        d = self.dim
        x = as_device(x)
        xs = x.reshape(-1, d).t().contiguous()
        la, l0 = self._params(self.loc, 0.0)
        sa, s0 = self._params(self.scale, 1.0)
        n = max(xs.shape[1], la.shape[1] if la is not None else 1,
                sa.shape[1] if sa is not None else 1)
        if xs.shape[1] == 1 and n > 1:             # one observation against N kernels
            xs = xs.expand(d, n).contiguous()
        ctx = context()
        out = empty(n)
        L = np.ascontiguousarray(self.L)
        _lib.check(ctx.lib.smcb_mvnormal_logpdf(ctx.handle, ptr(xs), ptr(la), self._hp(l0), ptr(sa),
                                                self._hp(s0), self._hp(L), d, ptr(out), n))
        return out

    def posterior(self, x, Sigma=None):
        """particles/distributions.py:984-1009: X_1..X_n ~ N(theta, Sigma), theta ~ self; scale must be one."""
        import scipy.linalg as sla
        if np.any(_host(self.scale) != 1.0):
            raise ValueError("posterior of MvNormal: scale must be one.")
        x = _host(x)
        n = x.shape[0]
        Sigma = np.eye(self.dim) if Sigma is None else _host(Sigma)
        Siginv = sla.inv(Sigma)
        covinv = sla.inv(self.cov)
        Sigpost = sla.inv(covinv + n * Siginv)
        loc = _host(self.loc)
        m = np.full(self.dim, float(loc)) if loc.ndim == 0 else loc
        mupost = Sigpost @ (m @ covinv + Siginv @ np.sum(x, axis=0))
        return MvNormal(loc=mupost, cov=Sigpost)


# ---------------------------------------------------------------------------------------------------------------------
# laws with a device sampler in csrc/smcb_dists.cuh (smcb_dist_rvs)
# ---------------------------------------------------------------------------------------------------------------------
class InvGamma(_KernelLaw):
    """Inverse Gamma(a, b) -- particles/distributions.py:358-377 (scipy.stats.invgamma(a, scale=b)); draws
    b / Gamma(a, 1) from the device Gamma sampler."""
    _law = _lib.LAW_INVGAMMA

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = a, b

    def _params(self):
        return self.a, self.b

    def posterior(self, x):
        """particles/distributions.py:374-376: X_1..X_n ~ N(0, theta), theta ~ self."""
        x = _host(x)
        return InvGamma(a=self.a + 0.5 * x.size, b=self.b + 0.5 * np.sum(x ** 2))


class LogNormal(_KernelLaw):
    """Law of exp(X), X ~ N(mu, sigma^2) -- particles/distributions.py:379-396."""
    _law = _lib.LAW_LOGNORMAL

    def __init__(self, mu=0.0, sigma=1.0):
        self.mu, self.sigma = mu, sigma

    def _params(self):
        return self.mu, self.sigma


class TruncNormal(_KernelLaw):
    """N(mu, sigma^2) truncated to [a, b] -- particles/distributions.py:475-505.  The log mass is computed in log
    space (finite in either far tail) and the draws are exact (smcb_dists.cuh: truncnorm_std_rvs)."""
    _law = _lib.LAW_TRUNCNORMAL

    def __init__(self, mu=0.0, sigma=1.0, a=0.0, b=1.0):
        self.mu, self.sigma, self.a, self.b = mu, sigma, a, b
        self.au = (a - mu) / sigma
        self.bu = (b - mu) / sigma

    def _params(self):
        return self.mu, self.sigma, self.a, self.b

    def posterior(self, x, s=1.0):
        """particles/distributions.py:499-505: X_1..X_n ~ N(theta, s^2), theta ~ self."""
        x = _host(x)
        pr0 = 1.0 / _host(self.sigma) ** 2
        prd = x.size / s ** 2
        varp = 1.0 / (pr0 + prd)
        mu = varp * (pr0 * _host(self.mu) + prd * x.mean())
        return TruncNormal(mu=mu, sigma=np.sqrt(varp), a=self.a, b=self.b)


class FlatNormal(ProbDist):
    """Normal with infinite variance, the law of a missing value -- particles/distributions.py:435-451: log-density
    zero of the broadcast shape of x and loc, draws loc + NaN."""

    def __init__(self, loc=0.0):
        self.loc = loc

    def logpdf(self, x):
        return torch.zeros(np.broadcast_shapes(np.shape(x), np.shape(self.loc)), dtype=torch.float64, device="cuda")

    def rvs(self, size=None):
        sz = 1 if size is None else int(size)
        loc = as_device(self.loc) if isinstance(self.loc, (torch.Tensor, np.ndarray)) else float(self.loc)
        return loc + torch.full((sz,), float("nan"), dtype=torch.float64, device="cuda")


class Binomial(DiscreteDist, _KernelLaw):
    """Binomial(n, p) -- particles/distributions.py:535-549.  logpdf is scipy.stats.binom.logpmf (Loader's
    saddle-point form: accurate for large n); draws by inversion while n min(p, 1 - p) < 10, BTRS otherwise."""
    _law = _lib.LAW_BINOMIAL

    def __init__(self, n=1, p=0.5):
        self.n, self.p = n, p

    def _params(self):
        return self.n, self.p


class Geometric(DiscreteDist, _KernelLaw):
    """Geometric(p) on 1, 2, ... -- particles/distributions.py:552-565."""
    _law = _lib.LAW_GEOMETRIC

    def __init__(self, p=0.5):
        self.p = p

    def _params(self):
        return (self.p,)


class NegativeBinomial(DiscreteDist, _KernelLaw):
    """Number of failures before the n-th success, p the success probability -- particles/distributions.py:568-595.
    Draws as numpy.random.negative_binomial(n, p): Poisson(Gamma(n, scale (1 - p) / p)).  logpdf is
    scipy.stats.nbinom.logpmf(x, n, p), the law of those draws; the reference's line 592 passes (p, n) in swapped
    order (DESIGN.md section 5.16)."""
    _law = _lib.LAW_NEGBINOMIAL

    def __init__(self, n=1, p=0.5):
        self.n, self.p = n, p

    def _params(self):
        return self.n, self.p


class DiscreteUniform(DiscreteDist, _KernelLaw):
    """Uniform on lo, lo + 1, ..., hi - 1 -- particles/distributions.py:631-649."""
    _law = _lib.LAW_DISCRETEUNIFORM

    def __init__(self, lo=0, hi=2):
        self.lo, self.hi = lo, hi
        width = hi - lo
        self.log_norm_cst = width.double().log() if isinstance(width, torch.Tensor) else np.log(width)

    def _params(self):
        return self.lo, self.hi


# ---------------------------------------------------------------------------------------------------------------------
# transforms, mixtures, conditional laws: host composition over the device laws
# ---------------------------------------------------------------------------------------------------------------------
def _mod(x):
    """torch for tensors, NumPy for everything else."""
    return torch if isinstance(x, torch.Tensor) else np


class TransformedDist(ProbDist):
    """Law of Y = f(X), X ~ base_dist -- particles/distributions.py:657-697.  ``f``, ``finv`` and ``logJac`` take
    CUDA tensors (state-space models) and NumPy arrays (a field of a StructDist's structured array) alike."""

    def __init__(self, base_dist):
        self.base_dist = base_dist

    def error_msg(self, method):
        return f'method {method} not defined in class {self.__class__}'

    def f(self, x):
        raise NotImplementedError(self.error_msg("f"))

    def finv(self, x):
        """Inverse of f."""
        raise NotImplementedError(self.error_msg("finv"))

    def logJac(self, x):
        """Log of the Jacobian of finv."""
        raise NotImplementedError(self.error_msg("logJac"))

    def rvs(self, size=None):
        return self.f(self.base_dist.rvs(size=size))

    def logpdf(self, x):
        lp = self.base_dist.logpdf(self.finv(x))
        if isinstance(x, torch.Tensor):
            lp = as_device(lp)
        else:
            lp = _host(lp)
        return lp + self.logJac(x)


class LinearD(TransformedDist):
    """Y = a X + b -- particles/distributions.py:700-724."""

    def __init__(self, base_dist, a=1.0, b=0.0):
        self.a, self.b = a, b
        self.base_dist = base_dist

    def f(self, x):
        return self.a * x + self.b

    def finv(self, x):
        return (x - self.b) / self.a

    def logJac(self, x):
        return -np.log(self.a)


class LogD(TransformedDist):
    """Y = log(X) -- particles/distributions.py:727-746."""

    def f(self, x):
        return _mod(x).log(x)

    def finv(self, x):
        return _mod(x).exp(x)

    def logJac(self, x):
        return x


class LogitD(TransformedDist):
    """Y = logit((X - a) / (b - a)) -- particles/distributions.py:749-775.  logJac's log(1 + exp(x)) is a softplus,
    max(x, 0) + log1p(exp(-|x|)), finite where the reference's overflows (x > ~709; DESIGN.md section 5.16)."""

    def __init__(self, base_dist, a=0.0, b=1.0):
        self.a, self.b = a, b
        self.base_dist = base_dist

    def f(self, x):
        p = (x - self.a) / (self.b - self.a)
        return _mod(x).log(p / (1.0 - p))

    def finv(self, x):
        return self.a + (self.b - self.a) / (1.0 + _mod(x).exp(-x))

    def logJac(self, x):
        m = _mod(x)
        softplus = m.maximum(x, 0.0 * x) + m.log1p(m.exp(-m.abs(x)))
        return np.log(self.b - self.a) + x - 2.0 * softplus


class Mixture(ProbDist):
    """Mixture of k laws -- particles/distributions.py:783-816; pk (k,) or (N, k).  logpdf: the components' device
    log-densities, then one row log-sum-exp kernel; rvs: a categorical index per element from the context's
    Philox stream, then the chosen component's draw."""

    def __init__(self, pk, *components):
        self.pk = pk if isinstance(pk, torch.Tensor) else np.atleast_1d(pk)
        self.k = self.pk.shape[-1]
        if len(components) != self.k:
            raise ValueError("Size of pk and nr of components should match")
        self.components = components

    def _pk(self):
        """pk on the device; a (1, k) pk is the (k,) one"""
        pk = as_device(self.pk)
        return pk.reshape(-1) if pk.ndim == 2 and pk.shape[0] == 1 else pk

    def _length(self, pk, cols):
        """common length of the (n,) columns and the rows of a 2-D pk; length 1 broadcasts, as in NumPy"""
        lens = {int(v.shape[0]) for v in cols} | ({int(pk.shape[0])} if pk.ndim == 2 else set())
        if len(lens - {1}) > 1:
            raise ValueError(f"Mixture: operands could not be broadcast together with lengths {sorted(lens)}")
        return max(lens)

    def logpdf(self, x):
        lps = [as_device(cd.logpdf(x)).reshape(-1) for cd in self.components]
        pk = self._pk()
        n = self._length(pk, lps)
        lp = torch.stack([v.expand(n) for v in lps]).contiguous()
        logpk = torch.log(pk).contiguous()
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_mixture_logpdf(ctx.handle, ptr(lp), ptr(logpk), self.k if pk.ndim == 2 else 0,
                                               self.k, ptr(out), n))
        return out

    def rvs(self, size=None):
        pk = self._pk()
        xk = [as_device(cd.rvs(size=size)).reshape(-1) for cd in self.components]
        n = self._length(pk, xk)
        u = Uniform().rvs(size=n)
        idx = (torch.cumsum(pk, -1) < u[:, None]).sum(-1).clamp_(max=self.k - 1)     # searchsorted(cumsum(pk), u)
        return torch.stack([v.expand(n) for v in xk]).gather(0, idx.reshape(1, -1)).reshape(-1)


class Cond(ProbDist):
    """Conditional law in a StructDist -- particles/distributions.py:1130-1146: ``law`` maps the structured array
    drawn so far to a law."""

    def __init__(self, law, dim=1, dtype="float64"):
        self.law = law
        self.dim = dim
        self.dtype = dtype

    def __call__(self, x):
        return self.law(x)


class Dirichlet(ProbDist):
    """Dirichlet(alphas), alphas (d,) -- particles/distributions.py:854-885.  logpdf of rows x (N, d) (or one (d,)
    point) on the device, with scipy.stats.dirichlet's ValueError for points off the simplex (its tests and
    tolerance, |sum - 1| <= 1e-9); rvs (size, d) from device Gamma draws normalised in log space."""

    def __init__(self, alphas=None):
        if alphas is None:
            raise ValueError('Dirichlet: missing parameter alphas')
        self.alphas = alphas

    @property
    def dim(self):
        return self.alphas.shape[0]

    def _alpha(self):
        a = _host(self.alphas)
        if a.ndim != 1 or np.any(~(a > 0)):
            raise ValueError("All parameters must be greater than 0")
        return a

    def logpdf(self, x):
        from scipy.special import gammaln
        a = self._alpha()
        d = a.shape[0]
        xd = as_device(x)
        xd = xd.reshape(1, -1) if xd.ndim == 1 else xd
        if xd.shape[-1] == d - 1:                          # scipy appends the last coordinate
            xd = torch.cat([xd, 1.0 - xd.sum(-1, keepdim=True)], dim=-1)
        if xd.ndim != 2 or xd.shape[-1] != d:
            raise ValueError(f"Vector 'x' must have either the same number of entries as, or one entry fewer than, "
                             f"parameter vector 'a', but alpha.shape = {a.shape} and x.shape = {tuple(xd.shape)}.")
        xd = xd.contiguous()
        n = xd.shape[0]
        ctx = context()
        out = empty(n)
        bad = torch.zeros(1, dtype=torch.int32, device=out.device)
        _lib.check(ctx.lib.smcb_dirichlet_logpdf(ctx.handle, ptr(xd), d, ptr(as_device(a)), d,
                                                 float(gammaln(a.sum()) - gammaln(a).sum()), ptr(out), ptr(bad), n))
        flags = int(bad.item())
        if flags & _lib.DIRICHLET_RANGE and not flags & _lib.DIRICHLET_NAN:
            raise ValueError("Each entry in 'x' must be greater than or equal to zero, and smaller or equal one.")
        if flags & _lib.DIRICHLET_ZERO:
            raise ValueError("Each entry in 'x' must be greater than zero if its alpha is less than one.")
        if flags & _lib.DIRICHLET_SUM:
            raise ValueError("The input vector 'x' must lie within the normal simplex.")
        return out

    def rvs(self, size=1):
        a = self._alpha()
        n = 1 if size is None else int(size)
        ctx = context()
        out = empty((n, a.shape[0]))
        _lib.check(ctx.lib.smcb_dirichlet_rvs(ctx.handle, ptr(as_device(a)), a.shape[0], ptr(out), n))
        return out


class VaryingCovNormal(MvNormal):
    """Multivariate normal with one covariance matrix per particle -- particles/distributions.py:1012-1059.
    ``cov`` (N, d, d), d <= 8; the constructor computes the N Cholesky factors on the device (``.L``, an (N, d, d)
    tensor) and raises ValueError when a cov[n] is not positive definite.  ``loc``: scalar, (d,) or (N, d)."""

    def __init__(self, loc=0.0, cov=None):
        self.loc = loc
        err_msg = "VaryingCovNormal: argument cov must be a (N, d, d) array, \
                with d>1; cov[n, :, :] must be symmetric and positive"
        if cov is None or len(np.shape(cov)) != 3 or np.shape(cov)[1] != np.shape(cov)[2]:
            raise ValueError(err_msg)
        self.cov = as_device(cov)
        self.N, d, _ = self.cov.shape
        if d > 8:
            raise NotImplementedError(f"VaryingCovNormal: d = {d}; the device kernels take d <= 8")
        ctx = context()
        self.L = empty((self.N, d, d))
        bad = torch.zeros(1, dtype=torch.int32, device=self.L.device)
        _lib.check(ctx.lib.smcb_vcn_chol(ctx.handle, ptr(self.cov), d, ptr(self.L), ptr(bad), self.N))
        if int(bad.item()):
            raise ValueError(err_msg)

    def _rows(self, v, what):
        """-> (device rows, row stride): a scalar, a (d,) vector or a (1, d) row is one row for every particle (stride
        0), an (N, d) array one row per particle; any other shape is NumPy's broadcast ValueError."""
        d = self.dim
        v = as_device(v)
        if v.ndim == 0 or (v.ndim == 1 and v.shape[0] == 1):
            return v.reshape(1).expand(d).contiguous(), 0
        if v.ndim == 1 and v.shape[0] == d:
            return v, 0
        if v.ndim == 2 and v.shape[1] == d and v.shape[0] in (1, self.N):
            return v.contiguous(), (0 if v.shape[0] == 1 else d)
        raise ValueError(f"VaryingCovNormal: {what} of shape {tuple(v.shape)} does not broadcast against the "
                         f"({self.N}, {d}) particles")

    def rvs(self, size=None):
        N = self.N if size is None else int(size)
        if N != self.N:
            raise ValueError(f"VaryingCovNormal.rvs: size {N} for {self.N} covariance matrices")
        loc, loc_ld = self._rows(self.loc, "loc")
        ctx = context()
        out = empty((N, self.dim))
        _lib.check(ctx.lib.smcb_vcn_rvs(ctx.handle, ptr(loc), loc_ld, ptr(self.L), self.dim, ptr(out), N))
        return out

    def logpdf(self, x):
        xr, x_ld = self._rows(x, "x")
        loc, loc_ld = self._rows(self.loc, "loc")
        ctx = context()
        out = empty(self.N)
        _lib.check(ctx.lib.smcb_vcn_logpdf(ctx.handle, ptr(xr), x_ld, ptr(loc), loc_ld, ptr(self.L), self.dim,
                                           ptr(out), self.N))
        return out

    def posterior(self, x, Sigma=None):
        raise NotImplementedError
