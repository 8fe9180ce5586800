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


def _split(v):
    """scalar-or-array argument -> (device tensor or None, scalar).  A size-1 array or tensor is a scalar that
    broadcasts -- ``StateSpaceModel.simulate`` returns observations of shape (1,), and NumPy broadcasts
    ``data[t]`` against the (N,) particles (SURVEY.md section 9.10)."""
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


class Normal(LocScaleDist):
    """N(loc, scale^2) -- particles/distributions.py:267-285."""

    def _n(self, size, *arrs):
        """Common length of the array arguments (scalars broadcast); mismatched lengths are an error, as NumPy's
        broadcasting would make them."""
        lens = {int(a.shape[0]) for a in arrs if a is not None}
        if len(lens) > 1:
            raise ValueError(f"operands could not be broadcast together with lengths {sorted(lens)}")
        if lens:
            return lens.pop()
        return 1 if size is None else int(size)

    def rvs(self, size=None, z=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        zd = None if z is None else as_device(z)
        n = self._n(size, la, sa, zd)
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_normal_rvs(ctx.handle, ptr(la), l0, ptr(sa), s0, ptr(zd), ptr(out), n))
        return out

    def logpdf(self, x):
        xa, x0 = _split(x)
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = self._n(None, xa, la, sa)
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_normal_logpdf(ctx.handle, ptr(xa), x0, ptr(la), l0, ptr(sa), s0,
                                              ptr(out), n))
        return out


class _Univariate(ProbDist):
    """logpdf through the elementwise kernel smcb_logpdf1 (kinds: 0 Student, 1 Gamma, 2 Laplace, 3 Logistic)."""
    _kind = None

    def _call(self, x, p0, c0, a, b):
        xa, x0 = _split(x)
        aa, a0 = _split(a)
        ba, b0 = _split(b)
        lens = {int(v.shape[0]) for v in (xa, aa, ba) if v is not None}
        if len(lens) > 1:
            raise ValueError(f"operands could not be broadcast together with lengths {sorted(lens)}")
        n = lens.pop() if lens else 1
        ctx = context()
        out = empty(n)
        _lib.check(ctx.lib.smcb_logpdf1(ctx.handle, self._kind, ptr(xa), x0, float(p0), float(c0), ptr(aa), a0,
                                        ptr(ba), b0, ptr(out), n))
        return out


class Student(_Univariate):
    """Student(df, loc, scale) -- particles/distributions.py:417-433 (scipy.stats.t.logpdf); ``df`` scalar."""
    _kind = 0

    def __init__(self, df=3.0, loc=0.0, scale=1.0):
        self.df, self.loc, self.scale = df, loc, scale

    def logpdf(self, x):
        from scipy.special import gammaln
        df = float(self.df)
        c0 = gammaln(0.5 * (df + 1.0)) - gammaln(0.5 * df) - 0.5 * np.log(df * np.pi)
        return self._call(x, df, c0, self.loc, self.scale)

    def rvs(self, size=None):
        """loc + scale * z / sqrt(chi2_df / df): the normals from the context's Philox stream, the chi-square
        from torch's generator (the reference draws through scipy.stats.t.rvs)."""
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = la.shape[0] if la is not None else (sa.shape[0] if sa is not None else (1 if size is None else int(size)))
        z = Normal().rvs(size=n)
        g = torch.distributions.Chi2(torch.tensor(float(self.df), dtype=torch.float64, device=z.device)).sample((n,))
        t = z / torch.sqrt(g / float(self.df))
        return (la if la is not None else l0) + (sa if sa is not None else s0) * t


class Gamma(_Univariate):
    """Gamma(a, b), density prop. to x^(a-1) exp(-b x) -- particles/distributions.py:336-356; ``a`` scalar,
    ``b`` scalar or per-particle array."""
    _kind = 1

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = a, b
        self.scale = 1.0 / b

    def logpdf(self, x):
        from scipy.special import gammaln
        return self._call(x, float(self.a), -gammaln(float(self.a)), self.b, 1.0)

    def rvs(self, size=None):
        b = as_device(self.b) if isinstance(self.b, (torch.Tensor, np.ndarray)) else \
            torch.full((1 if size is None else int(size),), float(self.b), dtype=torch.float64, device="cuda")
        a = torch.full_like(b, float(self.a))
        return torch.distributions.Gamma(a, b).sample()


class Laplace(LocScaleDist, _Univariate):
    """particles/distributions.py:301-314."""
    _kind = 2

    def logpdf(self, x):
        return self._call(x, 0.0, 0.0, self.loc, self.scale)

    def rvs(self, size=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = la.shape[0] if la is not None else (sa.shape[0] if sa is not None else (1 if size is None else int(size)))
        u = torch.rand(n, dtype=torch.float64, device="cuda") - 0.5
        return (la if la is not None else l0) - (sa if sa is not None else s0) * torch.sign(u) * torch.log1p(-2 * u.abs())


class Logistic(LocScaleDist, _Univariate):
    """particles/distributions.py:288-299."""
    _kind = 3

    def logpdf(self, x):
        return self._call(x, 0.0, 0.0, self.loc, self.scale)

    def rvs(self, size=None):
        la, l0 = _split(self.loc)
        sa, s0 = _split(self.scale)
        n = la.shape[0] if la is not None else (sa.shape[0] if sa is not None else (1 if size is None else int(size)))
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


class Categorical(ProbDist):
    """Categorical(p), p (k,) or (N, k) -- particles/distributions.py:598-628."""
    dtype = np.int64

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


class Poisson(ProbDist):
    """Poisson(rate) -- particles/distributions.py:519-532 (logpdf on the device; ``rate`` a CUDA
    tensor or scalar, ``x`` the observed count).  scipy evaluates xlogy(k, mu) - gammaln(k+1) - mu."""
    dtype = np.int64

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
