"""IBIS (data tempering) without a GPU: the oracle (tests/ibis_oracle.py) against seeded runs of the LIVE
reference (tests/golden/golden_ibis.npz, made by tests/golden/make_golden_ibis.py), and the vector fields of
``distributions.StructDist``."""
import os

import numpy as np
import pytest
from scipy import stats

from oracle import samplers_numpy as sp
import ibis_oracle as ibo


@pytest.fixture(scope="module")
def gi():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_ibis.npz"))


@pytest.mark.parametrize("tag", ["wf", "std"])
def test_oracle_ibis_reproduces_reference_run(gi, tag):
    """Same seed, same stream order -> same run, waste-free and standard move (the tolerances of the tempering
    test: BLAS / LAPACK in the covariance, Cholesky and matmul leave last-bit differences)."""
    N, lc, seed, wf = (int(v) for v in gi["exact/%s/meta" % tag])
    np.random.seed(seed)
    out = ibo.run_ibis(ibo.LogisticIBISModel(gi["exact/data"]), N, wastefree=bool(wf), len_chain=lc, ESSrmin=0.5)
    assert out["rs_flags"] == [bool(v) for v in gi["exact/%s/rs_flags" % tag]]
    assert sum(out["rs_flags"]) > 5
    np.testing.assert_allclose(out["logLts"], gi["exact/%s/logLts" % tag], rtol=1e-12)
    np.testing.assert_allclose(out["ESSs"], gi["exact/%s/ESSs" % tag], rtol=1e-10)
    np.testing.assert_allclose(out["X"].theta, gi["exact/%s/theta" % tag], rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(out["X"].lpost, gi["exact/%s/lpost" % tag], rtol=1e-11)
    assert out["X"].N == N * (lc if wf else 1)


class _HostLaw:
    """A law with host draws (no device needed): the StructDist field logic only."""

    def __init__(self, dim, scale):
        self.dim, self.scale = dim, scale

    def rvs(self, size=None):
        z = np.random.standard_normal((size, self.dim) if self.dim > 1 else size)
        return self.scale * z

    def logpdf(self, x):
        return stats.norm.logpdf(x, scale=self.scale).reshape(len(x), -1).sum(axis=1)


def test_structdist_vector_field():
    """A law with dim > 1 gets a (name, float, (dim,)) field: dtype, rvs shapes and logpdf against SciPy."""
    from particles_b200.distributions import StructDist
    prior = StructDist({"beta": _HostLaw(3, 10.0), "sigma": _HostLaw(1, 2.0)})
    assert prior.dtype == [("beta", float, (3,)), ("sigma", float)]
    np.random.seed(0)
    th = prior.rvs(size=7)
    assert th.shape == (7,) and th["beta"].shape == (7, 3) and th["sigma"].shape == (7,)
    assert np.all(np.isfinite(th["beta"])) and np.unique(th["beta"]).size == 21
    want = (stats.multivariate_normal.logpdf(th["beta"], cov=100.0 * np.eye(3))
            + stats.norm.logpdf(th["sigma"], scale=2.0))
    np.testing.assert_allclose(prior.logpdf(th), want, rtol=1e-13)
    one = prior.rvs(size=1)
    assert one["beta"].shape == (1, 3)


def test_structdist_scalar_fields_unchanged():
    """Scalar-only priors keep their (name, float) fields, sorted names and (N,) draws."""
    from particles_b200.distributions import StructDist
    prior = StructDist({"rho": _HostLaw(1, 1.0), "a": _HostLaw(1, 3.0)})
    assert prior.dtype == [("a", float), ("rho", float)]
    np.random.seed(1)
    th = prior.rvs(size=5)
    assert th.dtype == np.dtype([("a", float), ("rho", float)]) and th.shape == (5,)
    np.random.seed(1)
    a = 3.0 * np.random.standard_normal(5)
    rho = np.random.standard_normal(5)
    assert np.array_equal(th["a"], a) and np.array_equal(th["rho"], rho)
    np.testing.assert_allclose(prior.logpdf(th), stats.norm.logpdf(a, scale=3.0) + stats.norm.logpdf(rho), rtol=1e-13)


def test_ibis_layout_of_prior_fields():
    """The (N, p) theta columns of each prior field, in the prior's field order."""
    from particles_b200.distributions import StructDist
    from particles_b200.smc_samplers import StaticModel, _layout
    prior = StructDist({"beta": _HostLaw(3, 1.0), "sigma": _HostLaw(1, 1.0), "z": _HostLaw(2, 1.0)})
    assert _layout(prior) == [("beta", slice(0, 3)), ("sigma", 3), ("z", slice(4, 6))]
    assert StaticModel(prior=prior).dim == 6


def test_ibis_refuses_models_it_cannot_run():
    """No device likelihood and no logpyt, or more than 20 parameters: NotImplementedError with a clear message."""
    from particles_b200.distributions import StructDist
    from particles_b200.smc_samplers import IBIS, StaticModel

    class Wide(StaticModel):
        def logpyt(self, theta, t):
            return 0.0

    with pytest.raises(NotImplementedError, match="logpyt"):
        IBIS(model=StaticModel(prior=StructDist({"b": _HostLaw(2, 1.0)})))
    with pytest.raises(NotImplementedError, match="d <= 20"):
        IBIS(model=Wide(prior=StructDist({"b": _HostLaw(21, 1.0)})))
    IBIS(model=Wide(prior=StructDist({"b": _HostLaw(20, 1.0)})))
