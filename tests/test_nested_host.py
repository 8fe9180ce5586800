"""Nested sampling SMC without a GPU: the oracle (tests/nested_oracle.py) against seeded runs of the LIVE reference
(tests/golden/golden_nested.npz, made by tests/golden/make_golden_nested.py), the host half of the device threshold
step (NumPy's percentile rule as order statistics plus ``_lerp``) against ``np.percentile``, and the constructor's
refusals."""
import os

import numpy as np
import pytest

import nested_oracle as nso
from oracle.samplers_numpy import LogisticModel
from particles_b200 import nested
from particles_b200 import smc_samplers as ssps


@pytest.fixture(scope="module")
def gn():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_nested.npz"))


@pytest.mark.parametrize("tag", ["wf", "std"])
def test_oracle_nested_reproduces_reference_run(gn, tag):
    """Same seed, same stream order -> same run, waste-free and standard move; theta / lpost at the tolerances of the
    IBIS and tempering tests (BLAS / LAPACK in the covariance, Cholesky and matmul leave last-bit differences)."""
    N, lc, seed, wf, alpha, eps, t = gn["exact/%s/meta" % tag]
    np.random.seed(int(seed))
    out = nso.run_nested(LogisticModel(gn["exact/data"]), int(N), wastefree=bool(wf), len_chain=int(lc),
                         ESSrmin=float(alpha), eps=float(eps))
    assert out["t"] == int(t) and out["t"] > 5
    assert out["lts"][-1] == np.inf and len(out["lts"]) == len(out["log_evid"]) == out["t"] + 1
    np.testing.assert_allclose(out["lts"], gn["exact/%s/lts" % tag], rtol=1e-12)
    np.testing.assert_allclose(out["log_evid"], gn["exact/%s/log_evid" % tag], rtol=1e-12)
    np.testing.assert_allclose(out["X"].theta, gn["exact/%s/theta" % tag], rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(out["X"].lpost, gn["exact/%s/lpost" % tag], rtol=1e-11)
    np.testing.assert_allclose(out["X"].llik, gn["exact/%s/llik" % tag], rtol=1e-11)


def test_golden_anchors_agree():
    """The reference's own NS-SMC and adaptive-tempering estimates of the same log-evidence agree within 3 sigma:
    the anchors the device runs are checked against are consistent with each other."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_nested.npz"))
    a, b = g["stat/ns_log_evid"], g["stat/tempering_logLt"]
    se = np.sqrt(a.var(ddof=1) / a.size + b.var(ddof=1) / b.size)
    assert abs(a.mean() - b.mean()) < 3.0 * se + 1e-3


def _cases():
    r = np.random.RandomState(5)
    for n in (1, 2, 3, 10, 1001, 100_003):
        yield "normal-%d" % n, r.standard_normal(n) * 40.0 - 200.0
        yield "ties-%d" % n, np.round(r.standard_normal(n) * 3.0)
        v = r.standard_normal(n)
        v[r.rand(n) < 0.3] = -np.inf
        yield "neginf-%d" % n, v
        yield "equal-%d" % n, np.full(n, -3.25)
        yield "allneginf-%d" % n, np.full(n, -np.inf)
        if n >= 3:
            v = r.standard_normal(n)
            v[: n // 2 + 1] = -np.inf
            yield "halfneginf-%d" % n, r.permutation(v)


CASES = list(_cases())
ALPHAS = (0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99)


@pytest.mark.parametrize("name,v", CASES, ids=[c[0] for c in CASES])
def test_percentile_rule_matches_numpy_bit_for_bit(name, v):
    """The host's (k0, k1, gamma) with _lerp over the sorted values gives the bits of np.percentile, NaN included
    (both statistics -inf), for every ESSrmin of the paper's sweep and its extremes."""
    s = np.sort(v)
    for alpha in ALPHAS:
        k0, k1, g = nested.percentile_rule(v.size, alpha)
        assert 0 <= k0 <= k1 <= min(k0 + 1, v.size - 1)
        got = nested.lerp(float(s[k0]), float(s[k1]), g)
        with np.errstate(invalid="ignore"):
            want = np.percentile(v, 100.0 * (1.0 - alpha))
        assert np.float64(got).tobytes() == np.float64(want).tobytes(), (name, alpha, got, want)


def test_percentile_rule_refuses_bad_essrmin():
    for alpha in (0.0, -0.1, 1.5):
        with pytest.raises(ValueError):
            nested.percentile_rule(10, alpha)


class _NoLik(ssps.StaticModel):
    pass


class _Prior:
    """A duck-typed prior of d scalar fields (no device needed: the constructor only reads the dtype)."""

    def __init__(self, d):
        self.dtype = [("x%d" % j, float) for j in range(d)]


class _WithLik(ssps.StaticModel):
    def logpyt(self, theta, t):
        return 0.0 * theta["x0"]


def test_constructor_refusals():
    with pytest.raises(NotImplementedError, match="neither a device likelihood nor a logpyt"):
        nested.NestedSamplingSMC(model=_NoLik(data=None, prior=_Prior(2)))
    with pytest.raises(NotImplementedError, match="neither"):
        nested.NestedSamplingSMC(model=None)
    with pytest.raises(NotImplementedError, match="d <= 20"):
        nested.NestedSamplingSMC(model=_WithLik(data=None, prior=_Prior(21)))
    fk = nested.NestedSamplingSMC(model=_WithLik(data=None, prior=_Prior(20)), len_chain=5, ESSrmin=0.3, eps=0.02)
    assert (fk.ESSrmin, fk.eps, fk.len_chain, fk.wastefree) == (0.3, 0.02, 5, True)
    assert fk.move.nsteps == 4
    fk = nested.NestedSamplingSMC(model=_WithLik(data=None, prior=_Prior(3)), wastefree=False)
    assert (fk.ESSrmin, fk.eps, fk.len_chain) == (0.1, 0.01, 10)
    assert isinstance(fk.move, ssps.AdaptiveMCMCSequence)
