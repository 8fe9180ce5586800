"""SMC samplers on binary spaces, the parts that need no device: the NumPy oracle against the live reference's
golden vectors (tests/golden/golden_binary.npz), the host-side NestedLogistic.fit against the reference's
coefficients, and the refusals of the public surface."""
import os

import numpy as np
import pytest

import binary_oracle as bo
from particles_b200 import binary_smc as bs, distributions as dists

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "golden_binary.npz"))
DESIGNS = {"p10": bo.small_design, "p104": bo.boston_like}


@pytest.mark.parametrize("tag", ["p10", "p104"])
@pytest.mark.parametrize("kind", ["bic", "bvs", "gprior"])
def test_oracle_models_match_reference(tag, kind):
    X, y = DESIGNS[tag]()
    np.testing.assert_array_equal(G[tag + "/Xy_sums"], [X.sum(), y.sum()])
    m = bo.VS(kind, X, y)
    g = G[tag + "/gamma"]
    len_gam, ldet, wtw = m.chol(g)
    np.testing.assert_array_equal(len_gam, G["%s/%s/len_gam" % (tag, kind)])
    np.testing.assert_array_equal(ldet, G["%s/%s/ldet" % (tag, kind)])
    np.testing.assert_array_equal(wtw, G["%s/%s/wtw" % (tag, kind)])
    np.testing.assert_array_equal(m.loglik(g), G["%s/%s/loglik" % (tag, kind)])
    c = G["%s/%s/consts" % (tag, kind)]
    np.testing.assert_allclose(np.hstack([m.iv2, m.coef_len, m.coef_log, m.coef_in_log]), c, rtol=1e-13, atol=0)


@pytest.mark.parametrize("tag", ["p10", "p104"])
def test_oracle_and_package_fit_match_reference(tag):
    W, x = G[tag + "/fit/W"], G[tag + "/fit/x"]
    for nl in (bo.NestedLogistic.fit(W, x), bs.NestedLogistic.fit(W, x)):
        np.testing.assert_array_equal(nl.edgy, G[tag + "/fit/edgy"])
        np.testing.assert_allclose(nl.coeffs, G[tag + "/fit/coeffs"], rtol=1e-10, atol=1e-10)
    nl = bo.NestedLogistic(G[tag + "/fit/coeffs"], G[tag + "/fit/edgy"])
    seed, size = G[tag + "/rvs/seed"]
    np.random.seed(seed)
    draws, us = nl.rvs(size)
    np.testing.assert_array_equal(draws, G[tag + "/rvs/x"])
    assert us.shape == (x.shape[1], size)
    np.testing.assert_array_equal(nl.logpdf(draws), G[tag + "/rvs/logpdf"])
    np.testing.assert_array_equal(nl.rvs(size, us)[0], draws)          # injected uniforms replay the draw


def test_oracle_tempering_run_matches_reference():
    X, y = bo.small_design()
    model = bo.VS("bvs", X, y, prior=bo.IIDBernoulli(0.5, X.shape[1]))
    N, P, seed = G["run/meta"]
    np.random.seed(seed)
    out = bo.run_binary_tempering(model, N, P)
    np.testing.assert_array_equal(out["exponents"], G["run/exponents"])
    np.testing.assert_allclose(out["logLt"], G["run/logLt"], rtol=1e-13)


def test_surface_refusals():
    r = np.random.RandomState(0)
    X, y = r.standard_normal((200, 129)), r.standard_normal(200)
    with pytest.raises(NotImplementedError, match="p <= 128"):
        bs.BIC(data=(X, y))
    with pytest.raises(NotImplementedError, match="p <= 128"):
        bs.NestedLogistic(np.zeros((129, 129)), np.zeros(129, dtype=bool))
    with pytest.raises(NotImplementedError, match="IID"):
        bs._bernoulli_q(dists.IID(dists.Normal(), 10), 10)
    with pytest.raises(NotImplementedError, match="IID"):
        bs._bernoulli_q(dists.IID(bs.Bernoulli(0.5), 9), 10)
    assert bs._bernoulli_q(dists.IID(bs.Bernoulli(0.3), 10), 10) == 0.3


def test_all_binary_words():
    w = bs.all_binary_words(4)
    assert w.shape == (16, 4) and len({tuple(r) for r in w}) == 16
    np.testing.assert_array_equal(w[5], [True, False, True, False])
