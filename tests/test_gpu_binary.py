"""SMC samplers on binary spaces on the device (particles_b200.binary_smc): the batched Cholesky and the three
models' log-likelihoods against the live reference's golden vectors and the NumPy oracle, the nested-logistic
proposal against the reference's draws, the fused waste-free move against the oracle's step-by-step chain, exact
answers at p = 10 by complete enumeration, and a Boston-shaped p = 104 run at N = 10^5."""
import os

import numpy as np
import pytest
import torch

import binary_oracle as bo
import particles_b200 as pb
from particles_b200 import binary_smc as bs, distributions as dists, smc_samplers as ssp
from particles_b200.smc_samplers import ThetaParticles

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "golden_binary.npz"))
DESIGNS = {"p10": bo.small_design, "p104": bo.boston_like}
KINDS = {"bic": bs.BIC, "bvs": bs.BayesianVS, "gprior": bs.BayesianVS_gprior}


def make(kind, X, y, q=0.5):
    prior = dists.IID(bs.Bernoulli(q), X.shape[1])
    m = bs.BIC(data=(X, y)) if kind == "bic" else KINDS[kind](data=(X, y), prior=prior)
    m.prior = prior
    return m


def host(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("tag", ["p10", "p104"])
@pytest.mark.parametrize("kind", ["bic", "bvs", "gprior"])
def test_vs_loglik_against_golden(tag, kind):
    X, y = DESIGNS[tag]()
    m = make(kind, X, y)
    g = G[tag + "/gamma"]
    np.testing.assert_allclose(np.hstack([m.iv2, m.coef_len, m.coef_log, m.coef_in_log]),
                               G["%s/%s/consts" % (tag, kind)], rtol=1e-11)
    len_gam, ldet, wtw = m.chol_intermediate(g)
    np.testing.assert_array_equal(host(len_gam), G["%s/%s/len_gam" % (tag, kind)])
    np.testing.assert_allclose(host(ldet), G["%s/%s/ldet" % (tag, kind)], rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(host(wtw), G["%s/%s/wtw" % (tag, kind)], rtol=1e-11, atol=0)
    np.testing.assert_allclose(host(m.loglik(g)), G["%s/%s/loglik" % (tag, kind)], rtol=1e-11, atol=0)
    ref = bo.IIDBernoulli(0.5, X.shape[1]).logpdf(g)
    x = ThetaParticles(theta=torch.as_tensor(g).cuda())
    m.target(x, 0.3)
    np.testing.assert_array_equal(host(x.lprior), ref)
    np.testing.assert_array_equal(host(x.lpost), host(x.lprior) + 0.3 * host(x.llik))


def test_vs_loglik_large_batch_against_oracle():
    X, y = bo.boston_like()
    m = make("bvs", X, y)
    o = bo.VS("bvs", X, y)
    r = np.random.RandomState(3)
    g = r.rand(100_000, X.shape[1]) < r.uniform(0.02, 0.3, (100_000, 1))
    ll = host(m.loglik(g))
    idx = r.choice(100_000, 400, replace=False)
    np.testing.assert_allclose(ll[idx], o.loglik(g[idx]), rtol=1e-11)
    assert np.all(np.isfinite(ll))


def test_not_positive_definite_raises():
    X, y = bo.small_design()
    g = np.zeros((3, X.shape[1]), dtype=bool)
    g[1, 2:6] = True
    vm2 = -1e4                                        # X^T X[gamma, gamma] + vm2 I is indefinite
    with pytest.raises(np.linalg.LinAlgError):
        bo.chol_and_friends(g, X.T @ X, X.T @ y, vm2)
    with pytest.raises(np.linalg.LinAlgError):
        bs.chol_and_friends(g, X.T @ X, X.T @ y, vm2)
    len_gam, ldet, wtw = bs.chol_and_friends(g[[0, 2]], X.T @ X, X.T @ y, vm2)   # empty gammas: (0, 0, 0)
    assert not host(len_gam).any() and not host(ldet).any() and not host(wtw).any()


@pytest.mark.parametrize("tag", ["p10", "p104"])
def test_nested_logistic_against_reference(tag):
    coeffs, edgy = G[tag + "/fit/coeffs"], G[tag + "/fit/edgy"]
    nl = bs.NestedLogistic(coeffs, edgy)
    seed, size = G[tag + "/rvs/seed"]
    np.random.seed(seed)
    _, us = bo.NestedLogistic(coeffs, edgy).rvs(size)
    x, lp = nl.rvs_and_logpdf(size=int(size), u=us)
    np.testing.assert_array_equal(host(x), G[tag + "/rvs/x"])
    np.testing.assert_allclose(host(lp), G[tag + "/rvs/logpdf"], rtol=1e-12)
    np.testing.assert_allclose(host(nl.logpdf(x)), G[tag + "/rvs/logpdf"], rtol=1e-12)
    p5 = nl.predict_prob(x, 5)
    np.testing.assert_allclose(np.broadcast_to(host(torch.as_tensor(p5)), (size,)),
                               np.broadcast_to(bo.NestedLogistic(coeffs, edgy).predict_prob(G[tag + "/rvs/x"], 5),
                                               (size,)), rtol=1e-13)


def _move_case(tag, kind, M, P, epn, seed):
    X, y = DESIGNS[tag]()
    p = X.shape[1]
    m, o = make(kind, X, y), bo.VS(kind, X, y, prior=bo.IIDBernoulli(0.5, p))
    tag2 = tag
    prop = bo.NestedLogistic(G[tag2 + "/fit/coeffs"], G[tag2 + "/fit/edgy"])
    np.random.seed(seed)
    x0 = bo.ThetaParticles(theta=prop.rvs(M)[0])
    bo.target(o, epn)(x0)
    xo, pbo, noise = bo.wf_move(x0, bo.target(o, epn), prop, P)
    xd = ThetaParticles(theta=torch.as_tensor(x0.theta).cuda())
    m.target(xd, epn)
    xd.shared["proposal"] = bs.NestedLogistic(prop.coeffs, prop.edgy)
    return m, xd, xo, pbo, noise


@pytest.mark.parametrize("tag,kind", [("p10", "bvs"), ("p10", "bic"), ("p104", "bvs"), ("p104", "gprior")])
def test_fused_move_against_oracle(tag, kind):
    M, P, epn = 64, 12, 0.4
    m, xd, xo, pbo, noise = _move_case(tag, kind, M, P, epn, 7)
    out = m.wf_move(xd, epn, P, noise=noise)
    np.testing.assert_array_equal(host(out.theta), xo.theta)
    np.testing.assert_allclose(host(out.llik), xo.llik, rtol=1e-11)
    np.testing.assert_allclose(host(out.lpost), xo.lpost, rtol=1e-11)
    np.testing.assert_array_equal(host(out.lprior), xo.lprior)
    np.testing.assert_allclose(host(out.shared["acc_rates"][-1]), pbo.mean(axis=1), rtol=1e-9, atol=1e-12)


def test_fused_move_seeded_determinism():
    M, P, epn = 256, 20, 0.5
    m, xd, _, _, _ = _move_case("p104", "bvs", M, P, epn, 8)
    runs = []
    for s in (5, 5, 6):
        pb.seed(s)
        runs.append(m.wf_move(xd, epn, P))
    for f in ("theta", "lprior", "llik", "lpost"):
        assert torch.equal(getattr(runs[0], f), getattr(runs[1], f)), f
    assert not torch.equal(runs[0].theta, runs[2].theta)
    acc = host(runs[0].shared["acc_rates"][-1])
    assert np.all((acc > 0) & (acc <= 1))


def _exact(model):
    gam, lp = model.complete_enum()
    lp = host(lp)
    mx = lp.max()
    w = np.exp(lp - mx)
    return mx + np.log(w.sum()), (w[:, None] * gam).sum(axis=0) / w.sum()


@pytest.mark.parametrize("kind", ["bvs", "gprior", "bic"])
def test_exact_answer_p10_waste_free(kind):
    X, y = bo.small_design()
    model = make(kind, X, y)
    logZ, incl = _exact(model)
    lz, mp = [], []
    for r in range(12):
        pb.seed(1000 + r)
        move = ssp.MCMCSequenceWF(mcmc=bs.BinaryMetropolis(), len_chain=40)
        pf = pb.SMC(fk=ssp.AdaptiveTempering(model, len_chain=40, move=move), N=100)
        pf.run()
        assert pf.X.shared["exponents"][-1] == 1.0
        lz.append(pf.logLt)
        W = host(pf.W)
        mp.append((W[:, None] * host(pf.X.theta)).sum(axis=0))
    lz, mp = np.array(lz), np.array(mp)
    se = lz.std(ddof=1) / np.sqrt(len(lz))
    assert abs(lz.mean() - logZ) < 4 * se + 1e-3, (lz.mean(), logZ, se)
    se_p = mp.std(axis=0, ddof=1) / np.sqrt(len(mp))
    assert np.all(np.abs(mp.mean(axis=0) - incl) < 4 * se_p + 2e-3), (mp.mean(axis=0), incl, se_p)


def test_exact_answer_p10_standard_move():
    X, y = bo.small_design()
    model = make("bvs", X, y)
    logZ, incl = _exact(model)
    lz = []
    for r in range(8):
        pb.seed(2000 + r)
        move = ssp.AdaptiveMCMCSequence(mcmc=bs.BinaryMetropolis(), len_chain=6)
        pf = pb.SMC(fk=ssp.AdaptiveTempering(model, wastefree=False, move=move), N=2000)
        pf.run()
        lz.append(pf.logLt)
    lz = np.array(lz)
    se = lz.std(ddof=1) / np.sqrt(len(lz))
    assert abs(lz.mean() - logZ) < 4 * se + 1e-3, (lz.mean(), logZ, se)


def test_resampling_gathers_bool_theta():
    th = torch.as_tensor(np.random.RandomState(0).rand(50, 7) < 0.5).cuda()
    x = ThetaParticles(theta=th, lpost=torch.arange(50, dtype=torch.float64, device="cuda"))
    A = torch.as_tensor([3, 3, 0, 49], dtype=torch.int64, device="cuda")
    xa = x[A]
    assert xa.theta.dtype == torch.bool and torch.equal(xa.theta, th[A])
    assert torch.equal(xa.lpost, x.lpost[A])


def test_boston_shaped_end_to_end():
    X, y = bo.boston_like()
    model = make("bvs", X, y)
    P = 1000
    pb.seed(3)
    move = ssp.MCMCSequenceWF(mcmc=bs.BinaryMetropolis(), len_chain=P)
    pf = pb.SMC(fk=ssp.AdaptiveTempering(model, len_chain=P, move=move), N=100)
    pf.run()
    assert pf.X.shared["exponents"][-1] == 1.0
    assert pf.X.theta.shape == (100 * P, 104)
    assert np.isfinite(pf.logLt)
    for ar in pf.X.shared["acc_rates"]:
        a = host(ar)
        assert np.all(np.isfinite(a)) and np.all((a > 0) & (a <= 1))
