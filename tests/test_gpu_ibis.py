"""IBIS on the device: the reweighting kernel (smcb_logistic_logpyt) and the prefix targets against the NumPy
oracle, ``SMC.run()``'s stretches of reweighting steps against the per-step iterator (bit for bit), the generic
``StaticModel`` path against the closed-form linear-regression posterior, and the fused logistic IBIS against the
live reference's runs (tests/golden/golden_ibis.npz)."""
import os

import numpy as np
import pytest
from scipy import stats

from oracle import samplers_numpy as sp
import ibis_oracle as ibo
from oracle import smc_numpy as orc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def host(t):
    return t.detach().cpu().numpy()


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def rowwise(theta, data, r0, K, lw):
    """Cumulative log-weights lw + sum_{r <= k} logpyt_r, one row at a time (the oracle's logpyt)."""
    m = ibo.LogisticIBISModel(data)
    out, w = [], lw.copy()
    for k in range(K):
        w = w + m.logpyt(theta, r0 + k)
        w[np.isnan(w)] = -np.inf
        out.append(w)
    return np.array(out)


@pytest.mark.parametrize("n", [1, 2, 1001, 100_003])
@pytest.mark.parametrize("d", [1, 4, 9, 20, 32])
def test_logpyt_scan_and_commit_vs_oracle(d, n):
    """Scan rows and commits against the oracle's row-by-row logpyt for K in {1, 7, 64} at r0 = 37 (not a multiple of
    the 32-row tile), with saturated logits; a commit through row k has the bits of scan row k; a one-row logpyt has
    the bits of a one-row target; every scan row normalises to the bits of the committed log-weights."""
    import torch
    from particles_b200 import smc_samplers as ssp
    from particles_b200.device import context, ptr
    r = np.random.RandomState(d * 7 + n % 97)
    r0, data = 37, sp.synthetic_logistic(37 + 64 + 5, d, seed=d)
    theta = r.randn(n, d) * 2.0
    theta[0] *= 40.0                                     # saturated logits
    lw = r.randn(n) * 3.0
    model = ssp.LogisticRegression(data=data)
    th = dev(theta)
    ctx = context()
    for K in (1, 7, 64):
        want = rowwise(theta, data, r0, K, lw)
        scratch = torch.empty((K, n), dtype=torch.float64, device="cuda")
        lwd = dev(lw)
        model.logpyt_rows(th, r0, K, lwd, scratch=scratch)
        assert np.array_equal(host(lwd), lw)             # a scan writes nothing else
        got = host(scratch)
        np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-11)
        lp0, ll0 = r.randn(n), r.randn(n)
        lpost, llik = dev(lp0), dev(ll0)
        model.logpyt_rows(th, r0, K, lwd, lpost, llik)
        assert np.array_equal(host(lwd), got[-1])        # commit through row K-1 == scan row K-1, bit for bit
        inc = want[-1] - lw
        np.testing.assert_allclose(host(lpost), lp0 + inc, rtol=1e-13, atol=1e-10)
        np.testing.assert_allclose(host(llik), ll0 + inc, rtol=1e-13, atol=1e-10)
        if n <= 1001:
            for k in range(K):                            # each scan row normalises like the committed lw
                lwk = dev(lw)
                model.logpyt_rows(th, r0, k + 1, lwk)
                s1, s2 = torch.empty(4, dtype=torch.float64, device="cuda"), torch.empty(4, dtype=torch.float64,
                                                                                          device="cuda")
                row = scratch[k].clone()
                ctx.lib.smcb_normalise(ctx.handle, ptr(row), n, None, ptr(s1))
                ctx.lib.smcb_normalise(ctx.handle, ptr(lwk), n, None, ptr(s2))
                assert np.array_equal(host(s1), host(s2)), (K, k)
    one = ssp.ThetaParticles(theta=th)
    single = ssp.LogisticRegression(data=data[r0:r0 + 1])
    single.target(one, 1.0)
    assert np.array_equal(host(model.logpyt(th, r0)), host(one.llik))      # same bits as a one-row target


def test_logpyt_rejects_rows_outside_the_data():
    from particles_b200 import smc_samplers as ssp
    model = ssp.LogisticRegression(data=sp.synthetic_logistic(10, 3, seed=1))
    th = dev(np.zeros((4, 3)))
    with pytest.raises(ValueError):
        model.logpyt_rows(th, 8, 3, dev(np.zeros(4)), scratch=dev(np.zeros((3, 4))))


def _oracle_ibis_target(m, t):
    return lambda theta: m.prior.logpdf(theta) + ibo.IBISSampler(m).loglik(theta, t)


def test_prefix_target_and_wf_move_vs_oracle():
    """target(x, 1, n_rows) and wf_move(x, 1, P, noise, n_rows) against the oracle's IBIS target at n_rows in
    {0, 1, t, T}: n_rows = 0 is the prior alone."""
    import torch
    from particles_b200 import smc_samplers as ssp
    d, M, P, T = 5, 700, 9, 180
    data = sp.synthetic_logistic(T, d, seed=5)
    r = np.random.RandomState(7)
    theta = r.randn(M, d)
    W = orc.exp_and_normalise(r.randn(M))
    z, u = r.standard_normal((P - 1, M, d)), r.rand(P - 1, M)
    m = ibo.LogisticIBISModel(data)
    mdev = ssp.LogisticRegression(data=data)
    for n_rows in (0, 1, 77, T):
        tgt = _oracle_ibis_target(m, n_rows - 1)
        xd = ssp.ThetaParticles(theta=dev(theta))
        mdev.target(xd, 1.0, n_rows=n_rows)
        np.testing.assert_allclose(host(xd.lpost), tgt(theta), rtol=1e-13, atol=1e-10)
        np.testing.assert_allclose(host(xd.lprior), m.prior.logpdf(theta), rtol=1e-13)
        if n_rows == 0:
            assert np.all(host(xd.llik) == 0.0) and np.array_equal(host(xd.lpost), host(xd.lprior))
        # the waste-free move with injected noise against MCMCSequenceWF over the oracle's target
        fk = sp.AdaptiveTemperingWF(m, len_chain=P)
        xo = sp.ThetaParticles(theta=theta.copy(), lpost=tgt(theta))
        fk.calibrate(W, xo)
        xs, x = [xo], xo
        for s in range(P - 1):
            x = x.copy()
            prop = x.theta + z[s] @ x.shared["chol_cov"].T
            lpp = tgt(prop)
            acc = u[s] < np.exp(np.clip(lpp - x.lpost, None, 0.0))
            x.theta[acc], x.lpost[acc] = prop[acc], lpp[acc]
            xs.append(x)
        ref = sp.ThetaParticles.concatenate(*xs)
        ssp.ArrayRandomWalk().calibrate(dev(W), xd)
        out = mdev.wf_move(xd, 1.0, P, noise=(z, u), n_rows=n_rows)
        lp = host(out.lpost).reshape(P, M)
        same = np.all(np.isclose(lp, ref.lpost.reshape(P, M), rtol=1e-9), axis=0)
        assert same.mean() > 0.99
        th = host(out.theta).reshape(P, M, d)
        np.testing.assert_allclose(th[:, same], ref.theta.reshape(P, M, d)[:, same], rtol=1e-9, atol=1e-12)
        if n_rows == 0:
            assert np.all(host(out.llik) == 0.0)


def _ibis_pf(data, wastefree, lc, N, ESSrmin, seed):
    import particles_b200 as pb
    from particles_b200 import smc_samplers as ssp
    fk = ssp.IBIS(model=ssp.LogisticRegression(data=data), wastefree=wastefree, len_chain=lc)
    return pb.SMC(fk=fk, N=N, ESSrmin=ESSrmin, seed=seed)


@pytest.mark.parametrize("wastefree,ESSrmin,K0,T", [
    (True, 0.5, 8, 150), (False, 0.5, 8, 150), (True, 1.0, 8, 60), (False, 1.0, 8, 60),
    (True, 0.5, 7, 131), (True, 0.05, 1024, 40), (False, 0.05, 1024, 40)])
def test_run_stretches_match_the_iterator(monkeypatch, wastefree, ESSrmin, K0, T):
    """``run()`` (stretches of reweighting steps, one host read each) against ``for _ in pf: pass`` with the same
    seed: identical summaries, rs_flags, theta, lpost and logLt.  ESSrmin = 1 leaves every stretch empty; K0 = 7
    makes the stretches end off the tiles; ESSrmin = 0.05 with K0 = 1024 runs a stretch into the last row."""
    import torch
    from particles_b200 import core
    from particles_b200.device import context
    monkeypatch.setattr(core, "IBIS_K0", K0)
    data = sp.synthetic_logistic(T, 4, seed=11)
    lc = 8 if wastefree else 4
    a = _ibis_pf(data, wastefree, lc, 100, ESSrmin, seed=5)
    for _ in a:
        pass
    b = _ibis_pf(data, wastefree, lc, 100, ESSrmin, seed=5)
    l0 = context().launches
    b.run()
    torch.cuda.synchronize()
    assert b._ibis_stats is not None and b.t == a.t == T
    st = b._ibis_stats
    assert a.summaries.rs_flags == b.summaries.rs_flags
    assert a.summaries.ESSs == b.summaries.ESSs
    assert a.summaries.logLts == b.summaries.logLts and a.logLt == b.logLt
    assert np.array_equal(host(a.X.theta), host(b.X.theta))
    assert np.array_equal(host(a.X.lpost), host(b.X.lpost))
    assert np.array_equal(host(a.X.llik), host(b.X.llik))
    assert np.array_equal(host(a.W), host(b.W))
    n_rs = sum(b.summaries.rs_flags)
    # every step is step 0, a resampling step, a step after a below-threshold step, or a row of a stretch
    assert st["reads"] == st["stretches"] and st["rows"] <= T - 1 - n_rs
    assert context().launches > l0
    if ESSrmin == 1.0:
        assert st["stretches"] == 0 and n_rs == T - 1
    else:
        assert st["stretches"] > 0 and st["rows"] >= T // 4 and st["stretches"] < st["rows"]
    if K0 == 1024:
        assert not b.summaries.rs_flags[-1] and st["last"] == T     # the final stretch ends at the last row


def test_linear_regression_static_model_vs_closed_form():
    """The reference's own IBIS check (tests/smc_samplers/linear_reg.py) through the generic StaticModel path, user
    logpyt on CUDA tensors: T = 30, d = 3, sigma = 0.1, prior scale 10, MvNormal field 'beta'.  Over 20 seeds the
    mean logLt is within 3 sigma (+ the Jensen bias sd^2 / 2) of the closed-form evidence, and the posterior mean
    and variance agree with the closed form."""
    import torch
    import particles_b200 as pb
    from particles_b200 import distributions as dists
    from particles_b200 import smc_samplers as ssp
    T, d, sig, scale = 30, 3, 0.1, 10.0
    r = np.random.RandomState(0)
    preds = r.randn(T, d)
    preds[:, 0] = 1.0
    response = preds @ np.array([0.3, 1.0, -0.2]) + sig * r.randn(T)
    data = np.empty((T, d + 1))
    data[:, 0], data[:, 1:] = response, preds
    evid = stats.multivariate_normal.logpdf(response, cov=sig ** 2 * np.eye(T) + scale ** 2 * preds @ preds.T)
    covp = np.linalg.inv(preds.T @ preds / sig ** 2 + np.eye(d) / scale ** 2)
    meanp = covp @ (preds.T @ response) / sig ** 2

    class LinearRegression(ssp.StaticModel):
        def logpyt(self, theta, t):
            assert isinstance(theta["beta"], torch.Tensor) and theta["beta"].is_cuda and theta["beta"].shape[1] == d
            lin = theta["beta"] @ self.data[t, 1:]
            return -0.5 * ((self.data[t, 0] - lin) / sig) ** 2 - np.log(sig) - 0.5 * np.log(2 * np.pi)

    prior = dists.StructDist({"beta": dists.MvNormal(scale=scale, cov=np.eye(d))})
    lls, means, varis = [], [], []
    for s in range(20):
        model = LinearRegression(data=data, prior=prior)
        pf = pb.SMC(fk=ssp.IBIS(model=model, len_chain=20), N=200, seed=300 + s)
        pf.run()
        assert getattr(pf, "_ibis_stats", None) is None          # user logpyt: the per-step loop
        assert pf.X.theta.shape == (4000, d)
        W = host(pf.W)
        th = host(pf.X.theta)
        m = W @ th
        lls.append(pf.logLt)
        means.append(m)
        varis.append(W @ (th - m) ** 2)
    lls, means, varis = np.array(lls), np.array(means), np.array(varis)
    sd = lls.std(ddof=1)
    assert abs(lls.mean() - evid) < 3 * sd / np.sqrt(20) + 0.5 * sd ** 2, (lls.mean(), evid, sd)
    msd = means.std(axis=0, ddof=1)
    assert np.all(np.abs(means.mean(0) - meanp) < 4 * msd / np.sqrt(20) + 1e-3 * np.sqrt(np.diag(covp)))
    np.testing.assert_allclose(varis.mean(0), np.diag(covp), rtol=0.1)


@pytest.fixture(scope="module")
def gi():
    return np.load(os.path.join(HERE, "golden", "golden_ibis.npz"))


def test_fused_logistic_ibis_vs_reference_runs_and_tempering(gi):
    """Fused logistic IBIS (device reweighting, stretches, one-launch waste-free move) against 12 runs of the
    reference on the same data: logLt mean and posterior mean within 3 sigma; its evidence agrees with
    AdaptiveTempering on the same data within the combined 3 sigma."""
    import particles_b200 as pb
    from particles_b200 import smc_samplers as ssp
    data = gi["stat/data"]
    N, P = (int(v) for v in gi["stat/meta"])
    ref_ll, ref_mean = gi["stat/logLt"], gi["stat/post_mean"]
    mu, sd = ref_ll.mean(), ref_ll.std(ddof=1)
    R = 8
    lls, means, tls = [], [], []
    for s in range(R):
        pf = _ibis_pf(data, True, P, N, 0.5, seed=60 + s)
        pf.run()
        assert pf._ibis_stats["stretches"] > 0
        W = host(pf.W)
        lls.append(pf.logLt)
        means.append(W @ host(pf.X.theta))
        tp = pb.SMC(fk=ssp.AdaptiveTempering(model=ssp.LogisticRegression(data=data), wastefree=True, len_chain=P),
                    N=N, ESSrmin=1.0, seed=90 + s)
        tp.run()
        tls.append(tp.logLt)
    lls, means, tls = np.array(lls), np.array(means), np.array(tls)
    assert abs(lls.mean() - mu) < 3 * sd * np.sqrt(1 / R + 1 / len(ref_ll)) + 1e-6, (lls, mu, sd)
    msd = ref_mean.std(axis=0, ddof=1)
    assert np.all(np.abs(means.mean(0) - ref_mean.mean(0)) < 3 * msd * np.sqrt(1 / R + 1 / 12) + 1e-3)
    comb = np.sqrt(lls.var(ddof=1) / R + tls.var(ddof=1) / R)
    assert abs(lls.mean() - tls.mean()) < 3 * comb + 1e-6, (lls.mean(), tls.mean(), comb)


def test_refusals():
    from particles_b200 import smc_samplers as ssp
    with pytest.raises(NotImplementedError, match="d <= 20"):
        ssp.IBIS(model=ssp.LogisticRegression(data=sp.synthetic_logistic(10, 21, seed=1)))
    with pytest.raises(NotImplementedError, match="logpyt"):
        ssp.IBIS(model=ssp.StaticModel(data=np.zeros((5, 2)), prior=None))
