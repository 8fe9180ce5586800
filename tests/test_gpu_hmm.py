"""Hidden Markov models on the H100: ``BaumWelch`` (csrc/smcb_hmm.cu) against the live reference's fixture
(tests/golden/golden_hmm.npz), against the long-double replay (tests/hmm_replay.py) at both tier edges with batches
wider than one wave, its trajectory draws against the replay of its own Philox draws and against the exact
marginals, a bootstrap filter on a ``GaussianHMM`` against the exact likelihood, and the edges of the surface."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hmm_oracle as oh  # noqa: E402
import hmm_replay as rp  # noqa: E402

CASES = ("a", "b", "c", "d", "e")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_hmm.npz"))


def host(x):
    return x.detach().cpu().numpy()


def fixture_model(g, c):
    from particles_b200 import hmm
    return hmm.GaussianHMM(trans_mat=g[c + "_trans"], init_dist=g[c + "_init"], mus=g[c + "_mus"],
                           sigmas=g[c + "_sigmas"])


def random_model(rng, K, B=None):
    lead = () if B is None else (B,)
    trans = rng.dirichlet(np.full(K, 0.5), size=lead + (K,)) + 0.2 * np.eye(K)
    trans /= trans.sum(-1, keepdims=True)
    init = rng.dirichlet(np.ones(K), size=lead) if B is not None else rng.dirichlet(np.ones(K))
    mus = rng.normal(0.0, 2.0, size=lead + (K,))
    sigmas = rng.uniform(0.5, 1.5, size=lead + (K,))
    return trans, init, mus, sigmas


def ulp_diff(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ia, ib = a.view(np.int64), b.view(np.int64)
    return np.abs(ia - ib)


# ------------------------------------------------------------------------------------------------------------------
# 1. against the reference's fixture
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES)
def test_against_fixture(g, c):
    from particles_b200 import hmm
    bw = hmm.BaumWelch(hmm=fixture_model(g, c), data=g[c + "_y"])
    bw.run()
    T = g[c + "_y"].shape[0]
    assert bw.t == T and len(bw.filt) == T and bw.smth.shape == (T, g[c + "_trans"].shape[0])
    assert int(ulp_diff(host(bw.logft), g[c + "_logft"]).max()) <= 2
    for k in ("pred", "filt", "smth", "logpyt"):
        np.testing.assert_allclose(host(getattr(bw, k)), g[c + "_" + k], rtol=0, atol=1e-12, err_msg=k)
    N = int(g["N_sample"])
    last, U = oh.reference_uniforms(int(g[c + "_sample_seed"]), N, T)
    paths = bw.sample(N, noise={"last": last, "U": U})
    assert paths.dtype == torch.int64 and paths.shape == (T, N)
    np.testing.assert_array_equal(host(paths), g[c + "_paths"])


def test_incremental_smoothing_of_fixture(g):
    from particles_b200 import hmm
    y = list(g["a_y"])
    bw = hmm.BaumWelch(hmm=fixture_model(g, "a"), data=y)
    rows = []
    for _ in range(30):
        bw.next()
        bw.backward()
        rows.append(host(bw.smth))
    np.testing.assert_allclose(np.concatenate(rows), g["a_smth_steps"], rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------
# 2. stepping
# ------------------------------------------------------------------------------------------------------------------
def test_next_equals_forward_and_appending_continues(g):
    from particles_b200 import hmm
    m = fixture_model(g, "b")
    y = g["b_y"]
    full = hmm.BaumWelch(hmm=m, data=y)
    full.forward()
    step = hmm.BaumWelch(hmm=m, data=y)
    for _ in step:
        pass
    with pytest.raises(StopIteration):
        step.next()
    for k in ("pred", "filt", "logpyt", "logft"):
        assert torch.equal(getattr(step, k), getattr(full, k)), k
    data = [torch.tensor([v], dtype=torch.float64, device="cuda") for v in y[:37]]
    grow = hmm.BaumWelch(hmm=m, data=data)
    grow.forward()
    data.extend(torch.tensor([v], dtype=torch.float64, device="cuda") for v in y[37:120])
    grow.next()
    grow.forward()
    data.extend(float(v) for v in y[120:])
    grow.forward()
    assert grow.t == y.shape[0]
    for k in ("pred", "filt", "logpyt", "logft"):
        assert torch.equal(getattr(grow, k), getattr(full, k)), k
    grow.backward()
    full.backward()
    assert torch.equal(grow.smth, full.smth)


# ------------------------------------------------------------------------------------------------------------------
# 3. tier edges, against the long-double replay; each batch row as run alone
# ------------------------------------------------------------------------------------------------------------------
def check_replay(trans, init, logft, out):
    r = rp.run(init, trans, logft)
    for k in ("pred", "filt", "smth", "logpyt"):
        np.testing.assert_allclose(out[k], r[k].astype(float), rtol=0, atol=1e-12, err_msg=k)


@pytest.mark.parametrize("K", [1, 2, 31, 32, 33, 64, 127, 128])
@pytest.mark.parametrize("B", [1, 1000])
def test_tier_edges_against_replay(K, B):
    from particles_b200 import hmm
    rng = np.random.RandomState(1000 * K + B)
    T = 200
    trans, init, mus, sigmas = random_model(rng, K, None if B == 1 else B)
    y = rng.normal(0.0, 2.0, size=(T,) if B == 1 else (B, T))
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas), data=y)
    bw.run()
    out = {k: host(getattr(bw, k)) for k in ("pred", "filt", "smth", "logpyt", "logft")}
    if B == 1:
        check_replay(trans, init, out["logft"], out)
        return
    for b in (0, 1, B // 2, B - 1):                   # rows in the first and the last wave
        row = {k: v[b] for k, v in out.items()}
        check_replay(trans[b], init[b], row["logft"], row)
        alone = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans[b], init_dist=init[b], mus=mus[b],
                                                  sigmas=sigmas[b]), data=y[b])
        alone.run()
        for k in ("pred", "filt", "smth", "logpyt", "logft"):
            np.testing.assert_array_equal(host(getattr(alone, k)), row[k], err_msg=f"{k} b={b}")


def test_batch_shares_unbatched_parameters():
    from particles_b200 import hmm
    rng = np.random.RandomState(3)
    K, B, T = 6, 40, 50
    trans, _, mus, sigmas = random_model(rng, K, B)
    init = rng.dirichlet(np.ones(K))
    y = rng.normal(size=(B, T))
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas), data=y)
    bw.run()
    paths = bw.sample(16, seed=5)
    assert paths.shape == (B, T, 16) and bw.smth.shape == (B, T, K) and bw.logpyt.shape == (B, T)
    alone = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans[7], init_dist=init, mus=mus[7], sigmas=sigmas[7]),
                          data=y[7])
    alone.run()
    assert torch.equal(alone.smth, bw.smth[7]) and torch.equal(alone.logpyt, bw.logpyt[7])


# ------------------------------------------------------------------------------------------------------------------
# 4. trajectory draws with the device's own uniforms
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [5, 40])
def test_sample_replays_device_draws(K):
    from particles_b200 import hmm
    rng = np.random.RandomState(K)
    T, N, seed = 120, 4096, 12345 + K
    trans, init, mus, sigmas = random_model(rng, K)
    y = rng.normal(0.0, 2.0, size=T)
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas), data=y)
    bw.run()
    paths = host(bw.sample(N, seed=seed))
    assert np.all(np.diff(paths[-1]) >= 0)                            # the last row is sorted, as the reference's
    U = rp.device_uniforms(seed, N, T)
    rpaths, gap = rp.sample(trans, host(bw.filt), paths[-1], U)
    bad = rpaths != paths
    print(f"K={K}: {int(bad.sum())} of {(T - 1) * N} draws differ from the replay")
    assert np.all(gap[bad] < 1e-13)
    again = host(bw.sample(N, seed=seed))
    other = host(bw.sample(N, seed=seed + 1))
    assert np.array_equal(again, paths) and not np.array_equal(other, paths)


def test_sample_frequencies_match_exact_marginals():
    from particles_b200 import hmm
    rng = np.random.RandomState(11)
    K, T, N = 4, 50, 2 ** 20
    trans, init, mus, sigmas = random_model(rng, K)
    y = rng.normal(0.0, 2.0, size=T)
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas), data=y)
    bw.run()
    paths = bw.sample(N, seed=99)
    freq = torch.stack([torch.bincount(paths[t], minlength=K) for t in range(T)]).double() / N
    smth = host(bw.smth)
    sd = np.sqrt(np.maximum(smth * (1 - smth), 1.0 / N) / N)          # sd floored at one count
    assert np.all(np.abs(host(freq) - smth) <= 5 * sd)
    r = rp.run(init, trans, host(bw.logft))
    xi = rp.two_slice(trans, r["pred"], r["filt"], r["smth"]).astype(float)       # (T-1, K, K)
    pair = torch.stack([torch.bincount(paths[t] * K + paths[t + 1], minlength=K * K) for t in range(T - 1)])
    pf = host(pair.double() / N).reshape(T - 1, K, K)
    sd = np.sqrt(np.maximum(xi * (1 - xi), 1.0 / N) / N)
    np.testing.assert_allclose(xi.sum(axis=(1, 2)), 1.0, atol=1e-12)
    assert np.all(np.abs(pf - xi) <= 5 * sd)


# ------------------------------------------------------------------------------------------------------------------
# 5. a bootstrap filter against the exact answer
# ------------------------------------------------------------------------------------------------------------------
def test_bootstrap_filter_against_exact():
    import particles_b200 as pb
    from particles_b200 import hmm, state_space_models as ssm
    rng = np.random.RandomState(21)
    K, T, N, R = 5, 100, 10 ** 4, 32
    trans, init, mus, sigmas = random_model(rng, K)
    m = hmm.GaussianHMM(trans_mat=trans, init_dist=init, mus=mus, sigmas=sigmas)
    _, y = m.simulate(T)
    bw = hmm.BaumWelch(hmm=m, data=y)
    bw.forward()
    exact = float(bw.logpyt.sum())
    ll, est = [], []
    for s in range(R):
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=m, data=y), N=N, seed=s)
        pf.run()
        ll.append(float(pf.logLt))
        X = pf.X.reshape(-1).long()
        est.append(host(torch.zeros(K, dtype=torch.float64, device="cuda").index_add_(0, X, pf.W)))
    ll, est = np.array(ll), np.array(est)
    assert abs(ll.mean() - exact) <= 4 * ll.std(ddof=1) / np.sqrt(R)
    se = est.std(axis=0, ddof=1) / np.sqrt(R) + 1e-9
    assert np.all(np.abs(est.mean(axis=0) - host(bw.filt[-1])) <= 6 * se)


# ------------------------------------------------------------------------------------------------------------------
# 6. edges
# ------------------------------------------------------------------------------------------------------------------
def test_one_state_and_one_step():
    from particles_b200 import hmm
    y = np.array([0.3, -1.0, 2.0])
    bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=np.ones((1, 1)), mus=np.zeros(1), sigmas=np.ones(1)), data=y)
    bw.run()
    assert torch.equal(bw.filt, torch.ones(3, 1, dtype=torch.float64, device="cuda"))
    np.testing.assert_allclose(host(bw.logpyt), oh.gaussian_logft([0.0], [1.0], y)[:, 0], rtol=0, atol=1e-15)
    assert torch.equal(bw.sample(8), torch.zeros(3, 8, dtype=torch.int64, device="cuda"))
    one = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=np.array([[0.5, 0.5], [0.5, 0.5]]), mus=np.zeros(2),
                                            sigmas=np.ones(2)), data=[0.1])
    one.backward()                                                    # runs forward: no step was taken
    assert one.t == 1 and torch.equal(one.smth, one.filt)
    assert one.sample(5).shape == (1, 5)


def test_zero_transitions_match_reference(g):
    from particles_b200 import hmm
    bw = hmm.BaumWelch(hmm=fixture_model(g, "d"), data=g["d_y"])
    bw.run()
    assert np.any(g["d_filt"] == 0.0)
    np.testing.assert_array_equal(host(bw.filt) == 0.0, g["d_filt"] == 0.0)
    np.testing.assert_allclose(host(bw.smth), g["d_smth"], rtol=0, atol=1e-12)


def test_errors():
    from particles_b200 import hmm
    with pytest.raises(ValueError, match="Transition Matrix is missing"):
        hmm.GaussianHMM(mus=np.zeros(2), sigmas=np.ones(2))
    with pytest.raises(AssertionError, match="Wrong shape for trans_mat or init_dist"):
        hmm.HMM(trans_mat=np.ones((2, 3)) / 3)
    with pytest.raises(AssertionError, match="Wrong shape for trans_mat or init_dist"):
        hmm.HMM(trans_mat=np.eye(3), init_dist=np.ones(2) / 2)
    big = hmm.GaussianHMM(trans_mat=np.full((129, 129), 1.0 / 129), mus=np.zeros(129), sigmas=np.ones(129))
    with pytest.raises(NotImplementedError, match="128"):
        hmm.BaumWelch(hmm=big, data=np.zeros(3))
    assert big.PX0().rvs(size=4).shape == (4,)                        # the plugin path is unaffected
