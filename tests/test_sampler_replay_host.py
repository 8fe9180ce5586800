"""The sampler replay (tests/sampler_replay.py) checked without a GPU: fed the NumPy oracle's own waste-free moves and
calibrations (oracle/samplers_numpy.py), it must predict every decision and row and accept every covariance and
factor -- and it must reject a flipped decision, a one-ulp change in a rejected row, two generation rows swapped, a
covariance with two off-diagonal entries swapped and a root one bracket off."""
import numpy as np
import pytest

from oracle import samplers_numpy as sp
from oracle import smc_numpy as orc
import philox_ref
import sampler_replay as sr


def fields(x):
    return {"theta": x.theta, "lprior": x.lprior, "llik": x.llik, "lpost": x.lpost}


def oracle_move(d, M, P, n_data, epn, seed):
    """An oracle MCMCSequenceWF move with injected draws: (generations, pb rows, z, u, L, data)."""
    data = sp.synthetic_logistic(n_data, d, seed=seed)
    r = np.random.RandomState(seed + 100)
    theta = r.randn(M, d)
    W = orc.exp_and_normalise(r.randn(M))
    z, u = r.standard_normal((P - 1, M, d)), r.rand(P - 1, M)
    fk = sp.AdaptiveTemperingWF(sp.LogisticModel(data), len_chain=P)
    x = sp.ThetaParticles(theta=theta)
    fk.target(epn)(x)
    fk.calibrate(W, x)
    L = x.shared["chol_cov"]
    gens, pbs = [fields(x)], []
    for s in range(P - 1):
        x = x.copy()
        xp = sp.ThetaParticles(theta=x.theta + z[s] @ L.T)
        fk.target(epn)(xp)
        pb = np.exp(np.clip(xp.lpost - x.lpost, None, 0.0))
        x.copyto(xp, where=u[s] < pb)
        gens.append(fields(x))
        pbs.append(pb)
    return gens, pbs, z, u, L, data


@pytest.mark.parametrize("d,M,P,n_data,epn", [(2, 40, 4, 30, 0.5), (3, 200, 6, 80, 1.0), (5, 300, 5, 120, 0.45),
                                              (12, 150, 4, 60, 0.2), (20, 120, 3, 200, 0.7), (25, 64, 3, 40, 0.0)])
def test_replay_predicts_oracle_move(d, M, P, n_data, epn):
    gens, pbs, z, u, L, data = oracle_move(d, M, P, n_data, epn, seed=d)
    n_acc = n_dec = 0
    for s in range(1, P):
        acc, decided = sr.check_generation(s, gens[s - 1], gens[s], pbs[s - 1], z[s - 1], u[s - 1], L, data, 5.0,
                                           epn, d)
        want = u[s - 1] < pbs[s - 1]
        assert np.array_equal(acc, want)              # every oracle decision is seen, decided or not
        n_acc += int(acc.sum())
        n_dec += int(decided.sum())
    assert 0 < n_acc < (P - 1) * M and n_dec >= 0.99 * (P - 1) * M


@pytest.mark.parametrize("d,n", [(1, 50), (2, 7), (6, 3001), (13, 400), (20, 2111)])
def test_replay_accepts_oracle_calibration(d, n):
    r = np.random.RandomState(d)
    theta = r.randn(n, d) @ np.tril(r.rand(d, d) + np.eye(d)).T + 3.0
    W = orc.exp_and_normalise(r.randn(n))
    m, cov = sp.wmean_and_cov(W, theta)
    cov = np.atleast_2d(cov)                                   # numpy.cov of one variable is 0-d
    sr.check_mean_cov(W, theta, m, cov, depth=n + 4)          # numpy's sums: any order of depth n
    L = np.linalg.cholesky(cov)
    sr.chol_backward_check(cov, L)


def test_tile_rows_and_tiers():
    """The shared-memory tiling of launch_wf: (200 KiB - 8 D^2) / (8 D) rows per tile."""
    assert [sr.tile_rows(D) for D in sr.TIERS] == [6396, 3192, 2121, 1584, 1260, 1042, 768]
    assert [sr.tier(d) for d in (1, 4, 5, 8, 9, 20, 21, 24, 25, 32)] == [4, 4, 8, 8, 12, 20, 24, 24, 32, 32]
    assert sr.wf_resident(16, 1584) and not sr.wf_resident(15, 1585)
    assert sr.wf_grid(32) == 1 and sr.wf_grid(33) == 2


def test_philox_replays_match_philox_ref():
    """The long-double Box-Muller of the counter layouts agrees with philox_ref's fp64 one to a few ulp, and the
    layouts differ where their counter words differ."""
    seed, call = 0x1234_5678_9ABC, (3 << 32) | 17
    n = 1001
    z = sr.rw_propose_normals(n, 5, call, seed)
    for j in range(0, 5, 2):
        w3 = ((3 << 16) | ((j >> 1) << 8) | philox_ref.PURPOSE_API)
        ref = philox_ref.normals(2 * n, call & 0xFFFFFFFF, seed, w3=w3)[0::2]   # pair i -> its first normal
        np.testing.assert_allclose(z[:, j].astype(np.float64), ref, rtol=8 * sr.EPS, atol=8 * sr.EPS)
    assert not np.allclose(z[:, 0].astype(float), z[:, 2].astype(float))
    u = sr.mh_accept_uniforms(n, call, seed)
    ref = philox_ref.uniforms(2 * n, call & 0xFFFFFFFF, seed, w3=(3 << 8) | philox_ref.PURPOSE_API)[0::2]
    assert np.array_equal(u, ref)
    zw = sr.wf_normals(n, 4, 3, call, seed)
    ref = philox_ref.normals(2 * n, call & 0xFFFFFFFF, seed, w3=(3 << 16) | (1 << 8) | philox_ref.PURPOSE_NORMAL)
    np.testing.assert_allclose(zw[:, 2].astype(np.float64), ref[0::2], rtol=8 * sr.EPS, atol=8 * sr.EPS)
    uw = sr.wf_uniforms(n, 2, call, seed)
    ref = philox_ref.uniforms(2 * n, call & 0xFFFFFFFF, seed, w3=(2 << 16) | philox_ref.PURPOSE_UNIFORM)[0::2]
    assert np.array_equal(uw, ref)


def device_like_root(lw, epn, alpha):
    """The device's 16-way, 11-pass bracketing with long-double ESS (no rounding near the grid points)."""
    n = lw.shape[0]
    lo, hi = 0.0, 1.0 - epn
    for p in range(sr.ROOT_PASSES):
        ess = [sr.ess_ld(lo + (hi - lo) * ((j + 1) / 16.0), lw) for j in range(16)]
        below = [j for j in range(16) if ess[j] < alpha * n]
        if not below:
            if p == 0:
                return 1.0
            j = 15
        else:
            j = below[0]
        lo, hi = lo + (hi - lo) * (j / 16.0), lo + (hi - lo) * ((j + 1) / 16.0)
    return epn + 0.5 * (lo + hi)


@pytest.mark.parametrize("n,scale,epn,alpha", [(5000, 40.0, 0.0, 0.5), (3001, 300.0, 0.013, 0.5),
                                               (2000, 5.0, 0.4, 0.99), (4000, 600.0, 0.2, 0.01)])
def test_root_check_accepts_the_bracketing_and_rejects_one_bracket_off(n, scale, epn, alpha):
    r = np.random.RandomState(n)
    lw = -np.abs(r.randn(n)) * scale - 3.0
    got = device_like_root(lw, epn, alpha)
    root = sr.root_ld(lw, epn, alpha)
    assert got < 1.0 and abs(got - root) <= 0.5 * sr.final_bracket(epn) * (1 + 1e-6)
    sr.check_root(lw, epn, alpha, got)
    sr.check_root(lw, epn, alpha, root)
    w0 = sr.final_bracket(epn)
    off = [got + w0, got - w0]
    rejected = 0
    for g in off:
        try:
            sr.check_root(lw, epn, alpha, g)
        except AssertionError:
            rejected += 1
    # the root lies in [got - w0 / 2, got + w0 / 2]: at least the side away from it is more than w0 / 2 off
    assert rejected >= 1
    with pytest.raises(AssertionError, match="ESS"):
        sr.check_root(lw, epn, alpha, got + 2 * w0 if abs(root - got - 2 * w0) > abs(root - got + 2 * w0)
                      else got - 2 * w0)


def test_root_check_special_values():
    """All-equal log-likelihoods and all -inf: 1.0; a single entry: 1.0."""
    sr.check_root(np.full(100, -4.0), 0.3, 0.5, 1.0)
    sr.check_root(np.array([2.5]), 0.0, 0.5, 1.0)
    with pytest.raises(AssertionError):
        sr.check_root(np.array([0.0, -50.0]), 0.0, 0.9, 1.0)


# ------------------------------------------------------------------------------------ negative controls
@pytest.fixture(scope="module")
def move():
    return oracle_move(6, 400, 4, 100, 0.6, seed=11)


def test_replay_rejects_a_flipped_accept(move):
    gens, pbs, z, u, L, data = move
    acc = u[0] < pbs[0]
    c = int(np.flatnonzero(acc & (pbs[0] > 2 * u[0]))[0])     # a clear accept
    out = {k: v.copy() for k, v in gens[1].items()}
    for k in out:
        out[k][c] = gens[0][k][c]
    with pytest.raises(AssertionError, match="rejected but"):
        sr.check_generation(1, gens[0], out, pbs[0], z[0], u[0], L, data, 5.0, 0.6, 6)


def test_replay_rejects_one_ulp_in_a_rejected_row(move):
    gens, pbs, z, u, L, data = move
    c = int(np.flatnonzero(~(u[0] < pbs[0]))[0])
    for k in ("llik", "lpost", "theta"):
        out = {kk: v.copy() for kk, v in gens[1].items()}
        out[k][c] = np.nextafter(out[k][c], np.inf)
        with pytest.raises(AssertionError, match="bit-identical|accepted but"):
            sr.check_generation(1, gens[0], out, pbs[0], z[0], u[0], L, data, 5.0, 0.6, 6)


def test_replay_rejects_swapped_generation_rows(move):
    gens, pbs, z, u, L, data = move
    with pytest.raises(AssertionError, match="generation 2"):
        sr.check_generation(2, gens[1], gens[3], pbs[1], z[1], u[1], L, data, 5.0, 0.6, 6)
    with pytest.raises(AssertionError, match="generation 3"):
        sr.check_generation(3, gens[3], gens[2], pbs[2], z[2], u[2], L, data, 5.0, 0.6, 6)


def test_replay_rejects_a_swapped_covariance():
    d, n = 5, 2000
    r = np.random.RandomState(4)
    theta = r.randn(n, d) @ np.tril(r.rand(d, d) + np.eye(d)).T
    W = orc.exp_and_normalise(r.randn(n))
    m, cov = sp.wmean_and_cov(W, theta)
    sr.check_mean_cov(W, theta, m, cov, depth=n + 4)
    bad = cov.copy()
    bad[1, 0], bad[2, 0] = cov[2, 0], cov[1, 0]
    bad[0, 1], bad[0, 2] = bad[1, 0], bad[2, 0]
    with pytest.raises(AssertionError, match="covariance"):
        sr.check_mean_cov(W, theta, m, bad, depth=n + 4)
    # and a factor that is not the covariance's: one off-diagonal entry of L moved by 1e-9
    L = np.linalg.cholesky(cov)
    L[3, 1] += 1e-9
    with pytest.raises(AssertionError, match="Cholesky"):
        sr.chol_backward_check(cov, L)
