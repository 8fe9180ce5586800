"""The conditional-SMC replay (tests/csmc_replay.py) on the CPU: it predicts every decision, ancestor, particle,
log-weight and trajectory index of the NumPy conditional SMC (``oracle.pmcmc_numpy.CSMC`` and ``draw_trajectory``)
for every model and kind the kernel builds, it rejects planted faults, and the rules it holds the kernel to for a
row with no positive weight and for a zero spacing uniform are the reference's."""
import numpy as np
import pytest

import csmc_replay as cr
from oracle import pmcmc_numpy as pmo
from oracle import smc_numpy as orc
from oracle.smoothing_numpy import px_logpt


def _built():
    from particles_b200.bank import _MAPS
    out = []
    for name, (_, _, proposal, _) in _MAPS.items():
        out.append((name, False))
        if proposal:
            out.append((name, True))
    return out


def _tmap(name, T, seed):
    from particles_b200.bank import ThetaMap
    r = np.random.RandomState(seed)
    y = r.poisson(2.0, T).astype(np.float64) if name == "DiscreteCox" else r.standard_normal(T)
    cls = type(name, (), {"__module__": "particles_b200.state_space_models"})
    return ThetaMap(cls, [], y)


def _run(name, guided, N, T, essrmin, pin, backward, seed=0):
    """One oracle conditional run with its noise, the pinned path taken from a second unconditional run."""
    m = _tmap(name, T, seed)
    fk, trans = cr.chain_objects(m, np.empty((1, 0)), guided)[0]
    r = np.random.RandomState(100 + seed)
    z, u, ud = r.standard_normal((2, T, N)), r.rand(2, T, N + 1), r.rand(2, T)
    xstar = None
    if pin:
        h = pmo.CSMC(fk, N=N, ESSrmin=essrmin, noise=orc.InjectedNoise(z[1], u[1])).run().hist
        xstar = pmo.draw_trajectory(h, px_logpt(fk.ssm), ud[1], False)[0]
    o = pmo.CSMC(fk, N=N, ESSrmin=essrmin, xstar=xstar, noise=orc.InjectedNoise(z[0], u[0])).run()
    h = o.hist
    traj, idx = pmo.draw_trajectory(h, px_logpt(fk.ssm), ud[0], backward)
    out = dict(fk=fk, trans=trans, X=np.stack(h["X"]), lw=np.stack(h["lw"]), A=np.stack(h["A"]),
               summ=cr.oracle_summaries(o), logLt=o.logLt, z=z[0], u=u[0], ud=ud[0], xstar=xstar, traj=traj, idx=idx)
    return out


def _check(rep, d, **over):
    d = dict(d, **over)
    return rep.check_chain(d["fk"], d["X"], d["lw"], d["A"], d["summ"], d["logLt"], d["z"], d["u"], xstar=d["xstar"],
                           traj=d["traj"], ud=d["ud"], trans=d["trans"])


# pin, draw, N: odd and even N, both draws, pin on and off
COMBOS = [(False, "genealogy", 31), (True, "backward", 40), (True, "genealogy", 33), (False, "backward", 26)]


@pytest.mark.parametrize("pin,draw,N", COMBOS)
@pytest.mark.parametrize("name,guided", _built())
def test_replay_predicts_the_oracle(name, guided, pin, draw, N):
    T, essrmin = 14, 0.9
    d = _run(name, guided, N, T, essrmin, pin, draw == "backward", seed=N)
    rep = cr.CsmcReplay(N, essrmin, pin, draw, x_exact=True)
    idx = _check(rep, d)
    assert np.array_equal(idx, d["idx"])
    assert rep.n_rs == int(d["summ"][:, 2].sum()) and rep.n_rs >= 1
    assert rep.n_und <= 2 and rep.n_near == 0


def _faulty():
    d = _run("LinearGauss", True, 40, 14, 0.8, True, True, seed=5)
    rs = np.flatnonzero(d["summ"][:, 2] != 0)
    assert rs.size >= 2
    return d, int(rs[0])


def test_replay_rejects_a_moved_ancestor():
    d, t = _faulty()
    A = d["A"].copy()
    A[t, 7] = (A[t, 7] + 1) % 40
    with pytest.raises(AssertionError, match="ancestor"):
        _check(cr.CsmcReplay(40, 0.8, True, "backward", x_exact=True), d, A=A)


def test_replay_rejects_a_one_ulp_particle():
    d, t = _faulty()
    X = d["X"].copy()
    X[t, 9] = np.nextafter(X[t, 9], np.inf)
    with pytest.raises(AssertionError, match="bit-identical"):
        _check(cr.CsmcReplay(40, 0.8, True, "backward", x_exact=True), d, X=X)


def test_replay_rejects_the_pinned_slot_weighted_from_its_resampled_ancestor():
    d, _ = _faulty()
    fk, N = d["fk"], 40
    for t in np.flatnonzero(d["summ"][:, 2] != 0):
        W = orc.exp_and_normalise(d["lw"][t - 1])
        a0 = int(orc.multinomial(W, N, d["u"][t])[0])         # the ancestor slot 0 drew before it was pinned
        if a0 != 0:
            break
    assert a0 != 0
    lw = d["lw"].copy()
    lw[t, 0] = orc.Weights(np.asarray(fk.logG(t, d["X"][t - 1][a0:a0 + 1], d["xstar"][t:t + 1]), dtype=float)).lw[0]
    assert lw[t, 0] != d["lw"][t, 0]
    with pytest.raises(AssertionError, match="lw"):
        _check(cr.CsmcReplay(N, 0.8, True, "backward", x_exact=True), d, lw=lw)


@pytest.mark.parametrize("draw", ["genealogy", "backward"])
def test_replay_rejects_a_trajectory_index_off_by_one(draw):
    d = _run("StochVol", False, 40, 14, 0.8, True, draw == "backward", seed=6)
    for t in (d["X"].shape[0] - 1, 5):
        traj = d["traj"].copy()
        traj[t] = d["X"][t, (d["idx"][t] + 1) % 40]
        with pytest.raises(AssertionError, match="trajectory"):
            _check(cr.CsmcReplay(40, 0.8, True, draw, x_exact=True), d, traj=traj)


def test_replay_rejects_a_flipped_decision():
    d, t = _faulty()
    summ = d["summ"].copy()
    summ[t + 1, 2] = 1.0 - summ[t + 1, 2]
    with pytest.raises(AssertionError, match="rs"):
        _check(cr.CsmcReplay(40, 0.8, True, "backward", x_exact=True), d, summ=summ)


def test_all_zero_row_gives_the_first_particle():
    """The reference's draw on weights that are all zero: exp_and_normalise gives NaN everywhere, and searchsorted of
    any u in that all-NaN CDF is 0."""
    N = 7
    lw = np.full(N, -np.inf)
    with np.errstate(invalid="ignore"):
        W = orc.exp_and_normalise(lw)
        cdf = np.cumsum(W)
    assert np.isnan(cdf).all()
    for u in (0.0, 1e-300, 0.3, 1.0 - 2.0 ** -53):
        assert min(int(np.searchsorted(cdf, u)), N - 1) == 0
        with np.errstate(invalid="ignore"):
            assert orc.multinomial_once(W, u) == 0
    # the replay holds a draw on such a row to 0
    from step_replay import LD
    rep = cr.CsmcReplay(N, 0.5, False, "backward")
    assert rep._draw(0, LD(1) * lw, np.zeros(N), 0.4, [0]) == 0 and rep.n_zero == 1
    with pytest.raises(AssertionError):
        rep._draw(0, LD(1) * lw, np.zeros(N), 0.4, [1])


def test_zero_spacing_uniform_gives_ancestor_zero():
    """u = 0 among the N + 1 spacing uniforms: the reference's uniform_spacings gives 0 before it and NaN from it on,
    and its inverse-CDF loop (``while su[n] > s``) then returns 0 for every grid point."""
    N = 9
    W = orc.exp_and_normalise(np.random.RandomState(1).standard_normal(N))
    W[0] = 0.0
    for i0 in (0, 4, N):
        u = np.random.RandomState(i0).rand(N + 1)
        u[i0] = 0.0
        with np.errstate(divide="ignore", invalid="ignore"):
            su = orc.uniform_spacings(N, u)
        assert np.all((su == 0) | np.isnan(su)) and np.isnan(su[i0:]).all()
        j, s, A = 0, W[0], []
        for v in su:                                          # particles/resampling.py:500-508
            while v > s:
                j += 1
                s += W[j]
            A.append(j)
        assert A == [0] * N
        rep = cr.CsmcReplay(N, 0.5, False, "genealogy")
        with np.errstate(divide="ignore"):
            lw = np.log(W)
        rep.check_ancestors(1, lw, u, np.zeros(N, dtype=np.int64))
        with pytest.raises(AssertionError):
            rep.check_ancestors(1, lw, u, np.arange(N))
        assert rep.n_u0 == 2


def test_device_noise_counters_are_disjoint():
    """The normals, the spacing uniforms and the trajectory uniform of a chain use disjoint Philox counters, and
    ``device_noise`` reads them from those counters."""
    for N, T in ((1, 3), (2, 2), (513, 4), (4097, 2)):
        c = cr.counters(N, T)
        assert not (c["normals"] & c["spacings"]) and not (c["normals"] & c["traj"]) and not (c["spacings"] & c["traj"])
        assert len(c["normals"]) == T * ((N + 1) // 2) and len(c["spacings"]) == T * ((N + 2) // 2)
    key = 0x0123456789ABCDEF
    z, u, ud = cr.device_noise(5, 3, key)
    from philox_ref import philox4x32_10, u53
    for t in range(3):
        w = philox4x32_10(np.uint32(0), np.uint32(0), np.uint32(t), np.uint32(cr.PURPOSE_TRAJ), key & 0xFFFFFFFF,
                          key >> 32)
        assert ud[t] == u53(w[0], w[1])
        w = philox4x32_10(np.uint32(2), np.uint32(0), np.uint32(t), np.uint32(2), key & 0xFFFFFFFF, key >> 32)
        assert u[t, 4] == u53(w[0], w[1]) and u[t, 5] == u53(w[2], w[3])
    assert z.shape == (3, 5) and u.shape == (3, 6)
