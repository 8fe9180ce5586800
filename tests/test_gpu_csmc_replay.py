"""The conditional SMC kernel (k_csmc, csrc/smcb_pmcmc.cu) step by step against a long-double replay
(tests/csmc_replay.py), with injected noise and with the kernel's own Philox draws.

The kernel runs 256 threads per chain over pairs of particles, scans the n weights and the n + 1 spacings in tiles
of 2048 entries, and its persistent grid (``runs.plan()``) loops each CTA over chains ``r += gridDim.x``.  The sizes
below reach two passes of the pair loop, a second scan tile of either scan, the shared-memory bound nmax, and a
second chain on a CTA; every case asserts the regime it is meant to reach on the device that runs it.  One launch
keeps every generation, so each step is replayed from the kernel's own generation t - 1."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import csmc_replay as cr  # noqa: E402
from particles_b200 import _lib, mcmc  # noqa: E402
from particles_b200.bank import FilterBank, ThetaMap, _MAPS  # noqa: E402
from particles_b200.device import as_device  # noqa: E402
from particles_b200.smc_samplers import _KeyCounter  # noqa: E402

BS, TILE = 256, 2048                       # kBatchBS, kScanItems * kBatchBS
PHILOX = dict(x_rtol=1e-12, x_atol=1e-12)  # the host's Box-Muller differs from the device's by a few ulp
INJ = dict(x_rtol=1e-13, x_atol=1e-14)


def host(t):
    return t.detach().cpu().numpy()


def _data(name, T, seed=0):
    r = np.random.RandomState(seed)
    if name == "DiscreteCox":
        return r.poisson(2.0, T).astype(np.float64)
    return r.standard_normal(T)


def _tmap(name, T, names=(), seed=0):
    cls = type(name, (), {"__module__": "particles_b200.state_space_models"})
    return ThetaMap(cls, list(names), _data(name, T, seed))


def _rows(m, R, names=(), special=None):
    """(R, len(names)) parameter rows at the model's defaults; ``special``: {chain: {name: value}}."""
    rows = np.array([[float(m.defaults[k]) if m.defaults[k] is not None else 0.0 for k in names]] * R)
    for r, kv in (special or {}).items():
        for k, v in kv.items():
            rows[r, list(names).index(k)] = v
    return rows.reshape(R, len(names))


class Case:
    """R chains of one model / kind at N: the device buffers, the replay's objects, and the checks."""

    def __init__(self, name, kind, N, R, T, essrmin, draw, names=(), special=None, data2d=None, seed=7):
        self.m = _tmap(name, T, names)
        self.kind, self.N, self.R, self.T, self.essrmin, self.draw = kind, N, R, T, essrmin, draw
        self.rows = _rows(self.m, R, names, special)
        self.data2d = data2d
        self.runs = mcmc._CsmcRuns(self.m, kind, N, R, essrmin, draw)
        if data2d is not None:
            self.runs.data = as_device(np.ascontiguousarray(data2d))
        self.keys = _KeyCounter(seed)
        self.runs.set_rows(self.rows, self.keys)
        self.nmax, self.grid = self.runs.plan()
        self.objs = cr.chain_objects(self.m, self.rows, kind == _lib.FK_GUIDED, data2d)

    def regime(self):
        """(pair-loop passes, weight scan tiles, spacing scan tiles, most chains on one CTA)."""
        N = self.N
        return -(-((N + 1) // 2) // BS), -(-N // TILE), -(-(N + 1) // TILE), -(-self.R // self.grid)

    def run(self, pin, noise=None):
        summ = torch.zeros((self.R, self.T, 4), dtype=torch.float64, device="cuda")
        dn = None if noise is None else {k: as_device(np.ascontiguousarray(v)) for k, v in noise.items()}
        self.runs.run(pin, noise=dn, summaries=summ)
        torch.cuda.synchronize()
        self.summ, self.noise, self.pin = summ, noise, pin

    def pinned_from_previous(self):
        """x* of chain r: the trajectory the previous launch drew for chain r + 1; then fresh keys."""
        self.runs.xstar.copy_(torch.roll(self.runs.traj, -1, dims=0))
        self.runs.set_rows(self.rows, self.keys)

    def check(self, chains, **tol):
        N, T = self.N, self.T
        rep = cr.CsmcReplay(N, self.essrmin, self.pin, self.draw, **(tol or (INJ if self.noise else PHILOX)))
        idx = torch.as_tensor(sorted(set(int(c) for c in chains)), device="cuda")
        sel = lambda a: host(a.index_select(0, idx))                                       # noqa: E731
        X, lw, A = sel(self.runs.X)[:, :, :N], sel(self.runs.lw)[:, :, :N], sel(self.runs.A)[:, :, :N]
        summ, traj, logLt, xs = sel(self.summ), sel(self.runs.traj), sel(self.runs.logLt), sel(self.runs.xstar)
        keys = host(self.runs.key).view(np.uint64)
        out = {}
        for i, r in enumerate(host(idx)):
            if self.noise is not None:
                z, u, ud = self.noise["z"][r], self.noise["u"][r], self.noise["ud"][r]
            else:
                z, u, ud = cr.device_noise(N, T, int(keys[r]))
            fk, trans = self.objs[r]
            out[int(r)] = rep.check_chain(fk, X[i], lw[i], A[i], summ[i], logLt[i], z, u,
                                          xstar=xs[i] if self.pin else None, traj=traj[i], ud=ud, trans=trans)
        assert rep.n_und <= 2 + 1e-3 * rep.n_draws, (rep.n_und, rep.n_draws)
        return rep, out


def _chains(c, extra=()):
    """The chains to replay: the first two, the last of the first wave, every chain past it (a CTA's second)."""
    return [0, min(1, c.R - 1), c.grid - 1] + list(range(c.grid, c.R)) + list(extra)


def _wave(m, kind, N):
    """The persistent grid at N when there are more chains than CTAs: one wave (the plan allocates nothing)."""
    runs = mcmc._CsmcRuns(m, kind, N, 1, 0.5, "genealogy")
    runs.R = 1 << 20
    return runs.plan()[1]


# ---------------------------------------------------------------------------------------------- N and chains
def _nmax():
    m = _tmap("LinearGauss", 2)
    return mcmc._CsmcRuns(m, _lib.FK_BOOTSTRAP, 1, 1, 0.5, "genealogy").plan()[0]


SIZES = [1, 2, 3, 255, 256, 511, 512, 513, 2047, 2048, 2049, 4097, "nmax-1", "nmax"]


@pytest.mark.parametrize("i,size", list(enumerate(SIZES)))
def test_sizes_and_chains(i, size):
    """LinearGauss at every N tier, R = grid + 3 chains with one whose sigmaY = inf makes every weight -inf (a CTA's
    second chain); a pin-off launch with the device's draws, then a pinned launch whose x* are the trajectories of
    the first.  ESSrmin cycles through 0.5, 1 and 0; the draw alternates."""
    nmax = _nmax()
    N = {"nmax-1": nmax - 1, "nmax": nmax}.get(size, size)
    T = 30 if N <= 2049 else 6
    essrmin = (0.5, 1.0, 0.0)[i % 3]
    draw = ("genealogy", "backward")[i % 2]
    m = _tmap("LinearGauss", T)
    grid = _wave(m, _lib.FK_BOOTSTRAP, N)
    R = grid + 3
    dead = grid + 1
    c = Case("LinearGauss", _lib.FK_BOOTSTRAP, N, R, T, essrmin, draw, names=("sigmaY",),
             special={dead: {"sigmaY": np.inf}})
    assert c.grid == grid and c.nmax == nmax
    passes, wt, st, per_cta = c.regime()
    assert per_cta >= 2
    assert passes == (1 if N <= 512 else 2 if N <= 1024 else -(-((N + 1) // 2) // BS))
    assert (passes >= 2) == (N >= 513)                 # a second pass of the pair loop from N = 513 on
    if N == 2048:
        assert (wt, st) == (1, 2)                     # the spacings' entry n opens a second tile
    if N >= 2049:
        assert wt >= 2 and st >= 2
    for pin in (False, True):
        if pin:
            c.pinned_from_previous()
        c.run(pin)
        rep, _ = c.check(_chains(c))
        assert rep.n_draws > 0
        # the dead chain: NaN summaries everywhere, trajectory index 0 at every step
        assert np.isnan(host(c.summ[dead, :, 0])).all() and np.isnan(c.runs.logLt[dead].item())
        if essrmin > 0 and N > 1:
            assert rep.n_rs > 0
        if essrmin == 0:
            assert rep.n_rs == 0


def test_above_the_bound_is_not_implemented():
    nmax = _nmax()
    m = _tmap("StochVol", 4)
    with pytest.raises(NotImplementedError):
        mcmc._CsmcRuns(m, _lib.FK_BOOTSTRAP, nmax + 1, 2, 0.5, "genealogy")
    mcmc._CsmcRuns(m, _lib.FK_BOOTSTRAP, nmax, 2, 0.5, "genealogy")


# ---------------------------------------------------------------------------------------------- models and kinds
def _built():
    out = []
    for name, (_, _, proposal, _) in _MAPS.items():
        out.append((name, _lib.FK_BOOTSTRAP))
        if proposal:
            out.append((name, _lib.FK_GUIDED))
    return out


@pytest.mark.parametrize("j,name,kind", [(j,) + nk for j, nk in enumerate(_built())])
def test_models_and_kinds(j, name, kind):
    """Every model and kind, with injected noise and then with the device's draws, pinned to the trajectories of an
    unconditional launch: ESSrmin and the draw mode vary across the cases."""
    N, R, T = 257, 6, 30
    essrmin = (0.5, 1.0, 0.0, 0.8)[j % 4]
    draw = ("backward", "genealogy")[j % 2]
    c = Case(name, kind, N, R, T, essrmin, draw, seed=11 + j)
    r = np.random.RandomState(j)
    noise = {"z": r.standard_normal((R, T, N)), "u": r.rand(R, T, N + 1), "ud": r.rand(R, T)}
    c.run(False, noise)
    rep, _ = c.check(range(R))
    c.pinned_from_previous()
    c.run(True, noise)
    rep, _ = c.check(range(R))
    c.run(True)
    rep2, _ = c.check(range(R))
    if essrmin > 0:
        assert rep.n_rs > 0 and rep2.n_rs > 0
    else:
        assert rep.n_rs == 0 and rep2.n_rs == 0


def test_per_chain_data_and_degenerate_rows():
    """Per-chain data rows (the regenerate_data layout), one with a NaN observation at T - 3: every slot's weight is
    -inf from there on while the earlier steps are finite, so the backward draws there see rows with no positive
    weight and must give 0.  Next to it: x* with a -inf state (logG = -inf), x* with a NaN state, u = 0 for every
    trajectory draw, and a zero among the spacing uniforms."""
    N, R, T = 300, 6, 30
    m = _tmap("StochVol", T)
    r = np.random.RandomState(5)
    data = r.standard_normal((R, T))
    data[2, T - 3] = np.nan
    for draw in ("backward", "genealogy"):
        c = Case("StochVol", _lib.FK_BOOTSTRAP, N, R, T, 0.7, draw, data2d=data, seed=3)
        noise = {"z": r.standard_normal((R, T, N)), "u": r.rand(R, T, N + 1), "ud": r.rand(R, T)}
        c.run(False, noise)
        c.pinned_from_previous()
        xs = c.runs.xstar.clone()
        xs[1, 4] = -np.inf
        xs[3, 7] = np.nan
        c.runs.xstar.copy_(xs)
        noise["ud"][4] = 0.0
        noise["u"][5, :, 17] = 0.0
        c.run(True, noise)
        rep, _ = c.check(range(R))
        summ = host(c.summ)
        assert np.isfinite(summ[2, :T - 3, 1]).all() and np.isnan(summ[2, T - 3:, 1]).all()
        assert np.isneginf(host(c.runs.lw[2, T - 1, :N])).all()
        if draw == "backward":
            assert rep.n_zero >= 2                     # rows T - 3, T - 4 ... of chain 2
        assert rep.n_u0 > 0                            # chain 5 resampled with an infinite spacing
        assert np.isneginf(host(c.runs.lw[1, 4, 0])) and np.isnan(host(c.runs.X[3, 7, 0]))


@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("essrmin", [0.0, 1.0])
def test_short_horizons(T, essrmin):
    for draw in ("genealogy", "backward"):
        c = Case("StochVol", _lib.FK_GUIDED, 33, 4, T, essrmin, draw, seed=T)
        c.run(False)
        c.check(range(4))
        c.pinned_from_previous()
        c.run(True)
        rep, _ = c.check(range(4))
        assert rep.n_rs == (T - 1 if essrmin == 1.0 else 0) * 4


# ---------------------------------------------------------------------------------------------- pin off: the bank
def _bank_tier(m, kind, N, R, essrmin):
    b = FilterBank(m.model, kind, "multinomial", N, R, as_device(m.data), m.n_params, essrmin,
                   shared_sc=None if m.shared_sc is None else as_device(m.shared_sc),
                   per_filter_sc=m.name == "Gordon_etal")
    return b, b.plan()[0]


@pytest.mark.parametrize("name,which", [("Gordon_etal", 2049), ("DiscreteCox", "nmax"), ("StochVol", "streaming")])
def test_pin_off_is_the_bank(name, which):
    """The unconditional pass gives the bits of FilterBank.advance with the same keys, at N = 2049, at nmax and at an
    N where the bank streams its filters from global memory (the csmc kernel has one tier)."""
    kind, T, essrmin = _lib.FK_BOOTSTRAP, 12, 0.99         # the last step resamples in some chains
    m = _tmap(name, T)
    nmax = _nmax()
    if which == "nmax":
        N = nmax
    elif which == "streaming":
        N = 6001
    else:
        N = which
    grid = _wave(m, kind, N)
    R = grid + 3
    c = Case(name, kind, N, R, T, essrmin, "genealogy")
    bank, tier = _bank_tier(m, kind, N, R, essrmin)
    if which == "streaming" or which == "nmax":
        assert tier == _lib.BATCH_STREAMING
    c.run(False)
    bank.params.copy_(c.runs.params)
    bank.key.copy_(c.runs.key)
    if bank.sc is not None:
        bank.sc.copy_(c.runs.sc)
    bsumm = torch.zeros_like(c.summ)
    A = torch.full((R, bank.ld), -1, dtype=torch.int64, device="cuda")
    bank.advance(T, restart=True, summaries=bsumm, A=A)
    assert torch.equal(c.summ, bsumm)
    assert torch.equal(c.runs.logLt, bank.logLt)
    last = (T - 1) & 1
    assert torch.equal(c.runs.X[:, T - 1, :N], bank.X[:, last, :N])
    assert torch.equal(c.runs.lw[:, T - 1, :N], bank.lw[:, :N])
    rs_last = host(c.summ[:, T - 1, 2]) > 0
    assert rs_last.any()
    for r in np.flatnonzero(rs_last):
        assert torch.equal(c.runs.A[r, T - 1, :N], A[r, :N])
    c.check([0, grid, R - 1])


# ---------------------------------------------------------------------------------------------- public layer
def test_public_csmc_is_the_replayed_launch():
    from particles_b200 import kalman, state_space_models as ssm
    T, N = 25, 1000
    y = [np.atleast_1d(v) for v in _data("LinearGauss", T, 5)]
    fk = ssm.Bootstrap(ssm=kalman.LinearGauss(rho=0.9, sigmaX=1.0, sigmaY=0.5), data=y)
    c0 = mcmc.CSMC(fk=fk, N=N, seed=3)
    c0.run()
    xstar = np.array([float(v) for v in c0.traj])
    c1 = mcmc.CSMC(fk=fk, N=N, xstar=list(xstar), seed=4)
    c1.run()
    runs = mcmc._CsmcRuns(c1._map, c1._kind, N, 1, 0.5, "genealogy")
    runs.set_rows(c1._row, _KeyCounter(4))
    runs.xstar[0] = as_device(xstar)
    summ = torch.zeros((1, T, 4), dtype=torch.float64, device="cuda")
    runs.run(True, summaries=summ)
    assert torch.equal(torch.stack(c1.hist.X), runs.X[0, :, :N])
    assert torch.equal(torch.stack(c1.hist.A), runs.A[0, :, :N])
    assert torch.equal(torch.stack([w.lw for w in c1.hist.wgts]), runs.lw[0, :, :N])
    assert np.array_equal(np.array(c1.traj), host(runs.traj[0])) and c1.logLt == runs.logLt[0].item()
    ofk = cr.chain_objects(c1._map, c1._row, False)[0][0]
    rep = cr.CsmcReplay(N, 0.5, True, "genealogy", **PHILOX)
    z, u, ud = cr.device_noise(N, T, int(host(runs.key).view(np.uint64)[0]))
    rep.check_chain(ofk, host(runs.X[0, :, :N]), host(runs.lw[0, :, :N]), host(runs.A[0, :, :N]), host(summ[0]),
                    runs.logLt[0].item(), z, u, xstar=xstar, traj=host(runs.traj[0]), ud=ud)
    assert rep.n_rs > 0


class _FixedTheta(mcmc.ParticleGibbs):
    def update_theta(self, theta, x):
        return theta


def test_particle_gibbs_backward_iteration_is_the_replayed_launch():
    from particles_b200 import distributions as dists, kalman
    T, K, N = 20, 5, 300
    th = dict(rho=0.9, sigmaX=1.0, sigmaY=0.5)
    y = _data("LinearGauss", T, 8)
    prior = dists.StructDist({k: dists.Normal(loc=v) for k, v in th.items()})
    theta0 = np.array([tuple(th.values())], dtype=[(k, float) for k in th])
    pg = _FixedTheta(niter=2, ssm_cls=kalman.LinearGauss, prior=prior, data=y, theta0=theta0, Nx=N,
                     backward_step=True, nchains=K, seed=2)
    pg.run()
    r = pg._runs
    X, lw, A, traj, logLt = (t.clone() for t in (r.X, r.lw, r.A, r.traj, r.logLt))
    assert np.array_equal(pg.x, host(traj))
    summ = torch.zeros((K, T, 4), dtype=torch.float64, device="cuda")
    r.run(True, summaries=summ)                        # the same launch again (same keys, rows and x*)
    assert torch.equal(r.X, X) and torch.equal(r.lw, lw) and torch.equal(r.A, A) and torch.equal(r.traj, traj)
    assert torch.equal(r.logLt, logLt)
    rows = mcmc._rows(pg.chain.theta[-1], pg.names)
    objs = cr.chain_objects(r.map, rows, False)
    rep = cr.CsmcReplay(N, 0.5, True, "backward", **PHILOX)
    keys = host(r.key).view(np.uint64)
    for k in range(K):
        z, u, ud = cr.device_noise(N, T, int(keys[k]))
        rep.check_chain(objs[k][0], host(X[k, :, :N]), host(lw[k, :, :N]), host(A[k, :, :N]), host(summ[k]),
                        logLt[k].item(), z, u, xstar=host(r.xstar[k]), traj=host(traj[k]), ud=ud, trans=objs[k][1])
