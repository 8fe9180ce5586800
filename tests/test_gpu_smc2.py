"""SMC^2 on the H100: the filter bank (csrc/smcb_bank.cu) against the batched filter and the single filter, its row
operations, and the sampler (smc_samplers.SMC2) against an exact answer and against the live reference's
statistics (tests/golden/golden_smc2.npz, tests/golden/make_golden_smc2.py)."""
import os
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_smc2.npz")
FK = {"boot": "Bootstrap", "guided": "GuidedPF", "apf": "AuxiliaryPF", "auxboot": "AuxiliaryBootstrap"}
SCHEMES = ["systematic", "stratified", "multinomial"]


def host(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _model(mname):
    from particles_b200 import kalman, state_space_models as ssm
    if mname == "sv":
        return ssm.StochVol, {"mu": (-1.2, -0.8), "rho": (0.9, 0.98), "sigma": (0.1, 0.3)}
    return kalman.LinearGauss, {"rho": (0.8, 0.95), "sigmaX": (0.5, 1.5), "sigmaY": (0.1, 0.5)}


def _setup(mname, R, T, seed=0):
    cls, ranges = _model(mname)
    rng = np.random.RandomState(seed)
    names = list(ranges)
    theta = np.stack([rng.uniform(*ranges[k], size=R) for k in names], axis=1)
    _, y = _simulate(mname, T, rng)
    return cls, names, theta, y


def _simulate(mname, T, rng):
    x = np.empty(T)
    if mname == "sv":
        x[0] = -1.0 + 0.2 / np.sqrt(1 - 0.95 ** 2) * rng.randn()
        for t in range(1, T):
            x[t] = -1.0 + 0.95 * (x[t - 1] + 1.0) + 0.2 * rng.randn()
        return x, np.exp(0.5 * x) * rng.randn(T)
    x[0] = rng.randn() / np.sqrt(1 - 0.81)
    for t in range(1, T):
        x[t] = 0.9 * x[t - 1] + rng.randn()
    return x, x + 0.3 * rng.randn(T)


def _bank(cls, names, theta, y, fk, scheme, N, keys, tier, essrmin=0.5):
    from particles_b200 import _lib, bank
    from particles_b200.device import as_device
    m = bank.ThetaMap(cls, names, y)
    kind = {"boot": _lib.FK_BOOTSTRAP, "guided": _lib.FK_GUIDED, "apf": _lib.FK_APF, "auxboot": _lib.FK_AUXBOOT}[fk]
    b = bank.FilterBank(m.model, kind, scheme, N, theta.shape[0], as_device(y), m.n_params, essrmin,
                        shared_sc=None if m.shared_sc is None else as_device(m.shared_sc),
                        per_filter_sc=m.step_consts(theta) is not None, tier=tier)
    b.set_rows(m.params(theta), m.step_consts(theta))
    b.key.copy_(torch.tensor(np.asarray(keys, dtype=np.uint64).view(np.int64)))
    return b


def _rows(b):
    return {k: host(getattr(b, k)).copy() for k in ("X", "lw", "state", "params", "key")}


@pytest.mark.parametrize("tier", ["resident", "streaming"])
@pytest.mark.parametrize("mname,fkname", [(m, f) for m in ("sv", "lg") for f in FK])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_split_invariance(mname, fkname, scheme, tier):
    """advance(0, t) then advance(t, T) == advance(0, T) == the batched filter (k_batch) with the same seeds, bit for
    bit: the last generation, the weights, logLt, every resampling flag and ESS, and the final ancestors; for
    t = 1, a split right after a step that decided to resample, and T - 1."""
    from particles_b200 import core, state_space_models as ssm
    N, T, R = 301, 40, 6
    cls, names, theta, y = _setup(mname, R, T)
    keys = [101 + 17 * r for r in range(R)]
    summ = torch.zeros((R, T, 4), dtype=torch.float64, device="cuda")
    A = torch.zeros((R, N + 1), dtype=torch.int64, device="cuda")
    one = _bank(cls, names, theta, y, fkname, scheme, N, keys, tier)
    one.advance(T, summaries=summ, A=A)
    table = host(summ)
    kws = [dict(fk=getattr(ssm, FK[fkname])(ssm=cls(**dict(zip(names, theta[r]))), data=list(y)), N=N,
                resampling=scheme) for r in range(R)]
    runs = core.run_batch(kws, keys, tier=tier)
    last = (T - 1) & 1
    for r, run in enumerate(runs):
        assert np.array_equal(run._table, table[r]), r
        assert np.array_equal(host(run.X), host(one.X[r, last, :N])), r
        assert np.array_equal(host(run.wgts.lw), host(one.lw[r, :N])), r
        if run.rs_flag:
            assert np.array_equal(host(run.A), host(A[r, :N])), r
    assert np.array_equal(host(one.logLt), table[:, -1, 1])
    rs_any = np.flatnonzero(table[:, 1:, 2].any(axis=0))
    splits = {1, T - 1} | ({int(rs_any[0]) + 1} if rs_any.size else set())
    for t in sorted(splits):
        b = _bank(cls, names, theta, y, fkname, scheme, N, keys, tier)
        s2 = torch.zeros_like(summ)
        b.advance(t, summaries=s2)
        b.advance(T, summaries=s2)
        assert np.array_equal(host(s2), table), t
        for k in ("lw", "state"):
            assert np.array_equal(host(getattr(b, k))[:, :N], host(getattr(one, k))[:, :N]), (t, k)
        assert np.array_equal(host(b.X[:, last, :N]), host(one.X[:, last, :N])), t


def test_one_filter_per_theta():
    """R filters with R distinct theta against R single SMC(fk=Bootstrap(StochVol(**theta_r)), seed=s_r) runs: >= 90 %
    agree in every flag and final ancestor, and on those logLt agrees to 1e-12 relative."""
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    N, T, R = 500, 50, 16
    cls, names, theta, y = _setup("sv", R, T, seed=4)
    keys = [7000 + 3 * r for r in range(R)]
    b = _bank(cls, names, theta, y, "boot", "systematic", N, keys, "auto")
    summ = torch.zeros((R, T, 4), dtype=torch.float64, device="cuda")
    A = torch.zeros((R, N), dtype=torch.int64, device="cuda")
    b.advance(T, summaries=summ, A=A)
    table = host(summ)
    agree = 0
    for r in range(R):
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=cls(**dict(zip(names, theta[r]))), data=list(y)), N=N, seed=keys[r])
        pf.run()
        same = pf.summaries.rs_flags == [bool(v) for v in table[r, :, 2]] and (
            not pf.rs_flag or np.array_equal(host(pf.A), host(A[r])))
        if same:
            agree += 1
            np.testing.assert_allclose(table[r, -1, 1], pf.logLt, rtol=1e-12)
    assert agree >= 0.9 * R, agree


@pytest.mark.parametrize("tier", ["resident", "streaming"])
def test_inactive_filters_untouched(tier):
    N, T, R = 200, 30, 10
    cls, names, theta, y = _setup("lg", R, T)
    b = _bank(cls, names, theta, y, "boot", "multinomial", N, range(1, R + 1), tier)
    b.advance(5)
    before = _rows(b)
    idx = torch.tensor([1, 4, 7], dtype=torch.int64, device="cuda")
    b.advance(20, idx=idx)
    after = _rows(b)
    st = after["state"]
    assert np.all(st[[1, 4, 7], 0] == 20) and np.all(np.delete(st[:, 0], [1, 4, 7]) == 5)
    for k in before:
        for r in range(R):
            if r not in (1, 4, 7):
                assert np.array_equal(before[k][r], after[k][r]), (k, r)
    b.advance(3, idx=idx)                        # already beyond t1: nothing changes
    assert all(np.array_equal(after[k], v) for k, v in _rows(b).items())


def test_gather_keys_and_continuation():
    """X[A]: every row bit-copied, the first copy of an ancestor keeps its key and continues exactly as the ancestor,
    later copies get fresh keys (no two filters share one) and diverge."""
    N, T, R = 256, 30, 8
    cls, names, theta, y = _setup("sv", R, T)
    b = _bank(cls, names, theta, y, "boot", "systematic", N, range(11, 11 + R), "auto")
    b.advance(10)
    A = torch.tensor([0, 0, 3, 3, 3, 5, 6, 6], dtype=torch.int64, device="cuda")
    g = b.gather(A, seed=1234, counter=500)
    src, dst = _rows(b), _rows(g)
    a = host(A)
    for k in ("X", "lw", "state", "params"):
        assert np.array_equal(dst[k], src[k][a]), k
    assert len(set(dst["key"].tolist())) == R
    first = [0, 2, 5, 6]
    assert np.array_equal(dst["key"][first], src["key"][a[first]])
    b.advance(T)
    g.advance(T)
    lb, lg_ = host(b.logLt), host(g.logLt)
    assert np.array_equal(lg_[first], lb[a[first]])
    for i in (1, 3, 4, 7):
        assert lg_[i] != lb[a[i]], i


def test_merge_and_keys():
    N, T, R = 128, 20, 12
    cls, names, theta, y = _setup("lg", R, T)
    cur = _bank(cls, names, theta, y, "boot", "systematic", N, range(R), "auto")
    prop = _bank(cls, names, theta[::-1].copy(), y, "boot", "systematic", N, range(100, 100 + R), "auto")
    cur.advance(8)
    prop.fresh_keys(seed=9, counter=0)
    keys = host(prop.key)
    assert len(set(keys.tolist())) == R
    prop.advance(8)
    acc = torch.tensor([1, 0, 1, 1, 0, 0, 0, 1, 0, 1, 1, 0], dtype=torch.uint8, device="cuda")
    c0, p0 = _rows(cur), _rows(prop)
    cur.merge(prop, acc)
    c1 = _rows(cur)
    m = host(acc).astype(bool)
    for k in c0:
        assert np.array_equal(c1[k][m], p0[k][m]) and np.array_equal(c1[k][~m], c0[k][~m]), k


# ---------------------------------------------------------------------------------------------- the sampler
def _lg_exact(y, grid, a, b):
    """log p(y_0:t) for every t and the posterior mean / sd of sigmaY at T, by a Kalman filter on a fine grid of
    sigmaY (LinearGauss rho = 0.9, sigmaX = 1, sigma0 = sigmaX / sqrt(1 - rho^2)) and a Gamma(a, b) prior."""
    from scipy import stats
    T = len(y)
    ll = np.zeros((grid.size, T))
    m, P = np.zeros(grid.size), np.full(grid.size, 1.0 / (1 - 0.81))
    for t in range(T):
        if t > 0:
            m, P = 0.9 * m, 0.81 * P + 1.0
        S = P + grid ** 2
        ll[:, t] = stats.norm.logpdf(y[t], loc=m, scale=np.sqrt(S))
        K = P / S
        m, P = m + K * (y[t] - m), (1 - K) * P
    cum = np.cumsum(ll, axis=1)
    lw = cum + stats.gamma.logpdf(grid, a, scale=1.0 / b)[:, None]
    dx = grid[1] - grid[0]
    mx = lw.max(axis=0)
    evid = mx + np.log(np.exp(lw - mx).sum(axis=0) * dx)
    w = np.exp(lw[:, -1] - mx[-1])
    w /= w.sum()
    mean = float((w * grid).sum())
    return evid, mean, float(np.sqrt((w * (grid - mean) ** 2).sum()))


def _smc2_runs(y, seeds, N, **kw):
    import particles_b200 as pb
    from particles_b200 import distributions as dists, kalman, smc_samplers as ss
    out = []
    for s in seeds:
        fk = ss.SMC2(ssm_cls=kalman.LinearGauss, prior=dists.StructDist({"sigmaY": dists.Gamma(a=2.0, b=4.0)}),
                     data=y, **kw)
        torch.manual_seed(s)                    # the Gamma prior draws from torch's generator
        pf = pb.SMC(fk=fk, N=N, seed=s)
        pf.run()
        post = float(torch.sum(pf.W * pf.X.theta_dev[:, 0]))
        out.append((np.array(pf.summaries.logLts), post, list(pf.X.shared["Nxs"]), pf))
    return out


@pytest.mark.parametrize("cfg", ["std", "wf", "exch"])
def test_exact_answer(cfg):
    """LinearGauss with sigmaY unknown (Gamma(2, 4) prior), T = 100: 8 runs of SMC^2 (N = 1000, or 200 chains of
    10 waste-free, len_chain = 10) against the exact evidence trajectory and posterior mean from a Kalman filter on a
    grid of 20001 values of sigmaY.  The standard error comes from the runs' spread; log-evidence estimates are biased
    low by about var / 2 (Jensen), so the bound is 3 SE + var / 2 at t in {9, 49, 99}; the posterior mean within
    3 SE + 0.002 (grid quadrature).  Calibration: smaller samplers (N = 300, len_chain = 5, or the exchange run
    started at Nx = 20) are biased by more than this bound -- the posterior mean by about 0.02 (0.16 posterior sd),
    the evidence of a run started at Nx = 20 by about -0.2."""
    rng = np.random.RandomState(5)
    _, y = _simulate("lg", 100, rng)
    grid = np.linspace(1e-4, 2.0, 20001)
    evid, mean, sd = _lg_exact(y, grid, 2.0, 4.0)
    kw = {"std": dict(wastefree=False, len_chain=10), "wf": dict(wastefree=True, len_chain=10),
          "exch": dict(wastefree=False, len_chain=10, init_Nx=50, ar_to_increase_Nx=0.35)}[cfg]
    runs = _smc2_runs(y, range(1, 9), 1000 if cfg != "wf" else 200, init_Nx=kw.pop("init_Nx", 100), **kw)
    ll = np.array([r[0] for r in runs])
    post = np.array([r[1] for r in runs])
    for t in (9, 49, 99):
        v = ll[:, t].var(ddof=1)
        se = np.sqrt(v / len(runs))
        assert abs(ll[:, t].mean() - evid[t]) < 3 * se + v / 2 + 1e-3, (t, ll[:, t].mean(), evid[t], se)
    se = post.std(ddof=1) / np.sqrt(len(runs))
    assert abs(post.mean() - mean) < 3 * se + 0.002, (post.mean(), mean, se, sd)
    if cfg == "exch":
        assert all(max(r[2]) > 50 for r in runs)             # the exchange step ran
        assert all(r[3].X.bank.N == r[2][-1] for r in runs)
    else:
        assert all(set(r[2]) == {100} for r in runs)


@pytest.mark.parametrize("cfg", ["std", "wf", "exch"])
def test_against_reference(golden, cfg):
    """Same configuration as tests/golden/make_golden_smc2.py: the means of logLt (t in {9, 29, 49}) and of the
    posterior mean of sigmaY agree with the live reference's within 3 sigma of the combined spread."""
    from particles_b200 import distributions as dists  # noqa: F401
    y = golden["data"]
    kw = {"std": dict(wastefree=False), "wf": dict(wastefree=True),
          "exch": dict(wastefree=False, init_Nx=20, ar_to_increase_Nx=1.0)}[cfg]
    runs = _smc2_runs(y, range(1, 17), 200, len_chain=5, init_Nx=kw.pop("init_Nx", 50), **kw)
    ll = np.array([r[0] for r in runs])
    post = np.array([r[1] for r in runs])
    ref_ll, ref_post = golden[cfg + "/logLts"], golden[cfg + "/post_mean"]
    for mine, theirs in [(ll[:, t], ref_ll[:, t]) for t in (9, 29, 49)] + [(post, ref_post)]:
        se = np.sqrt(mine.var(ddof=1) / mine.size + theirs.var(ddof=1) / theirs.size)
        assert abs(mine.mean() - theirs.mean()) < 3 * se + 1e-9, (mine.mean(), theirs.mean(), se)


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return len([x for x in w if "synchroniz" in str(x.message)])


def test_determinism_and_syncs():
    """The same seed gives the same bits twice, another seed other bits; host syncs: at most 2 per SMC^2 step
    without a move (the ESS test, and the logLt of the summaries), and a bounded number per MCMC step."""
    import particles_b200 as pb
    from particles_b200 import distributions as dists, kalman, smc_samplers as ss
    rng = np.random.RandomState(5)
    _, y = _simulate("lg", 40, rng)

    def run(seed, log=None):
        fk = ss.SMC2(ssm_cls=kalman.LinearGauss, prior=dists.StructDist({"sigmaY": dists.Uniform(a=0.05, b=1.0)}),
                     data=y, init_Nx=50, len_chain=4)
        pf = pb.SMC(fk=fk, N=100, seed=seed)
        moves = []
        orig = fk.move.mcmc.step
        fk.move.mcmc.step = lambda x, target: moves.append(1) or orig(x, target)
        n = _count_syncs(pf.run)
        if log is not None:
            log.append((n, len(moves)))
        return np.array(pf.summaries.logLts), host(pf.X.theta_dev), host(pf.X.bank.X)

    log = []
    a, b, c = run(3, log), run(3), run(4)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
    assert not np.array_equal(a[0], c[0])
    syncs, mh = log[0]
    T = len(y)
    assert syncs <= 2 * T + 8 * mh, (syncs, mh)


def test_book_configuration_runs(golden):
    """The book's StochVolLeverage example on the GBP/USD returns, truncated to 60 observations: pf.X.theta['rho'],
    shared['Nxs'] and summaries.logLts behave as the reference's."""
    import particles_b200 as pb
    from particles_b200 import distributions as dists, smc_samplers as ss, state_space_models as ssm
    prior = dists.StructDist({"mu": dists.Normal(scale=2.0), "sigma": dists.Gamma(a=2.0, b=2.0),
                              "rho": dists.Beta(a=9.0, b=1.0), "phi": dists.Uniform(a=-1.0, b=1.0)})
    y = golden["gbp_usd"][:60]
    torch.manual_seed(0)
    fk = ss.SMC2(ssm_cls=ssm.StochVolLeverage, prior=prior, data=y, init_Nx=100, ar_to_increase_Nx=0.1,
                 wastefree=False, len_chain=6)
    pf = pb.SMC(fk=fk, N=500, seed=1)
    pf.run()
    th = pf.X.theta
    assert th.dtype.names == ("mu", "phi", "rho", "sigma") and th["rho"].shape == (500,)
    assert np.all((th["rho"] > 0) & (th["rho"] < 1)) and np.all(np.abs(th["phi"]) <= 1)
    assert len(pf.X.shared["Nxs"]) == 60 and pf.X.shared["Nxs"][0] == 100
    assert len(pf.summaries.logLts) == 60 and np.all(np.isfinite(pf.summaries.logLts))
    assert pf.X.bank.N == pf.X.shared["Nxs"][-1]
    assert "Nx=" in str(pf)
    m = fk.default_moments(pf.W, pf.X)
    assert m["mean"].dtype.names == th.dtype.names


REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")


def _stand_in():
    """particles / particles.core / particles.smc_samplers / particles.state_space_models with the reference's names:
    an SMC2 object with the reference's attributes, and StochVol."""
    import types
    mods = {n: types.ModuleType(n) for n in ("particles", "particles.core", "particles.smc_samplers",
                                             "particles.state_space_models")}

    class SMC:
        def __init__(self, *a, **k):
            raise RuntimeError("the stand-in reference has no engine")

    class StochVol:
        pass

    class Bootstrap:
        pass

    class AdaptiveMCMCSequence:
        def __init__(self, len_chain=10):
            self.nsteps = len_chain - 1

    class SMC2:
        def __init__(self, ssm_cls=None, prior=None, data=None, smc_options=None, fk_cls=None, init_Nx=100,
                     ar_to_increase_Nx=-1.0, wastefree=True, len_chain=10):
            self.smc_options = {"collect": "off"}
            self.smc_options.update(smc_options or {})
            self.ssm_cls, self.prior, self.data, self.init_Nx = ssm_cls, prior, data, init_Nx
            self.fk_cls = Bootstrap if fk_cls is None else fk_cls
            self.ar_to_increase_Nx, self.wastefree, self.len_chain = ar_to_increase_Nx, wastefree, len_chain
            self.move = AdaptiveMCMCSequence(len_chain=len_chain)

    for cls, mod in ((SMC, "particles.core"), (StochVol, "particles.state_space_models"),
                     (Bootstrap, "particles.state_space_models"), (SMC2, "particles.smc_samplers"),
                     (AdaptiveMCMCSequence, "particles.smc_samplers")):
        cls.__module__ = mod
        setattr(mods[mod], cls.__name__, cls)
    pkg = mods["particles"]
    pkg.core, pkg.smc_samplers, pkg.state_space_models, pkg.SMC = (mods["particles.core"], mods["particles.smc_samplers"],
                                                                    mods["particles.state_space_models"], SMC)
    pkg.__path__ = []
    return mods


@pytest.fixture()
def reference():
    import sys
    saved = {k: v for k, v in sys.modules.items() if k == "particles" or k.startswith("particles.")}
    for k in saved:
        del sys.modules[k]
    live = os.path.isdir(os.path.join(REF, "particles"))
    if live:
        sys.path.insert(0, REF)
    else:
        sys.modules.update(_stand_in())
    import particles
    yield particles, live
    for k in [k for k in sys.modules if k == "particles" or k.startswith("particles.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    if live:
        sys.path.remove(REF)


def test_install_runs_reference_smc2(reference, golden):
    """After install(), the reference's SMC2 object handed to particles.SMC runs on the filter bank."""
    import particles_b200 as pb
    from particles_b200 import distributions as dists, smc_samplers as ss
    particles, live = reference
    import particles.smc_samplers as rss
    import particles.state_space_models as rssm
    prior = dists.StructDist({"mu": dists.Normal(scale=2.0), "sigma": dists.Gamma(a=2.0, b=2.0),
                              "rho": dists.Beta(a=9.0, b=1.0)})
    fk = rss.SMC2(ssm_cls=rssm.StochVol, prior=prior, data=golden["gbp_usd"][:40], init_Nx=50,
                  ar_to_increase_Nx=0.1, wastefree=False, len_chain=4)
    uninstall = pb.install()
    try:
        torch.manual_seed(0)
        pf = particles.SMC(fk=fk, N=200, seed=2) if not live else particles.SMC(fk=fk, N=200)
        pf.run()
    finally:
        uninstall()
    assert isinstance(pf, pb.SMC) and isinstance(pf.fk, ss.SMC2)
    assert isinstance(pf.X, ss.SMC2Particles) and pf.X.theta["rho"].shape == (200,)
    assert len(pf.summaries.logLts) == 40 and np.isfinite(pf.logLt)
    assert ss.from_reference_smc2(ss.SMC2) is None           # anything else keeps its path
