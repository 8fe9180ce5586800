"""The fused step kernel at the sizes where all its branches run, step by step against a high-precision replay
(tests/step_replay.py), and the batched filter and the filter bank past one scan tile.

The step kernel's grid is one CTA per SM, each owning a contiguous range of pairs (smcb_filter.cu), so its
size-dependent branches -- the slab schedule of the streaming pass, the 8 pipelined scan groups and their 32-slot
prefix ring, the unstaged scatter with its heavy-entry queue, the double-buffered multinomial tiles and their
uncovered-tile search, the hint repair of the counted move -- only run when every CTA owns many particles.  Each case
below asserts the regime it is meant to reach on the device that runs it.  The filter is stepped one step at a time
(a fused pair never crosses a batch boundary) and its buffers are read after every step; the same filter run in one
``step(T)`` with fused pairs must then leave the same bits."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import smc_numpy as orc  # noqa: E402
import philox_ref  # noqa: E402
from step_replay import StepReplay, step_grid  # noqa: E402

SCAN_TILE, OUT_TILE, HINT_CAP, HEAVY, GROUP_Q, STAGE = 512, 1024, 2048, 48, 8, 4096
U_TOP = 1.0 - 2.0 ** -53


def host(t):
    return t.detach().cpu().numpy()


def lst(y):
    return [np.atleast_1d(v) for v in y]


def n_sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def size(name):
    g = min(n_sm(), 256)
    return {"full": 1024 * g + 3, "full_even": 1024 * g + 4, "1e6": 1_000_003, "1e6_even": 1_000_002,
            "ring": int(1.4 * 16384 * g) | 1}[name]


def assert_regime(name, N):
    """The size reaches the branches it is meant for on this device."""
    g, chunk = step_grid(N, n_sm())
    entries = 2 * chunk
    assert g == min(n_sm(), 256), (name, N, g)                      # a full grid
    if name.startswith("full"):
        assert -(-entries // OUT_TILE) == 2, (name, N, chunk)        # two output tiles per CTA
    elif name.startswith("1e6"):
        assert entries // SCAN_TILE > 8 and entries // OUT_TILE > 2, (name, N, chunk)   # every scan group, several tiles
    else:
        assert -(-entries // SCAN_TILE) > 32, (name, N, chunk)       # the prefix ring wraps
    return chunk


def models(golden):
    from particles_b200 import kalman, state_space_models as ssm
    mv = golden["data/mvlg_seed5_T30"]
    out = {
        "sv": (ssm.StochVol(), orc.StochVol(), lst(golden["data/sv_seed1_T1000"][:20]), None),
        "lg": (kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
               lst(golden["data/lg_seed2_T100"][:20]), None),
        "gordon": (ssm.Gordon_etal(), orc.Gordon_etal(), lst(golden["data/gordon_seed3_T50"][:20]), None),
        "thetalog": (ssm.ThetaLogistic(), orc.ThetaLogistic(), lst(golden["data/thetalogistic_seed4_T50"][:20]), None),
        "cox": (ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), orc.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9),
                lst(golden["data/cox_seed6_T60"][:20]), None),
        "svlev": (ssm.StochVolLeverage(phi=-0.6), orc.StochVolLeverage(phi=-0.6), lst(golden["data/svlev_seed7_T60"][:20]),
                  None),
        "bearings": (ssm.BearingsOnly(), orc.BearingsOnly(), list(golden["data/bearings_seed0_T40"].reshape(-1, 1)[:20]), 2),
    }
    for d in (2, 3, 4):
        out[f"mvlg{d}"] = (kalman.MVLinearGauss_Guarniero_etal(0.4, d), orc.MVLinearGauss_Guarniero_etal(0.4, d),
                           [np.ascontiguousarray(v[:d]) for v in mv], d)
    return out


FK = {"boot": "Bootstrap", "guided": "GuidedPF", "apf": "AuxiliaryPF", "auxboot": "AuxiliaryBootstrap"}


def host_uniforms(scheme, N, t, seed):
    """The uniforms the device's Philox stream gives step t, as the reference consumes them."""
    if scheme == "systematic":
        return philox_ref.uniforms(2, t, seed)[:1]
    return philox_ref.uniforms(N if scheme == "stratified" else N + 1, t, seed)


def host_normals(N, t, seed, nz):
    if nz is None:
        return philox_ref.normals(N, t, seed)
    return np.stack([philox_ref.normals(N, t, seed, comp=c) for c in range(nz)], axis=1)


def engine_out(e):
    return {"summ": e.summ.clone(), "X0": e.X[0].clone(), "X1": e.X[1].clone(), "lw0": e.lw[0].clone(),
            "lw1": e.lw[1].clone(), "A": e.A.clone()}


def replay_run(monkeypatch, dev_m, orc_m, y, nz, fkname, scheme, essrmin, N, T, chunk, noise=None, seed=77,
               x_exact=False, keep=False):
    """Step a fused filter one step at a time and check every step against the replay; then the production schedule
    (one step(T), SMCB_FUSE = 1 and 2) must leave the same buffers.  ``noise``: None (device Philox with ``seed``) or
    (z, u) in the layout of SMC(noise=...).  Returns the per-step results of the replay (with ``keep``, a resampling
    step's offspring counts, ancestors, grid points and CDF too) and the replay."""
    from particles_b200 import state_space_models as ssm
    from particles_b200.core import _FusedEngine
    fk_d = getattr(ssm, FK[fkname])(ssm=dev_m, data=y[:T])
    fk_o = getattr(orc, FK[fkname])(orc_m, y[:T])
    spec = ssm.fused_spec(fk_d)
    assert spec is not None
    tol = dict(x_rtol=1e-13, x_atol=1e-14) if noise is not None else dict(x_rtol=1e-12, x_atol=1e-12)
    rep = StepReplay(fk_o, N, scheme, essrmin, chunk=chunk, x_exact=x_exact, **tol)
    nu = {"systematic": 1, "stratified": N, "multinomial": N + 1}[scheme]

    def noise_of(t):
        if noise is None:
            return host_normals(N, t, seed, nz), (host_uniforms(scheme, N, t, seed) if t > 0 else None)
        z, u = noise
        return (z[t] if nz is None else z[t].T), u[t][:nu]

    monkeypatch.setenv("SMCB_FUSE", "1")
    e = _FusedEngine(spec, N, scheme, essrmin, seed, noise=noise)
    e.A.zero_()
    steps = []
    with np.errstate(all="ignore"):
        for t in range(T):
            e.step(1)
            X = host(e.X[t & 1])
            X = X if X.ndim == 1 else np.ascontiguousarray(X.T)
            lw = host(e.lw[t & 1])
            summ = host(e.summ)
            z, u = noise_of(t)
            if t == 0:
                rep.check_init(z, X, lw)
                steps.append({"rs": False})
            else:
                rs = summ[t, 2] != 0
                out = rep.check_step(t, Xp, lwp, summ, z, u, X, lw,
                                     A=host(e.A) if rs else None, cdf=host(e.cdf) if rs else None,
                                     scratch=host(e.scratch) if rs and scheme == "multinomial" else None)
                if rs and keep:
                    scr = host(e.scratch) if scheme == "multinomial" else None
                    out["A"], out["su"], out["cdf"] = host(e.A), rep.grid_points(u, scr), host(e.cdf)
                steps.append({k: v for k, v in out.items() if keep and k not in ("X", "lw")} | {"rs": rs})
            Xp, lwp = X, lw
        rep.check_last(T, Xp, lwp, summ)
    torch.cuda.synchronize()
    ref = engine_out(e)
    e.close()
    for mode in (1, 2):
        monkeypatch.setenv("SMCB_FUSE", str(mode))
        f = _FusedEngine(spec, N, scheme, essrmin, seed, noise=noise)
        f.A.zero_()
        f.step(T)
        torch.cuda.synchronize()
        out = engine_out(f)
        f.close()
        for k in ref:
            assert torch.equal(out[k], ref[k]), f"SMCB_FUSE={mode}: {k} differs from the stepped run"
    return steps, rep


# model, Feynman-Kac kind, scheme, ESSrmin, size, noise ("inj" or "philox")
_SV = [("sv", fk, sch, (0.8, 1.0)[i % 2], "full", ("inj", "philox")[(i // 2) % 2])
       for i, (fk, sch) in enumerate((fk, sch) for fk in FK for sch in ("systematic", "stratified", "multinomial"))]
CASES = _SV + [
    ("lg", "boot", "stratified", 0.8, "full", "inj"), ("lg", "guided", "multinomial", 1.0, "full", "philox"),
    ("lg", "apf", "systematic", 0.8, "full", "inj"), ("gordon", "boot", "multinomial", 0.8, "full", "inj"),
    ("thetalog", "boot", "systematic", 1.0, "full", "philox"), ("cox", "boot", "stratified", 0.8, "full", "inj"),
    ("svlev", "boot", "multinomial", 0.8, "full", "philox"), ("mvlg2", "guided", "systematic", 0.8, "full", "inj"),
    ("mvlg3", "apf", "stratified", 0.8, "full_even", "philox"), ("mvlg4", "guided", "multinomial", 1.0, "full_even", "inj"),
    ("bearings", "boot", "systematic", 0.8, "full", "inj"),
    # about 15 scan tiles and 8 multinomial output tiles per CTA
    ("sv", "boot", "systematic", 0.8, "1e6", "philox"), ("sv", "guided", "stratified", 1.0, "1e6", "inj"),
    ("sv", "apf", "multinomial", 0.8, "1e6", "philox"), ("sv", "auxboot", "stratified", 0.8, "1e6", "inj"),
    ("lg", "boot", "multinomial", 1.0, "1e6", "inj"), ("lg", "guided", "systematic", 0.8, "1e6", "philox"),
    ("lg", "apf", "stratified", 0.8, "1e6", "inj"), ("gordon", "boot", "systematic", 0.8, "1e6", "philox"),
    ("thetalog", "boot", "multinomial", 0.8, "1e6", "inj"), ("cox", "boot", "stratified", 1.0, "1e6", "philox"),
    ("svlev", "boot", "systematic", 0.8, "1e6", "inj"), ("mvlg2", "apf", "stratified", 0.8, "1e6", "inj"),
    ("mvlg3", "guided", "multinomial", 0.8, "1e6_even", "philox"), ("mvlg4", "apf", "systematic", 0.8, "1e6", "inj"),
    ("bearings", "boot", "stratified", 0.8, "1e6_even", "philox"),
    # more than 32 scan tiles per CTA: the prefix ring wraps
    ("sv", "boot", "systematic", 1.0, "ring", "philox"), ("sv", "boot", "stratified", 0.8, "ring", "inj"),
    ("sv", "boot", "multinomial", 1.0, "ring", "inj"),
]
T_OF = {"full": 12, "full_even": 12, "1e6": 10, "1e6_even": 10, "ring": 8}


def _id(c):
    return "-".join(str(v) for v in c)


@pytest.mark.parametrize("mname,fkname,scheme,essrmin,sname,src", CASES, ids=[_id(c) for c in CASES])
def test_fused_step_vs_replay(golden, monkeypatch, mname, fkname, scheme, essrmin, sname, src):
    N, T = size(sname), T_OF[sname]
    chunk = assert_regime(sname, N)
    dev_m, orc_m, y, nz = models(golden)[mname]
    noise = None
    if src == "inj":
        r = np.random.RandomState(N % 1000 + T)
        z = r.standard_normal((T, N) if nz is None else (T, nz, N))
        noise = (z, r.rand(T, N + 1))
    steps, rep = replay_run(monkeypatch, dev_m, orc_m, y, nz, fkname, scheme, essrmin, N, T, chunk, noise=noise,
                            x_exact=(mname == "sv" and fkname == "boot" and src == "inj"))
    if essrmin == 1.0:          # every step but one where all weights are equal (ESS = N: the guided filters' step 0)
        assert rep.n_rs >= T - 2


# ------------------------------------------------------------------------------------------ degenerate weights
def tile_ids(N, chunk, tile):
    """Per entry (or output) index: the id of its tile of `tile` entries, counted from the start of its CTA's range."""
    i = np.arange(N)
    per = 2 * chunk
    b = i // per
    return b * (-(-per // tile)) + (i - b * per) // tile


def scatter_regimes(counts, N, chunk):
    """(largest number of outputs one scan tile owns, largest number of entries with more than kHeavy offspring in
    one scan tile)."""
    ids = tile_ids(N, chunk, SCAN_TILE)
    return int(np.bincount(ids, weights=counts).max()), int(np.bincount(ids, weights=counts > HEAVY).max())


def widest_output_tile(A, N, chunk):
    """The largest span of CDF entries one multinomial output tile searches (A is non-decreasing)."""
    ids = tile_ids(N, chunk, OUT_TILE)
    starts = np.flatnonzero(np.r_[True, ids[1:] != ids[:-1]])
    ends = np.r_[starts[1:], N] - 1
    return int((A[ends] - A[starts] + 1).max())


def sharp_lg(sigmaY):
    from particles_b200 import kalman
    kw = dict(sigmaX=1.0, sigmaY=sigmaY, rho=0.9)
    return kalman.LinearGauss(**kw), orc.LinearGauss(**kw)


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_scattered_survivors(golden, monkeypatch, scheme):
    """A sharp observation density (sigma_Y = 1e-4) over particles in random order: a few hundred of 1e6 keep a
    non-zero weight, between long runs of zero weights; one step has an outlying observation, so one entry takes
    (nearly) every output.  Unstaged scatter, heavy entries, galloping hint repairs and uncovered multinomial tiles."""
    N, T = size("1e6"), 6
    chunk = assert_regime("1e6", N)
    dev_m, orc_m = sharp_lg(1e-4)
    y = lst([0.0, 0.3, -0.5, 4.0, 0.1, 0.0])
    r = np.random.RandomState(3)
    noise = (r.standard_normal((T, N)), r.rand(T, N + 1))
    steps, rep = replay_run(monkeypatch, dev_m, orc_m, y, None, "boot", scheme, 0.5, N, T, chunk, noise=noise,
                            keep=True)
    assert rep.n_rs == T - 1
    outs, heavy = zip(*[scatter_regimes(s["counts"], N, chunk) for s in steps if s["rs"]])
    assert max(outs) > HINT_CAP                                   # a tile too long for the hint buffer
    assert min(int((s["counts"] > 0).sum()) for s in steps if s["rs"]) < 1000
    if scheme == "multinomial":
        assert max(widest_output_tile(s["A"], N, chunk) for s in steps if s["rs"]) > STAGE   # uncovered tile


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_contiguous_survivors(golden, monkeypatch, scheme):
    """Particles sorted at step 0 and moved without noise stay sorted: the mass sits in one contiguous window, and
    more than kGroupQ entries with more than kHeavy offspring each share one scan tile (the heavy queue overflows)."""
    N, T = size("1e6"), 6
    chunk = assert_regime("1e6", N)
    dev_m, orc_m = sharp_lg(1e-3)
    y = lst([0.3 * 0.9 ** t for t in range(T)])
    r = np.random.RandomState(4)
    z = np.zeros((T, N))
    z[0] = np.sort(r.standard_normal(N))
    noise = (z, r.rand(T, N + 1))
    steps, rep = replay_run(monkeypatch, dev_m, orc_m, y, None, "boot", scheme, 0.5, N, T, chunk, noise=noise,
                            keep=True)
    assert rep.n_rs > 0
    regimes = [scatter_regimes(s["counts"], N, chunk) for s in steps if s["rs"]]
    assert any(o > HINT_CAP and h > GROUP_Q for o, h in regimes), regimes


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_near_equal_weights(golden, monkeypatch, scheme):
    """All particles equal but the last, whose weight underflows to exactly 0: N - 1 equal CDF steps, ESS = N - 1, so
    ESSrmin = 1 resamples every step.  The uniforms are the extreme ones (0 and 1 - 2^-53) or, on odd steps, chosen
    so that every grid point lands on a CDF entry up to rounding: searchsorted's 'left' ties, bit for bit."""
    N, T = size("1e6"), 6
    chunk = assert_regime("1e6", N)
    dev_m, orc_m = sharp_lg(0.2)
    y = lst([0.0] * T)
    z = np.zeros((T, N))
    z[:, N - 1] = 100.0
    u = np.empty((T, N + 1))
    for t in range(T):
        if t % 2:                           # su_k = k / (N - 1) = cdf[k - 1] up to rounding
            if scheme == "multinomial":
                u[t] = 0.5
                u[t, 0] = u[t, N] = U_TOP
            else:
                u[t] = 0.0 if scheme == "systematic" else np.minimum(np.arange(N + 1) / (N - 1), U_TOP)
        else:
            u[t] = 0.0 if t % 4 == 0 and scheme != "multinomial" else U_TOP
    steps, rep = replay_run(monkeypatch, dev_m, orc_m, y, None, "boot", scheme, 1.0, N, T, chunk, noise=(z, u),
                            keep=True)
    assert rep.n_rs == T - 1
    tied = 0.0
    for s in steps[1:]:
        assert s["counts"][N - 1] <= 1                      # the zero-weight entry: at most the clamped last output
        A, su, cdf = s["A"], s["su"], s["cdf"]
        d = np.minimum(np.abs(su - cdf[A]), np.abs(su - cdf[np.maximum(A - 1, 0)]))
        tied = max(tied, float(np.mean(d[1:] <= 1e-12)))   # a CDF step is 1 / (N - 1) = 1e-6
    if scheme != "systematic":
        assert tied > 0.9, tied


# ------------------------------------------------------------------------------------------ batched filter, bank
def batch_models():
    from particles_b200 import kalman, state_space_models as ssm
    return {"sv": (ssm.StochVol(), orc.StochVol(), "data/sv_seed1_T1000"),
            "lg": (kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
                   "data/lg_seed2_T100")}


BATCH_CASES = [(m, f, s) for m in ("sv", "lg") for f in ("boot", "guided", "apf")
               for s in ("systematic", "stratified", "multinomial")]


@pytest.mark.parametrize("mname,fkname,scheme", BATCH_CASES)
def test_batched_multi_tile_vs_oracle(golden, mname, fkname, scheme):
    """The batched filter (k_batch, scan tiles of 2048 entries) past one tile, on the tier smcb_batch_plan picks and
    on the other one where the run fits it: rs_flags, ESS, logLt, X and A as in the single-tile oracle test, and at
    most one multinomial run diverging at a tie."""
    from particles_b200 import _lib, core, state_space_models as ssm
    dev_m, orc_m, dkey = batch_models()[mname]
    T = 20
    y = lst(golden[dkey][:T])
    mid = 4001 if scheme == "multinomial" else 4097
    diverged = 0
    for N, tiers in [(2049, ("resident", "streaming")), (mid, ("resident", "streaming")),
                     (20001, ("streaming",)), (65537, ("streaming",))]:
        R = 3
        rng = np.random.RandomState(N)
        noise = [(rng.standard_normal((T, N)), rng.rand(T, N + 1)) for _ in range(R)]
        kws = [dict(fk=getattr(ssm, FK[fkname])(ssm=dev_m, data=y), N=N, resampling=scheme, ESSrmin=e)
               for e in (0.5, 0.8, 0.99)]
        key, _ = core.batch_key(kws[0])
        auto = core.plan_group(key, R)[0]
        assert auto == (_lib.BATCH_RESIDENT if N < 5000 else _lib.BATCH_STREAMING), (N, auto)
        nu = {"systematic": 1, "stratified": N, "multinomial": N + 1}[scheme]
        refs = []
        for r, kw in enumerate(kws):
            z, u = noise[r]
            ref = orc.SMC(getattr(orc, FK[fkname])(orc_m, y), N=N, resampling=scheme, ESSrmin=kw["ESSrmin"],
                          noise=orc.InjectedNoise(z, [row[:nu] for row in u]))
            with np.errstate(all="ignore"):
                ref.run()
            refs.append(ref)
        for tier in tiers:
            runs = core.run_batch(kws, [11, 12, 13], noise=noise, tier=tier)
            for r, (pf, ref) in enumerate(zip(runs, refs)):
                try:
                    assert pf.summaries.rs_flags == ref.rs_flags, (N, tier, r)
                    np.testing.assert_allclose(pf.summaries.ESSs, ref.ESSs, rtol=1e-10)
                    np.testing.assert_allclose(pf.summaries.logLts, ref.logLts, rtol=1e-11, atol=1e-10)
                    np.testing.assert_allclose(host(pf.X), ref.X, rtol=1e-11, atol=1e-13)
                    if mname == "sv" and fkname == "boot":
                        assert np.array_equal(host(pf.X), ref.X)
                    if ref.rs_flag:
                        assert np.array_equal(host(pf.A), ref.A)
                except AssertionError:
                    if scheme != "multinomial":
                        raise
                    diverged += 1
    assert diverged <= 1, diverged


@pytest.mark.parametrize("tier", ["auto", "streaming"])
@pytest.mark.parametrize("mname,fkname", [("sv", "boot"), ("sv", "apf"), ("lg", "guided")])
@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
def test_bank_multi_tile_vs_batched(mname, fkname, scheme, tier):
    """One FilterBank.advance over T steps is the batched filter with the same keys, bit for bit, past one scan tile:
    the summary table, the last generation, the weights and the final ancestors."""
    from particles_b200 import _lib, bank, core, kalman, state_space_models as ssm
    from particles_b200.device import as_device
    T, R = 30, 3
    cls, names = (ssm.StochVol, ["mu", "rho", "sigma"]) if mname == "sv" else \
        (kalman.LinearGauss, ["rho", "sigmaX", "sigmaY"])
    theta = np.array([[-1.0, 0.95, 0.2], [-0.9, 0.9, 0.25], [-1.1, 0.97, 0.15]]) if mname == "sv" else \
        np.array([[0.9, 1.0, 0.3], [0.85, 1.2, 0.4], [0.95, 0.8, 0.2]])
    y = orc.config2_data(T, 3) if mname == "sv" else 1.5 * np.sin(np.arange(T))
    keys = [501 + 13 * r for r in range(R)]
    kind = {"boot": _lib.FK_BOOTSTRAP, "guided": _lib.FK_GUIDED, "apf": _lib.FK_APF}[fkname]
    for N in (4097, 20001):
        m = bank.ThetaMap(cls, names, y)
        b = bank.FilterBank(m.model, kind, scheme, N, R, as_device(y), m.n_params, 0.5,
                            shared_sc=None if m.shared_sc is None else as_device(m.shared_sc),
                            per_filter_sc=m.step_consts(theta) is not None, tier=tier)
        b.set_rows(m.params(theta), m.step_consts(theta))
        b.key.copy_(torch.tensor(np.asarray(keys, dtype=np.uint64).view(np.int64)))
        summ = torch.zeros((R, T, 4), dtype=torch.float64, device="cuda")
        A = torch.zeros((R, N + 1), dtype=torch.int64, device="cuda")
        b.advance(T, summaries=summ, A=A)
        table = host(summ)
        kws = [dict(fk=getattr(ssm, FK[fkname])(ssm=cls(**dict(zip(names, theta[r]))), data=lst(y)), N=N,
                    resampling=scheme) for r in range(R)]
        runs = core.run_batch(kws, keys, tier=tier)
        last = (T - 1) & 1
        assert table[:, 1:, 2].any()
        for r, run in enumerate(runs):
            assert np.array_equal(run._table, table[r]), (N, r)
            assert np.array_equal(host(run.X), host(b.X[r, last, :N])), (N, r)
            assert np.array_equal(host(run.wgts.lw), host(b.lw[r, :N])), (N, r)
            if run.rs_flag:
                assert np.array_equal(host(run.A), host(A[r, :N])), (N, r)
