"""The smoothing kernels on the H100, one time step at a time against the long-double replay of
tests/smoothing_replay.py: FFBS ON2 / MCMC / hybrid reject (csrc/smcb_smooth.cu), the PaRIS draws, ON2 backward
weights and Phi updates (csrc/smcb_online.cu) and the two-filter kernels (csrc/smcb_twofilter.cu), at the tile, CTA,
warp and row-block edges, on every device model, with injected draws and with the kernels' own Philox draws."""
import numpy as np
import pytest
import torch

import smoothing_replay as sr

pytestmark = pytest.mark.gpu
SEED = 20261017


def _model(name):
    from particles_b200 import kalman, state_space_models as ssm
    return {"sv": lambda: ssm.StochVol(), "svl": lambda: ssm.StochVolLeverage(phi=-0.5),
            "lg": lambda: kalman.LinearGauss(rho=0.8), "gordon": lambda: ssm.Gordon_etal(),
            "theta": lambda: ssm.ThetaLogistic(), "cox": lambda: ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9),
            "bearings": lambda: ssm.BearingsOnly(), "mvlg2": lambda: kalman.MVLinearGauss_Guarniero_etal(0.4, 2),
            "mvlg3": lambda: kalman.MVLinearGauss_Guarniero_etal(0.4, 3),
            "mvlg4": lambda: kalman.MVLinearGauss_Guarniero_etal(0.4, 4)}[name]()


ONE_D = ["sv", "svl", "lg", "gordon", "theta", "cox"]
MODELS = ONE_D + ["bearings", "mvlg2", "mvlg3", "mvlg4"]


def _fk(model, T, bound=None):
    from particles_b200 import state_space_models as ssm
    cls = type(model)
    if bound is not None:
        sub = type(cls.__name__ + "_bounded", (cls,), {"upper_bound_log_pt": lambda self, t: float(bound)})
        m2 = sub.__new__(sub)
        m2.__dict__.update(model.__dict__)
        model = m2
    dy = getattr(model, "dy", 1)
    return ssm.Bootstrap(ssm=model, data=[np.full(dy, 0.3)] * T)


def _states(name, N, T, r):
    """(T, N, D) host states that keep the backward weights informative: each generation moves its ancestors'
    locations by the model's own transition (Bearings: its Dirac components exactly)."""
    model = _model(name)
    spec = sr_spec(model, T)
    tr = sr.Trans(spec)
    D = spec["dim"]
    X = np.empty((T, N, D))
    X[0] = r.standard_normal((N, D))
    if name == "bearings":
        X[0, :, 2:] = 1.0 + 0.01 * r.standard_normal((N, 2))
    for t in range(1, T):
        a = r.randint(0, N, N)
        xp = X[t - 1][a]
        if name == "bearings":
            X[t, :, :2] = xp[:, :2] + model.sigmaX * r.standard_normal((N, 2))
            X[t, :, 2] = xp[:, 0] + xp[:, 2]
            X[t, :, 3] = xp[:, 1] + xp[:, 3]
        elif name.startswith("mvlg"):
            X[t] = xp @ tr.F.T + r.standard_normal((N, D)) @ tr.L.T
        else:
            loc = sr.f64(tr.loc1(t, xp[:, 0])[0])
            X[t, :, 0] = loc + tr.s * r.standard_normal(N)
    return spec, tr, X


def sr_spec(model, T):
    from particles_b200 import state_space_models as ssm
    return ssm.transition_spec(_fk(model, T))


def history(name, N, T, seed=0, soa=False, lw=None, bound=None, X=None):
    """A ParticleHistory of device tensors: row-major (N, D) particles, or the fused layout's strided (N, D) views
    of (D, N) buffers (soa=True)."""
    from particles_b200 import resampling as rs
    from particles_b200.smoothing import ParticleHistory
    r = np.random.RandomState(seed)
    spec, tr, Xs = _states(name, N, T, r)
    if X is not None:
        Xs = X
    D = spec["dim"]
    lw = r.standard_normal((T, N)) if lw is None else lw
    h = ParticleHistory(_fk(_model(name), T, bound), False)
    for t in range(T):
        if D == 1:
            x = torch.from_numpy(Xs[t, :, 0].copy()).cuda()
        elif soa:
            x = torch.from_numpy(np.ascontiguousarray(Xs[t].T)).cuda().t()
        else:
            x = torch.from_numpy(np.ascontiguousarray(Xs[t])).cuda()
        h.X.append(x)
        h.A.append(None if t == 0 else torch.from_numpy(r.randint(0, N, N)).cuda())
        h.wgts.append(rs.Weights(lw=torch.from_numpy(np.ascontiguousarray(lw[t])).cuda()))
    return h, tr, Xs, lw


def check_on2(h, tr, X, lw, idx, u, rows=None):
    """Every t: the draws of the chosen trajectories against the long-double rows.  Returns (near edges, zero
    rows)."""
    T, M = idx.shape
    rows = np.arange(M) if rows is None else rows
    near = zero = 0
    for t in range(T - 1):
        v, b = sr.row_values(tr, t + 1, X[t], lw[t], X[t + 1][idx[t + 1, rows]])
        a, z = sr.exact_draw_check(v, b, u[rows, t], idx[t, rows])
        near, zero = near + a, zero + z
    return near, zero


# ----------------------------------------------------------------------------------------------------------- ON2
ON2_CASES = [(1, 1, "lg"), (31, 255, "sv"), (32, 256, "cox"), (33, 257, "gordon"), (255, 1000, "theta"),
             (256, 33, "svl"), (257, 1, "bearings"), (513, 257, "mvlg2"), (4097, 256, "mvlg3"), (300, 1000, "mvlg4")]


@pytest.mark.parametrize("N,M,name", ON2_CASES, ids=lambda c: str(c))
@pytest.mark.parametrize("draws", ["injected", "device"])
def test_on2_replay(N, M, name, draws):
    T = 4
    h, tr, X, lw = history(name, N, T, seed=N + M, soa=(N % 2 == 1))
    r = np.random.RandomState(M)
    idx_T = r.randint(0, N, M)
    if draws == "injected":
        u = r.rand(M, T - 1)
        h.backward_sampling_ON2(M, seed=SEED, noise={"idx_T": idx_T, "u": u})
    else:
        h.backward_sampling_ON2(M, seed=SEED, noise={"idx_T": idx_T})
        js = np.arange(M)[:, None]
        u = sr.smooth_uniforms(SEED, 0, js, np.arange(T - 1)[None, :], 0, sr.PURPOSE_EXACT)[0]   # idx_T given: call 0
    idx = h._bs_idx.cpu().numpy()
    assert np.array_equal(idx[-1], idx_T)
    near, _ = check_on2(h, tr, X, lw, idx, u)
    assert near <= 2
    if N > sr.SM_BLOCK and M > 1:
        assert (idx[:-1] >= sr.SM_BLOCK).any()            # pass 2 went past the first tile


def test_on2_large_and_last_tile_straggler():
    """N = 20000 (79 tiles), M = 2048 (8 CTAs), T = 3; in the first CTA every trajectory but one finds its draw in
    the first tile, and that one needs the last particle of the last tile."""
    N, M, T = 20000, 2048, 3
    r = np.random.RandomState(5)
    _, tr, X = _states("lg", N, T, r)
    lw = np.full((T, N), -60.0)
    lw[:, :sr.SM_BLOCK] = 0.0
    X[1, -1, 0] = 40.0                                    # far from every target but one at 0.8 * 40
    X[2, 7, 0] = 32.0
    h, tr, X, lw = history("lg", N, T, seed=5, lw=lw, X=X)
    idx_T = r.randint(0, N, M)
    idx_T[3] = 7
    u = r.rand(M, T - 1) * 0.99
    h.backward_sampling_ON2(M, noise={"idx_T": idx_T, "u": u})
    idx = h._bs_idx.cpu().numpy()
    assert idx[1, 3] == N - 1
    others = np.delete(np.arange(sr.SM_BLOCK), 3)
    assert (idx[0, others] < sr.SM_BLOCK).all() and (idx[1, others] < sr.SM_BLOCK).all()
    rows = np.concatenate([np.arange(300), np.arange(M - 300, M)])
    check_on2(h, tr, X, lw, idx, u, rows)


def test_on2_zero_rows_nan_and_degenerate_weights():
    """All-zero rows give 0 (a lw_t of -inf everywhere; a Bearings Dirac no ancestor matches); a NaN term weighs
    zero; T = 1 and N = 1."""
    N, M, T = 300, 257, 4
    lw = np.random.RandomState(1).standard_normal((T, N))
    lw[1] = -np.inf
    lw[2, 5] = np.nan
    h, tr, X, lw = history("sv", N, T, seed=2, lw=lw)
    X[2, 6, 0] = np.nan                                   # a NaN state: NaN terms in every row of t = 2
    h.X[2] = torch.from_numpy(X[2, :, 0].copy()).cuda()
    r = np.random.RandomState(3)
    u = r.rand(M, T - 1)
    h.backward_sampling_ON2(M, noise={"idx_T": r.randint(0, N, M), "u": u})
    idx = h._bs_idx.cpu().numpy()
    assert (idx[1] == 0).all()
    assert (idx[2] != 5).all() and (idx[2] != 6).all()
    _, zero = check_on2(h, tr, X, lw, idx, u)
    assert zero == M
    # Bearings: targets whose Dirac components match no ancestor
    hb, trb, Xb, lwb = history("bearings", N, T, seed=4)
    Xb[2, :40, 2] += 1e-6
    hb.X[2] = torch.from_numpy(np.ascontiguousarray(Xb[2])).cuda()
    idx_T = r.randint(0, N, M)
    ub = r.rand(M, T - 1)
    hb.backward_sampling_ON2(M, noise={"idx_T": idx_T, "u": ub})
    ib = hb._bs_idx.cpu().numpy()
    _, zero = check_on2(hb, trb, Xb, lwb, ib, ub)
    assert zero > 0 and (ib[1][ib[2] < 40] == 0).all()
    # T = 1, N = 1
    h1, _, X1, _ = history("lg", 1, 1, seed=0)
    p = h1.backward_sampling_ON2(5, noise={"idx_T": np.zeros(5, dtype=np.int64)})
    assert torch.equal(p[0], torch.full((5,), float(X1[0, 0, 0]), dtype=torch.float64, device="cuda"))


def test_on2_u_zero_never_draws_a_zero_weight_particle():
    """An injected u = 0 (the reference's rand() can return it): the target is 0 and the draw is the first particle
    of positive weight, never a leading particle of weight zero."""
    N, M, T = 300, 64, 3
    lw = np.random.RandomState(0).standard_normal((T, N))
    lw[:, :7] = -np.inf
    h, tr, X, lw = history("lg", N, T, seed=9, lw=lw)
    h.backward_sampling_ON2(M, noise={"idx_T": np.arange(M) + 10, "u": np.zeros((M, T - 1))})
    idx = h._bs_idx.cpu().numpy()
    assert (idx[:-1] == 7).all()


# ---------------------------------------------------------------------------------------------------------- MCMC
@pytest.mark.parametrize("nsteps", [0, 1, 3])
@pytest.mark.parametrize("name", ["gordon", "mvlg3"])
def test_mcmc_replay_on_fused_history(nsteps, name):
    """A fused filter's history (SoA states, steps without resampling), the kernel's own proposals: draw_cdf on the
    CDF bits of ParticleHistory._cdfs, the counter of call 1 (the final-time multinomial draw takes call 0)."""
    import particles_b200 as pb
    from particles_b200 import state_space_models as ssm
    T, N, M = 8, 300, 257
    model = _model(name)
    y = [np.atleast_1d(np.asarray(v.cpu() if hasattr(v, "cpu") else v, dtype=np.float64)).reshape(-1)
         for v in model.simulate(T)[1]]
    pf = pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, store_history=True, seed=3, ESSrmin=0.3)
    assert pf.fused
    pf.run()
    h = pf.hist
    assert not all(pf.summaries.rs_flags)
    tr = sr.Trans(ssm.transition_spec(h.fk))
    h.backward_sampling_mcmc(M, nsteps=nsteps, seed=SEED)
    idx = h._bs_idx.cpu().numpy()
    X = [sr.as_rows(x.cpu().numpy()) for x in h.X]
    A = [None] + [a.cpu().numpy() for a in h.A[1:]]
    cdf = h._cdfs(N, h.X[0].device).cpu().numpy()[:, :N]
    undecided = 0
    for t in range(T - 1):
        start = A[t + 1][idx[t + 1]]
        if nsteps == 0:
            assert np.array_equal(idx[t], start)
            continue
        u0, u1 = sr.smooth_uniforms(SEED, 1, np.arange(M)[None, :], t, np.arange(nsteps)[:, None], sr.PURPOSE_SMOOTH)
        props = sr.draw_cdf(cdf[t], u0)
        got, sure = sr.mcmc_step(tr, t, X[t], X[t + 1][idx[t + 1]], start, props, np.log(u1))
        assert np.array_equal(got[sure], idx[t][sure]), t
        undecided += int((~sure).sum())
    assert undecided <= 2


# -------------------------------------------------------------------------------------------------------- reject
@pytest.mark.parametrize("M", [33, 257])
@pytest.mark.parametrize("loose", [0.0, 3.0])
def test_reject_replay(M, loose):
    T, N = 5, 300
    name = "sv" if M == 33 else "cox"
    model = _model(name)
    tight = -0.5 * np.log(2 * np.pi) - np.log(model.sigma)
    bound = tight + loose
    h, tr, X, lw = history(name, N, T, seed=M, bound=bound)
    r = np.random.RandomState(M + 1)
    idx_T = r.randint(0, N, M)
    cdf = h._cdfs(N, h.X[0].device).cpu().numpy()[:, :N]
    stragglers = fallback = 0
    for mt in sorted({0, 1, 4, 5, 36, 37, M}):
        h.backward_sampling_reject(M, max_trials=mt, seed=SEED, noise={"idx_T": idx_T})
        idx = h._bs_idx.cpu().numpy()
        acc_rate = h.acc_rate
        for t in range(T - 1):
            xn = X[t + 1][idx[t + 1]]
            props, lus = sr.device_trials(SEED, 0, np.arange(M), t, mt, cdf[t])
            first, choice, sure = sr.reject_trials(tr, t + 1, X[t], xn, props, lus, bound)
            assert sure.all()
            ok = first >= 0
            assert np.array_equal(idx[t][ok], choice[ok]), (mt, t)
            stragglers += int((first >= 4).sum())        # past kSoloTrials: a warp round
            nprop = np.where(ok, first + 1, mt)
            if nprop.sum():
                assert acc_rate[t] == ok.sum() / nprop.sum(), (mt, t)
            else:
                assert np.isnan(acc_rate[t])
            if (~ok).any():
                fallback += int((~ok).sum())
                u = sr.smooth_uniforms(SEED, 0, np.arange(M), t, 0, sr.PURPOSE_EXACT)[0]
                v, b = sr.row_values(tr, t + 1, X[t], lw[t], xn[~ok])
                sr.exact_draw_check(v, b, u[~ok], idx[t][~ok])
    assert stragglers > 0 and fallback > 0


def test_reject_fallback_all_zero_row_and_plugin_path():
    """The exact fallback on a row with no positive weight gives 0, in the kernel and on the plugin path."""
    from particles_b200 import state_space_models as ssm
    T, N, M = 4, 300, 40
    lw = np.random.RandomState(0).standard_normal((T, N))
    lw[1] = -np.inf
    h, tr, X, lw = history("sv", N, T, seed=1, lw=lw, bound=0.0)
    noise = {"idx_T": np.arange(M)}
    h.backward_sampling_reject(M, max_trials=0, noise=noise)
    assert (h._bs_idx.cpu().numpy()[1] == 0).all()

    class Plugin(ssm.Bootstrap):
        def logpt(self, t, xp, x):
            return ssm.Bootstrap.logpt(self, t, xp, x)
    h.fk = Plugin(ssm=h.fk.ssm, data=h.fk.data)
    assert ssm.transition_spec(h.fk) is None
    for fn in (lambda: h.backward_sampling_reject(M, max_trials=0, noise=noise),
               lambda: h.backward_sampling_ON2(M, noise=noise)):
        fn()
        assert (h._bs_idx.cpu().numpy()[1] == 0).all()


# --------------------------------------------------------------------------------------------------------- PaRIS
def _gens(name, N, r, lw_prev=None):
    from particles_b200.collectors import _Gen
    spec, tr, X = _states(name, N, 6, r)
    t = 4
    lwp = r.standard_normal(N) if lw_prev is None else lw_prev
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    x = (lambda a: dev(a[:, 0])) if spec["dim"] == 1 else dev
    gp = _Gen(t - 1, x(X[t - 1]), dev(lwp), None)
    g = _Gen(t, x(X[t]), dev(r.standard_normal(N)), None)
    return spec, tr, X[t - 1], X[t], lwp, gp, g


@pytest.mark.parametrize("Np,N", [(1, 257), (2, 129), (3, 100)])
def test_paris_replay(Np, N):
    from particles_b200 import _lib, resampling as rs
    from particles_b200.collectors import _online_desc, _run
    r = np.random.RandomState(Np)
    spec, tr, Xp, X, lwp, gp, g = _gens("gordon", N, r)
    cdf = rs.cumsum(rs.exp_and_normalise(gp.lw))
    cdf_h = cdf.cpu().numpy()
    bound = -0.5 * np.log(2 * np.pi) - np.log(tr.s)
    seed = 987654321
    K = N * Np
    hit_straggler = hit_fallback = 0
    for mt in (0, 1, 4, 5, 36, 37, N):
        B = torch.empty((N, Np), dtype=torch.int64, device="cuda")
        counts = torch.zeros(2, dtype=torch.int64, device="cuda")
        _run(_online_desc(_lib.ONLINE_PARIS, spec, gp, g, Np=Np, max_trials=mt, seed=seed, log_bound=bound, B=B,
                          counts=counts, cdf=cdf), B)
        Bh, ch = B.cpu().numpy().reshape(-1), counts.cpu().numpy()
        js = np.arange(K)
        xn = sr.as_rows(X)[js // Np]
        props, lus = sr.device_trials(sr.paris_seed(seed), g.t, js, 0, mt, cdf_h)
        first, choice, sure = sr.reject_trials(tr, g.t, Xp, xn, props, lus, bound)
        assert sure.all()
        ok = first >= 0
        assert np.array_equal(Bh[ok], choice[ok]), mt
        assert ch[0] == ok.sum() and ch[1] == np.where(ok, first + 1, mt).sum(), (mt, ch)
        hit_straggler += int((first >= 4).sum())    # past kSoloTrials: a warp round
        if (~ok).any():
            hit_fallback += 1
            u = sr.smooth_uniforms(sr.paris_seed(seed), g.t, js, 0, 0, sr.PURPOSE_EXACT)[0]
            v, b = sr.row_values(tr, g.t, Xp, lwp, xn[~ok])
            sr.exact_draw_check(v, b, u[~ok], Bh[~ok])
        # PHI_PARIS on these draws
        Kc = 3
        phi_prev = r.standard_normal((N, Kc))
        psi = r.standard_normal((K, Kc))
        phi = torch.empty((N, Kc), dtype=torch.float64, device="cuda")
        _run(_online_desc(_lib.ONLINE_PHI_PARIS, None, gp, g, Np=Np, k=Kc, B=B,
                          phi_prev=torch.from_numpy(phi_prev).cuda(), psi=torch.from_numpy(psi).cuda(), phi=phi), phi)
        sr.phi_paris_check(Bh, Np, phi_prev, psi, phi.cpu().numpy())
    assert hit_straggler > 0 and hit_fallback > 0


def test_paris_fallback_all_zero_row():
    from particles_b200 import _lib
    from particles_b200.collectors import _online_desc, _run
    r = np.random.RandomState(0)
    N = 70
    spec, tr, Xp, X, lwp, gp, g = _gens("lg", N, r, lw_prev=np.full(70, -np.inf))
    B = torch.full((N, 2), 5, dtype=torch.int64, device="cuda")
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    _run(_online_desc(_lib.ONLINE_PARIS, spec, gp, g, Np=2, max_trials=0, seed=1, log_bound=0.0, B=B,
                      counts=counts), B)
    assert (B.cpu().numpy() == 0).all() and counts.cpu().numpy().tolist() == [0, 0]


# ------------------------------------------------------------------------------------------------ online ON2
@pytest.mark.parametrize("N", [1, 255, 257, 4097])
@pytest.mark.parametrize("name", ["gordon", "theta", "mvlg2"])
def test_online_on2_weights_and_phi(N, name):
    """Row blocks with rows % 4 in {1, 2, 3} and row0 > 0 (and the whole range), K in {1, 3}."""
    from particles_b200 import _lib
    from particles_b200.collectors import _online_desc, _run
    r = np.random.RandomState(N)
    spec, tr, Xp, X, lwp, gp, g = _gens(name, N, r)
    blocks = [(r0, rows) for r0, rows in ((1, 5), (3, 2), (7, 3), (N - 97, 97)) if 0 < r0 and r0 + rows <= N]
    if N <= 257:
        blocks.append((0, N))
    for r0, rows in blocks:
        om = torch.empty((rows, N), dtype=torch.float64, device="cuda")
        _run(_online_desc(_lib.ONLINE_ON2_W, spec, gp, g, row0=r0, rows=rows, omega=om), om)
        omh = om.cpu().numpy()
        sr.on2_weights_check(tr, g.t, Xp, lwp, sr.as_rows(X)[r0:r0 + rows], omh)
        for K in (1, 3):
            phi_prev, psi = r.standard_normal((N, K)), r.standard_normal((rows, N, K))
            phi = torch.empty((rows, K), dtype=torch.float64, device="cuda")
            _run(_online_desc(_lib.ONLINE_PHI_ON2, None, gp, g, rows=rows, k=K, omega=om,
                              phi_prev=torch.from_numpy(phi_prev).cuda(),
                              psi=torch.from_numpy(psi.reshape(rows * N, K)).cuda(), phi=phi), phi)
            sr.phi_on2_check(omh, phi_prev, psi, phi.cpu().numpy())


# ------------------------------------------------------------------------------------------------- two-filter
@pytest.mark.parametrize("name", ONE_D)
def test_twofilter_replay(name):
    """ON2_ROWS in row blocks (Ninfo = 259: rows % 4 = 3, 257 rows past the first CTA's 4) over N = 300 forward
    particles; ON_LOGW with both modifiers.  Gordon's step constant is that of t + 1."""
    from particles_b200 import _lib
    from particles_b200.smoothing import ParticleHistory
    T, N, Ni, t = 6, 300, 259, 2
    r = np.random.RandomState(len(name))
    spec, tr, X = _states(name, N, T, r)
    _, _, Xi = _states(name, Ni, T, r)
    x, xi = X[t, :, 0], Xi[T - 2 - t, :, 0]
    lw = r.standard_normal(N)
    psi = r.standard_normal((Ni, N))
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()        # noqa: E731
    L = torch.empty(Ni, dtype=torch.float64, device="cuda")
    S = torch.empty(Ni, dtype=torch.float64, device="cuda")
    h = ParticleHistory(_fk(_model(name), T), False)
    for r0, rows in ((0, 5), (5, 254)):
        h._tf_desc(_lib.TF_ON2_ROWS, spec, t, d(x), d(xi), row0=r0, rows=rows, lw=d(lw), psi=d(psi[r0:r0 + rows]),
                   L=L, S=S)
    sr.on2_rows_check(tr, t, x, lw, xi, psi, L.cpu().numpy(), S.cpu().numpy())
    M = 1000
    I, J = r.randint(0, Ni, M), r.randint(0, N, M)
    mf, mi = r.standard_normal(N), r.standard_normal(Ni)
    lo, xf, xg = (torch.empty(M, dtype=torch.float64, device="cuda") for _ in range(3))
    h._tf_desc(_lib.TF_ON_LOGW, spec, t, d(x), d(xi), M=M, I=d(I), J=d(J), mf=d(mf), mi=d(mi), log_omega=lo, xf=xf,
               xi=xg)
    sr.on_logw_check(tr, t, x, xi, I, J, mf, mi, lo.cpu().numpy())
    assert np.array_equal(xf.cpu().numpy(), x[J]) and np.array_equal(xg.cpu().numpy(), xi[I])
