"""The sampler kernels of csrc/smcb_sampler.cu against the high-precision reference of tests/sampler_replay.py, at every
dimension tier, across the tier boundaries, with the data streamed through shared memory and with the device's own
Philox draws replayed on the host.

Every case asserts the branch it is named for: the D tier the dispatch picks, resident or streamed data in the fused
waste-free move (``tile_rows(D) >= n_rows``), and more than one CTA where a size is meant to span several.  The fused
move is checked one generation at a time from the kernel's own previous row (``check_generation``), so each tolerance
covers one generation.  Inputs are synthetic and seeded.  The file takes about 65 s of pytest time on an H100 80GB
HBM3 at a 700 W power limit, most of it in the long-double host references."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import samplers_numpy as sp  # noqa: E402
import sampler_replay as sr  # noqa: E402

SCALE = 5.0                                            # the prior scale of BASELINE config 5


def host(t):
    return t.detach().cpu().numpy()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


@pytest.fixture(scope="module")
def ctx():
    from particles_b200.device import context
    return context()


def lib_call(ctx, name, *args):
    from particles_b200 import _lib
    _lib.check(getattr(ctx.lib, name)(ctx.handle, *args))


def P(t):
    from particles_b200.device import ptr
    return ptr(t)


# ------------------------------------------------------------------------------------ smcb_logistic_target
TARGET_CASES = list(dict.fromkeys([(d, 257, 33) for d in (1, 2, 3, 4, 5, 8, 9, 12, 13, 16, 17, 20, 21, 24, 25, 31, 32)]
                                  + [(d, n, nd) for d in (5, 20) for n in (1, 2, 100_003) for nd in (1, 32)]
                                  + [(d, 257, nd) for d in (3, 17, 32) for nd in (1, 31, 32, 33, 1000)]))


def special_rows(theta):
    """Rows 0..7: saturated logits, zero, a NaN, +inf and -inf coordinates, 1e300 (the dot product overflows)."""
    n, d = theta.shape
    if n < 8:
        return theta
    theta = theta.copy()
    theta[0] *= 400.0
    theta[1] = 0.0
    theta[2, d // 2] = np.nan
    theta[3, 0] = np.inf
    theta[4, d - 1] = -np.inf
    theta[5] = 1e300
    theta[6] = -theta[0]
    return theta


@pytest.mark.parametrize("d,n,n_data", TARGET_CASES)
def test_logistic_target(ctx, d, n, n_data):
    D = sr.tier(d)
    data = sp.synthetic_logistic(n_data, d, seed=d + n_data) if n_data > 1 else np.random.RandomState(d).randn(1, d)
    r = np.random.RandomState(n + d)
    theta = special_rows(r.randn(n, d) * 2.0)
    if n > 1000:
        assert sr.target_grid(n) > 1                   # many CTAs
    # the rows checked: all of them up to 2000, else the specials, CTA edges and a random sample
    if n <= 2000:
        rows = np.arange(n)
    else:
        edges = np.arange(0, n, 2 * sr.SAMP_BLOCK)
        rows = np.unique(np.concatenate([np.arange(8), edges, edges - 1, np.arange(n - 3, n),
                                         r.randint(0, n, 600)]))
        rows = rows[(rows >= 0) & (rows < n)]
    from particles_b200 import smc_samplers as ssp
    model = ssp.LogisticRegression(data=data, prior_scale=SCALE)
    for epn in (0.0, 0.37, 1.0):
        x = ssp.ThetaParticles(theta=dev(theta))
        model.target(x, epn)
        # dot product: one chain of D fmas; rows summed in order
        (lp, ll, post), (bp, bl, bpost) = sr.target_bounds(theta[rows], data, SCALE, epn, D, D, n_data)
        sr.assert_close(f"d={d} epn={epn} lprior", host(x.lprior)[rows], lp, bp, "particle")
        sr.assert_close(f"d={d} epn={epn} llik", host(x.llik)[rows], ll, bl, "particle")
        sr.assert_close(f"d={d} epn={epn} lpost", host(x.lpost)[rows], post, bpost, "particle")
        if n >= 8:
            # a NaN parameter: NaN prior, -inf log-likelihood (NaN -> -inf after the row sum)
            assert np.isnan(host(x.lprior)[2]) and host(x.llik)[2] == -np.inf


# ------------------------------------------------------------------------------------ smcb_rw_propose
def lower_factor(d, seed, scale=0.3):
    r = np.random.RandomState(seed)
    L = np.tril(r.randn(d, d) * 0.2) + np.diag(1.0 + r.rand(d))
    return scale * L


@pytest.mark.parametrize("d", range(1, 33))
def test_rw_propose(ctx, d):
    n = 128 * 3 + 37 + d                                  # several CTAs, a partial last one
    r = np.random.RandomState(d)
    theta = r.randn(n, d) * 3.0
    L = lower_factor(d, d)
    th, Ld, out = dev(theta), dev(L), torch.empty((n, d), dtype=torch.float64, device="cuda")
    z = r.standard_normal((n, d))
    lib_call(ctx, "smcb_rw_propose", P(th), n, d, P(Ld), P(dev(z)), P(out))
    prop, b = sr.propose_ld(theta, z, L)
    sr.assert_close(f"d={d} injected proposal", host(out), prop, b, "particle")
    seed = 0xC0FFEE + d
    ctx.seed(seed)                                        # resets the API call counter: calls 0, 1, ...
    for call in (0, 1):
        lib_call(ctx, "smcb_rw_propose", P(th), n, d, P(Ld), P(None), P(out))
        zd = sr.rw_propose_normals(n, d, call, seed)
        prop, b = sr.propose_ld(theta, zd, L)
        b = b + sr.propose_bound_z(zd, L, sr.Z_REL)
        sr.assert_close(f"d={d} device-drawn proposal, call {call}", host(out), prop, b, "particle")


# ------------------------------------------------------------------------------------ smcb_mh_accept(_flags)
def mh_inputs(n, d, seed, specials):
    r = np.random.RandomState(seed)
    theta, theta_p = r.randn(n, d), r.randn(n, d)
    lpr, lpr_p = r.randn(n), r.randn(n)
    ll, ll_p = r.randn(n), r.randn(n)
    lpost = r.randn(n) * 2.0
    lpost_p = lpost + r.randn(n) * 2.0
    u = r.rand(n)
    if specials:
        lpost_p[0] = np.nan                               # NaN on either side: pb NaN, reject
        lpost[1] = np.nan
        lpost_p[2], lpost[3] = -np.inf, -np.inf           # -inf proposal: reject; -inf current: accept
        lpost[4] = lpost_p[4] = -np.inf                   # both -inf: NaN, reject
        lpost_p[5], u[5] = lpost[5] + 0.5, 1.0            # lp_acc >= 0, u = 1.0: reject (strict <)
        lpost_p[6], u[6] = lpost[6], np.nextafter(1.0, 0.0)   # lp_acc = 0, u just below 1: accept
        lpost_p[7], u[7] = -np.inf, 0.0                   # lp_acc = -inf, u = 0: reject
    return theta, theta_p, lpr, lpr_p, ll, ll_p, lpost, lpost_p, u


@pytest.mark.parametrize("n", [1, 127, 128, 129, 1_000_003])
@pytest.mark.parametrize("mode", ["injected", "device"])
@pytest.mark.parametrize("specials", [False, True])
def test_mh_accept(ctx, n, mode, specials):
    if specials and n < 8:
        pytest.skip("needs 8 particles for the special rows")
    d = 3
    theta, theta_p, lpr, lpr_p, ll, ll_p, lpost, lpost_p, u = mh_inputs(n, d, n, specials)
    grid = -(-n // sr.SAMP_BLOCK)
    if n > 1000:
        assert grid > 1000                                # the mean crosses many CTAs
    cur = [dev(a) for a in (theta, lpr, ll, lpost)]
    pro = [dev(a) for a in (theta_p, lpr_p, ll_p, lpost_p)]
    mean = torch.empty(1, dtype=torch.float64, device="cuda")
    flags = torch.empty(n, dtype=torch.uint8, device="cuda")
    if mode == "device":
        seed = 0xBEEF + n
        ctx.seed(seed)
        lib_call(ctx, "smcb_uniform", P(torch.empty(4, dtype=torch.float64, device="cuda")), 4)   # call 0
        u = sr.mh_accept_uniforms(n, 1, seed)                                                    # call 1
        uin = None
    else:
        uin = dev(u)
    lib_call(ctx, "smcb_mh_accept_flags", n, d, *[P(t) for t in cur], *[P(t) for t in pro], P(uin), P(mean), P(flags))
    with np.errstate(invalid="ignore"):
        lp_acc = lpost_p - lpost + 0.0                    # the same IEEE subtraction as the kernel
        pb = np.exp(np.minimum(lp_acc, 0.0))
    pb[np.isnan(lp_acc)] = np.nan
    # the device's exp is within 1 ulp of NumPy's: a draw within 2 ulp of pb may go either way
    acc, decided = sr.decisions(u, lp_acc.astype(sr.LD), 2 * sr.EPS * np.ones(n))
    fl = host(flags).astype(bool)
    k0 = 8 if specials else 0                             # rows 5 and 6 are ties on purpose, pinned below
    assert (~decided[k0:]).sum() <= n // 1000, int((~decided[k0:]).sum())
    bad = decided & (fl != acc)
    assert not bad.any(), int(np.flatnonzero(bad)[0])
    if specials and mode == "injected":
        assert fl[:8].tolist() == [False, False, False, True, False, False, True, False]
    elif specials:
        assert fl[:3].tolist() == [False, False, False] and fl[3] and not fl[4] and not fl[7]
    # state: accepted rows are the proposal's bits, the others untouched
    for got, a, b in zip(cur, (theta, lpr, ll, lpost), (theta_p, lpr_p, ll_p, lpost_p)):
        want = np.where(fl.reshape((-1,) + (1,) * (a.ndim - 1)), b, a)
        assert np.array_equal(host(got).view(np.int64), want.view(np.int64))
    m = float(host(mean)[0])
    if specials:
        assert np.isnan(m)                                # NumPy's mean of an array with a NaN
    else:
        # per-thread pb (1 ulp of exp), then 5 shuffle levels, 4 warps and the CTAs in order: depth 10 + grid
        want = pb.astype(sr.LD).sum() / n
        assert abs(m - float(want)) <= float(sr.gamma(10 + grid)) * float(want) + sr.EPS * float(want), (m, want)


def test_mh_accept_workspace_bound(ctx):
    """Past 65536 CTAs of 128 particles the block partials do not fit the workspace: a clean error, nothing launched."""
    from particles_b200 import _lib
    n = sr.WS_PARTIALS * sr.SAMP_BLOCK + 1
    a = torch.zeros(n, dtype=torch.float64, device="cuda")
    mean = torch.empty(1, dtype=torch.float64, device="cuda")
    launches = ctx.launches
    with pytest.raises((ValueError, _lib.SmcbError), match="workspace"):
        lib_call(ctx, "smcb_mh_accept_flags", n, 1, P(a), P(a), P(a), P(a), P(a), P(a), P(a), P(a), P(a), P(mean),
                 P(None))
    assert ctx.launches == launches


# ------------------------------------------------------------------------------------ smcb_rw_calibrate and pieces
def weights(kind, n, r):
    if kind == "random":
        w = np.exp(r.randn(n))
    elif kind == "zeros":
        w = np.exp(r.randn(n))
        w[r.rand(n) < 0.3] = 0.0
        w[0] = 1.0
    elif kind == "dominant":
        w = np.full(n, 1e-12 / max(n - 1, 1))
        w[n // 2] = 1.0 - 1e-12
    else:                                                 # unnormalised
        return np.exp(r.randn(n) * 3.0) * 1e3
    return w / w.sum()


def thetas(kind, n, d, r):
    if kind == "unit":
        return r.randn(n, d) @ np.tril(r.rand(d, d) * 0.5 + np.eye(d)).T
    if kind == "offset":
        return 1e6 + r.randn(n, d) * np.linspace(1.0, 2.0, d) - 2e6 * (np.arange(d) % 2)
    # condition number ~1e10: the coordinates' scales run from 1 to 1e-5 after a random rotation
    Q, _ = np.linalg.qr(r.randn(d, d))
    return (r.randn(n, d) * np.logspace(0, -5, d)) @ Q.T


def calibrate_all(ctx, W, theta, scale):
    """(s0, tri, L from smcb_rw_calibrate, L from the same sums through smcb_chol_from_sums, L unscaled)."""
    n, d = theta.shape
    Wd, th = dev(W), dev(theta)
    s0 = torch.empty(d + 1, dtype=torch.float64, device="cuda")
    lib_call(ctx, "smcb_wcov_sums", P(Wd), P(th), n, d, P(None), P(s0))
    mean = (s0[:d] / s0[d]).contiguous()
    tri = torch.empty(d * (d + 1) // 2, dtype=torch.float64, device="cuda")
    lib_call(ctx, "smcb_wcov_sums", P(Wd), P(th), n, d, P(mean), P(tri))
    sw = s0[d:].contiguous()
    Ls = [torch.empty((d, d), dtype=torch.float64, device="cuda") for _ in range(3)]
    lib_call(ctx, "smcb_rw_calibrate", P(Wd), P(th), n, d, scale, P(Ls[0]))
    lib_call(ctx, "smcb_chol_from_sums", P(tri), P(sw), d, scale, P(Ls[1]))
    lib_call(ctx, "smcb_chol_from_sums", P(tri), P(sw), d, 1.0, P(Ls[2]))
    return host(s0), host(tri), [host(L) for L in Ls]


CAL_CASES = ([(d, 2111, "random", "unit") for d in range(1, 21)]
             + [(d, n, "random", "unit") for d in (3, 20) for n in (1, 2, 7, 8, 9, 1_000_003)]
             + [(4, 10_000_000, "random", "unit")]
             + [(6, 3001, w, "unit") for w in ("zeros", "dominant", "unnormalised")]
             + [(d, 5000, "random", t) for d in (6, 20) for t in ("offset", "illcond")])


@pytest.mark.parametrize("d,n,wkind,tkind", CAL_CASES)
def test_rw_calibrate(ctx, d, n, wkind, tkind):
    r = np.random.RandomState(d * 7 + n % 1000)
    W, theta = weights(wkind, n, r), thetas(tkind, n, d, r)
    if n >= 1_000_000:
        assert sr.ctl_grid_wcov(n) == sr.CTL_GRID          # a full grid of CTAs
    scale = 2.38 / np.sqrt(d)
    s0, tri, (Lcal, Lsum, L1) = calibrate_all(ctx, W, theta, scale)
    mean, cov = sr.check_wcov(W, theta, s0, tri)
    # smcb_rw_calibrate = the same sums, the same quotients, the same factorisation: the same bits
    assert np.array_equal(Lcal.view(np.int64), Lsum.view(np.int64))
    if n > d:
        # the factor of exactly the fp64 covariance the kernel formed, judged by its backward error
        cov64 = sr.unpack_tri(tri, d) / s0[d]
        assert np.all(np.isfinite(L1)), L1
        sr.chol_backward_check(cov64, L1)
        assert np.array_equal(Lsum, L1 * scale)           # scaling by 2.38 / sqrt(d) is one rounding of each entry


@pytest.mark.parametrize("k", [1, 2, 3, 8])
@pytest.mark.parametrize("d", [3, 20])
def test_sharded_calibration(ctx, k, d):
    """The rows split into k shards, combined with shares as ShardedAdaptiveTempering._calibrate does, against the
    long-double values and smcb_rw_calibrate on all rows."""
    n = 40_001
    r = np.random.RandomState(k + d)
    W, theta = weights("random", n, r), thetas("unit", n, d, r)
    edges = np.linspace(0, n, k + 1).astype(int)
    Wd = dev(W)
    S = Wd.sum()
    s0 = torch.zeros(d + 1, dtype=torch.float64, device="cuda")
    parts = []
    for a, b in zip(edges[:-1], edges[1:]):
        Wl = (Wd[a:b] / Wd[a:b].sum()).contiguous()
        share = float((Wd[a:b].sum() / S).item())
        th = dev(theta[a:b])
        out = torch.empty(d + 1, dtype=torch.float64, device="cuda")
        lib_call(ctx, "smcb_wcov_sums", P(Wl), P(th), b - a, d, P(None), P(out))
        s0 += out * share
        parts.append((Wl, th, share, b - a))
    mean = (s0[:d] / s0[d]).contiguous()
    tri = torch.zeros(d * (d + 1) // 2, dtype=torch.float64, device="cuda")
    for Wl, th, share, m in parts:
        out = torch.empty(d * (d + 1) // 2, dtype=torch.float64, device="cuda")
        lib_call(ctx, "smcb_wcov_sums", P(Wl), P(th), m, d, P(mean), P(out))
        tri += out * share
    L1 = torch.empty((d, d), dtype=torch.float64, device="cuda")
    lib_call(ctx, "smcb_chol_from_sums", P(tri), P(s0[d:].contiguous()), d, 1.0, P(L1))
    # per term: the shard's sum of weights (its depth), W / S_k, the share S_k / S (S: a sum over the n weights), the
    # product by the share and the sum over the k shards
    depth = sr.wcov_depth(-(-n // k), k)
    extra = n + 4
    Wn = W / float(S.item())
    sr.check_wcov(Wn, theta, host(s0), host(tri), depth=depth, extra=extra)
    cov_k = sr.unpack_tri(host(tri), d) / host(s0)[d]
    sr.chol_backward_check(cov_k, host(L1))
    # against the unsharded calibration: L L^T of both within their backward errors and the two covariances' bounds
    s0_1, tri_1, (_, _, L1_1) = calibrate_all(ctx, W, theta, 1.0)
    cov_1 = sr.unpack_tri(tri_1, d) / s0_1[d]
    A, B = host(L1), L1_1
    gap = np.abs(A @ A.T - B @ B.T)
    allow = (sr.gamma(d + 2) * (np.abs(A) @ np.abs(A).T + np.abs(B) @ np.abs(B).T)
             + np.abs(cov_k - cov_1) + 4 * sr.EPS * np.abs(cov_1))
    assert np.all(gap <= allow + 1e-300), float((gap - allow).max())


@pytest.mark.parametrize("n", [1, 1000, 100_003])
@pytest.mark.parametrize("k", [1, 3])
def test_essl_grid(ctx, n, k):
    """The 32 sums of one root pass (shifted by the global maximum) against long-double sums, per shard and summed."""
    r = np.random.RandomState(n + k)
    lw = -np.abs(r.randn(n)) * 30.0 - 2.0
    lw[r.rand(n) < 0.1] = -np.inf
    lw[0] = -2.0
    lo, hi = 0.0123, 0.4567
    mx = dev(np.array([lw.max()]))
    edges = np.linspace(0, n, k + 1).astype(int)
    tot = np.zeros(32)
    depth = 0
    for a, b in zip(edges[:-1], edges[1:]):
        if b == a:
            continue
        out = torch.empty(32, dtype=torch.float64, device="cuda")
        lib_call(ctx, "smcb_essl_grid", P(dev(lw[a:b])), b - a, lo, hi, P(mx), P(out))
        tot += host(out)
        g = sr.ctl_grid_root(b - a)
        depth = max(depth, -(-(b - a) // (g * sr.CTL_BLOCK)) + 5 + 8 + g)
    a_ = lw.astype(sr.LD) - sr.LD(lw.max())
    for j in range(16):
        dj = lo + (hi - lo) * ((j + 1) / 16.0)
        with np.errstate(invalid="ignore"):
            e = np.exp(sr.LD(dj) * a_)
        e[np.isnan(e)] = 0
        s, q = e.sum(), (e * e).sum()
        ef = e.astype(np.float64)
        fin = np.isfinite(a_)
        # per term: lw - max, the candidate exponent (one fma or two roundings of dj: 2 u dj) and the product, then
        # fexp_neg's 1.5 ulp; q's terms square that; the sums have the pass's depth plus the k shards
        ab = np.abs(np.where(fin, a_, 0).astype(np.float64))
        rel = sr.U * (3 * dj * ab + 3)
        bs = (ef * rel).sum() + sr.gamma(depth + k) * float(s)
        bq = 2 * (ef * ef * rel).sum() + sr.gamma(depth + k + 1) * float(q)
        sr.assert_close(f"s_{j}", tot[2 * j:2 * j + 1], np.array([s]), np.array([bs]))
        sr.assert_close(f"q_{j}", tot[2 * j + 1:2 * j + 2], np.array([q]), np.array([bq]))


def test_sharded_next_exponent_world1(ctx):
    """ShardedAdaptiveTempering._next_exponent (host bracket decisions over smcb_essl_grid sums) against
    smcb_next_annealing_epn at world 1: within one final bracket -- the host forms lo + (hi - lo) j / 16 without the
    device's fma, so a grid point within rounding of alpha N may fall either way -- and both pass the root check."""
    from particles_b200 import smc_samplers as ssp
    from particles_b200.sharded_samplers import ShardedAdaptiveTempering
    sm = ShardedAdaptiveTempering(model=ssp.LogisticRegression(data=sp.synthetic_logistic(10, 2, seed=0)),
                                  M_local=4, len_chain=2, ESSrmin=0.5, seed=3)
    r = np.random.RandomState(5)
    for n, scale, epn in [(100_000, 40.0, 0.0), (5001, 300.0, 0.013), (20_000, 0.01, 0.2), (777, 7.0, 0.5)]:
        lw = -np.abs(r.randn(n)) * scale - 3.0
        a = sm._next_exponent(dev(lw), epn)
        b = ssp.next_annealing_epn(epn, 0.5, dev(lw))
        assert abs(a - b) <= sr.final_bracket(epn) * (1 + 1e-9) + 4 * sr.U, (n, a, b)
        sr.check_root(lw, epn, 0.5, a)
        sr.check_root(lw, epn, 0.5, b)


# ------------------------------------------------------------------------------------ next_annealing_epn
def root_inputs(name, r):
    if name == "half_neginf":
        lw = -np.abs(r.randn(20_000)) * 50.0
        lw[r.rand(20_000) < 0.5] = -np.inf
        return lw, 0.1, 0.3                               # ESS -> N / 2 as delta -> 0: the root needs alpha < 1 / 2
    if name == "equal":
        return np.full(5000, -3.25), 0.3, 0.5
    if name == "all_neginf":
        return np.full(1000, -np.inf), 0.0, 0.5
    if name == "n1":
        return np.array([-7.0]), 0.0, 0.5
    if name == "n2":
        return np.array([0.0, -100.0]), 0.0, 0.9
    if name == "epn_near_1":
        return -np.abs(r.randn(10_000)) * 1e10, 1.0 - 1e-9, 0.5
    if name.startswith("alpha"):
        return -np.abs(r.randn(30_000)) * 200.0, 0.05, float(name[5:])
    if name == "tiny_root":                               # the root sits near 1e-10
        return -np.abs(r.randn(50_000)) * 1e10, 0.0, 0.5
    if name == "n1e7":
        return -np.abs(r.randn(10_000_000)) * 60.0 - 1.0, 0.02, 0.5
    raise KeyError(name)


@pytest.mark.parametrize("name", ["half_neginf", "equal", "all_neginf", "n1", "n2", "epn_near_1", "alpha0.01",
                                  "alpha0.5", "alpha0.99", "tiny_root", "n1e7"])
def test_next_annealing_epn(ctx, name):
    from particles_b200 import smc_samplers as ssp
    r = np.random.RandomState(len(name))
    lw, epn, alpha = root_inputs(name, r)
    got = ssp.next_annealing_epn(epn, alpha, dev(lw))
    if name in ("equal", "all_neginf", "n1"):
        # ESS = N exactly at every exponent (all weights equal, or one particle); all -inf: every ESS is NaN, which
        # compares false against alpha N, so the whole step is taken -- as the reference's f(1 - epn) < 0 does
        assert got == 1.0
        return
    if name == "tiny_root":
        assert 1e-11 < got < 1e-9
    if name == "n2":
        assert got < 1.0
    if name == "n1e7":
        assert sr.ctl_grid_root(lw.shape[0]) == sr.CTL_GRID
    sr.check_root(lw, epn, alpha, got)


# ------------------------------------------------------------------------------------ smcb_logistic_wf_move
def wf_raw(ctx, theta0, lpr0, ll0, lp0, data_dev, n_rows, epn, L, P_, z=None, u=None):
    M, d = theta0.shape
    out = [torch.empty((P_ * M, d), dtype=torch.float64, device="cuda")] + [
        torch.empty(P_ * M, dtype=torch.float64, device="cuda") for _ in range(3)]
    pb = torch.empty((P_ - 1, M), dtype=torch.float64, device="cuda")
    lib_call(ctx, "smcb_logistic_wf_move", M, d, P_, P(theta0), P(lpr0), P(ll0), P(lp0), P(data_dev), n_rows, SCALE,
             epn, P(L), P(z), P(u), *[P(t) for t in out], P(pb))
    th, lpr, ll, lp = (host(t) for t in out)
    rows = [{"theta": th[s * M:(s + 1) * M], "lprior": lpr[s * M:(s + 1) * M], "llik": ll[s * M:(s + 1) * M],
             "lpost": lp[s * M:(s + 1) * M]} for s in range(P_)]
    return rows, host(pb)


def wf_case(d, n_rows, seed, n_total=None):
    """Data, starting points and a factor scaled to the tempered posterior, so both accepts and rejects occur."""
    data = sp.synthetic_logistic(n_total or n_rows, d, seed=seed)
    epn = min(1.0, 40.0 / n_rows)
    r = np.random.RandomState(seed + 1)
    sigma = 1.0 / np.sqrt(epn * n_rows * 0.15 + 1.0 / SCALE ** 2)
    theta0 = r.randn(d) * sigma * 0.5 + r.randn(64, d) * sigma * 0.5
    L = lower_factor(d, seed, scale=1.2 * sigma / np.sqrt(d))
    return data, epn, theta0, L


def run_wf(ctx, d, M, P_, n_rows, mode, seed, n_total=None, expect=None):
    D = sr.tier(d)
    resident = sr.wf_resident(d, n_rows)
    if expect is not None:
        assert resident == (expect == "resident"), (d, n_rows, sr.tile_rows(D))
    data, epn, base, L = wf_case(d, n_rows, seed, n_total)
    r = np.random.RandomState(seed + 2)
    theta0 = base[r.randint(0, base.shape[0], M)] + r.randn(M, d) * 1e-3
    from particles_b200 import smc_samplers as ssp
    model = ssp.LogisticRegression(data=data, prior_scale=SCALE)
    x = ssp.ThetaParticles(theta=dev(theta0))
    model.target(x, epn, n_rows=n_rows if n_total else None)
    Ld = dev(L)
    if mode == "injected":
        z, u = r.standard_normal((P_ - 1, M, d)), r.rand(P_ - 1, M)
        rows, pb = wf_raw(ctx, x.theta, x.lprior, x.llik, x.lpost, model.data, n_rows, epn, Ld, P_, dev(z), dev(u))
        zs = [z[s - 1] for s in range(1, P_)]
        us = [u[s - 1] for s in range(1, P_)]
        zrel = 0.0
    else:
        key = 0x5A5A0000 + seed
        ctx.seed(key)
        wf_raw(ctx, x.theta, x.lprior, x.llik, x.lpost, model.data, n_rows, epn, Ld, P_)          # call 0
        rows, pb = wf_raw(ctx, x.theta, x.lprior, x.llik, x.lpost, model.data, n_rows, epn, Ld, P_)  # call 1
        zs = [sr.wf_normals(M, d, s, 1, key) for s in range(1, P_)]
        us = [sr.wf_uniforms(M, s, 1, key) for s in range(1, P_)]
        zrel = sr.Z_REL
    assert np.array_equal(rows[0]["theta"], theta0)      # generation row 0: the starting points themselves
    dat = data[:n_rows]
    n_acc = n_dec = 0
    for s in range(1, P_):
        acc, decided = sr.check_generation(s, rows[s - 1], rows[s], pb[s - 1], zs[s - 1], us[s - 1], L, dat, SCALE,
                                           epn, d, z_rel=zrel)
        n_acc += int(acc.sum())
        n_dec += int(decided.sum())
    total = M * (P_ - 1)
    assert n_dec >= total - max(1, total // 1000)
    if total >= 60:
        assert 0 < n_acc < total, (n_acc, total)
    return resident


WF_TIER_CASES = [(D, branch) for D in sr.TIERS for branch in ("resident", "edge", "streamed")]


@pytest.mark.parametrize("mode", ["injected", "device"])
@pytest.mark.parametrize("D,branch", WF_TIER_CASES)
def test_wf_move_tiers(ctx, D, branch, mode):
    """Each tier at its largest d: n_rows = tile_rows(D) (resident), tile_rows(D) + 1 (streamed, a one-row last tile)
    and ~2.5 tile_rows(D) (streamed, a partial last tile); 33 chains (two CTAs, the second with one chain), P = 9."""
    t = sr.tile_rows(D)
    n_rows = {"resident": t, "edge": t + 1, "streamed": int(2.5 * t) + 7}[branch]
    assert sr.tier(D) == D
    run_wf(ctx, D, 33, 9, n_rows, mode, seed=D * 10 + len(branch),
           expect="resident" if branch == "resident" else "streamed")
    assert sr.wf_grid(33) == 2


WF_D_CASES = [(d, M, P_, n_rows) for d, M, P_, n_rows in [
    (1, 31, 9, 200), (3, 33, 2, 7000), (5, 1, 9, 3200), (17, 33, 9, 1300), (25, 31, 9, 800), (25, 33, 2, 200),
    (5, 4097, 2, 150), (20, 4097, 2, 100), (12, 1, 2, 50), (16, 4097, 9, 20), (32, 33, 9, 2)]]


@pytest.mark.parametrize("mode", ["injected", "device"])
@pytest.mark.parametrize("d,M,P_,n_rows", WF_D_CASES)
def test_wf_move_shapes(ctx, d, M, P_, n_rows, mode):
    """The d values off the tiers' tops (d = 1, 3, 5, 17, 25) and M in {1, 31, 33, 4097}, P in {2, 9}."""
    resident = run_wf(ctx, d, M, P_, n_rows, mode, seed=d * 100 + M)
    assert resident == (n_rows <= sr.tile_rows(sr.tier(d)))
    if M > 32:
        assert sr.wf_grid(M) > 1


def test_wf_move_eeg_shape(ctx):
    """The reference's EEG data set has 14980 rows of 15 predictors (d = 16 with the intercept): streamed at D = 16."""
    assert not run_wf(ctx, 16, 33, 9, 14980, "device", seed=14980) and sr.tier(16) == 16


def test_wf_move_ibis_prefix(ctx):
    """IBIS moves target the first n_rows of a longer data set: n_rows > tile_rows(12) streams the prefix only."""
    assert sr.tile_rows(12) < 2500
    assert not run_wf(ctx, 12, 40, 5, 2500, "device", seed=7, n_total=4000)


# ------------------------------------------------------------------------------------ degenerate calibrations
@pytest.mark.parametrize("d", [1, 2, 7, 20])
def test_zero_covariance_leaves_the_chains_alone(ctx, d):
    """One weight 1 and the rest 0: every deviation is exactly 0, so the covariance is exactly 0.  The reference's
    numpy.linalg.cholesky raises LinAlgError here; this project keeps running: for d >= 2 the factor is non-finite
    (0 / 0 below the first pivot), every proposal has a NaN log-prior, every pb is NaN and nothing is accepted; for
    d = 1 the factor is 0 and the proposal is the current point.  Either way one random-walk step and one waste-free
    move leave theta, lprior, llik and lpost bit for bit as they were -- except that for d = 1 the move's kernel
    re-evaluates the (accepted, identical) point with its own row order, so llik and lpost may change in the last
    bits there, within the log-likelihood's rounding bound."""
    from particles_b200 import smc_samplers as ssp
    n, M, P_ = 300, 300, 4
    data = sp.synthetic_logistic(50, d, seed=d)
    r = np.random.RandomState(d)
    theta = r.randn(n, d)
    W = np.zeros(n)
    W[17] = 1.0
    model = ssp.LogisticRegression(data=data, prior_scale=SCALE)
    x = ssp.ThetaParticles(theta=dev(theta))
    model.target(x, 0.5)
    rw = ssp.ArrayRandomWalk()
    rw.calibrate(dev(W), x)
    L = host(x.shared["chol_cov"])
    if d == 1:
        assert L[0, 0] == 0.0
    else:
        assert not np.all(np.isfinite(L))
    before = {k: host(getattr(x, k)).copy() for k in ("theta", "lprior", "llik", "lpost")}
    ctx.seed(99)
    out = model.wf_move(x, 0.5, P_)
    rw.step(x, lambda xx: model.target(xx, 0.5))
    for k, v in before.items():
        assert np.array_equal(host(getattr(x, k)).view(np.int64), v.view(np.int64)), k
    for s in range(P_):
        rows = {k: host(getattr(out, k))[s * M:(s + 1) * M] for k in before}
        assert np.array_equal(rows["theta"].view(np.int64), before["theta"].view(np.int64)), s
        assert np.array_equal(rows["lprior"].view(np.int64), before["lprior"].view(np.int64)), s
        if d > 1 or s == 0:
            for k in ("llik", "lpost"):
                assert np.array_equal(rows[k].view(np.int64), before[k].view(np.int64)), (k, s)
        else:
            D = sr.tier(d)
            (_, ll, post), (_, bl, bpost) = sr.target_bounds(theta, data, SCALE, 0.5, D, D // 2 + 1, data.shape[0] + 4)
            sr.assert_close("d = 1 llik", rows["llik"], ll, bl, "chain")
            sr.assert_close("d = 1 lpost", rows["lpost"], post, bpost, "chain")


@pytest.mark.parametrize("d,n", [(5, 2), (8, 8), (20, 3), (20, 20)])
def test_rank_deficient_covariance_never_reaches_theta(ctx, d, n):
    """n <= d rows: the covariance is singular, and rounding decides whether a late pivot is a tiny positive, zero or
    a tiny negative number (the reference raises LinAlgError).  Whatever the factor, no NaN or inf reaches theta after
    a step or a waste-free move: a non-finite proposal has a NaN or -inf log-prior and is never accepted."""
    from particles_b200 import smc_samplers as ssp
    data = sp.synthetic_logistic(40, d, seed=d)
    r = np.random.RandomState(n + d)
    theta = r.randn(n, d)
    model = ssp.LogisticRegression(data=data, prior_scale=SCALE)
    x = ssp.ThetaParticles(theta=dev(theta))
    model.target(x, 0.7)
    rw = ssp.ArrayRandomWalk()
    rw.calibrate(dev(np.full(n, 1.0 / n)), x)
    ctx.seed(5)
    out = model.wf_move(x, 0.7, 5)
    assert np.all(np.isfinite(host(out.theta)))
    assert not np.any(np.isnan(host(out.lpost)))
    for _ in range(3):
        rw.step(x, lambda xx: model.target(xx, 0.7))
        assert np.all(np.isfinite(host(x.theta)))
        assert not np.any(np.isnan(host(x.lpost)))
