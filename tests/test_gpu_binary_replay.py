"""The binary-space kernels of csrc/smcb_binary.cu against the high-precision reference of tests/binary_replay.py, at
every warp tier, at the 32-bit word edges of p up to p = 128, with the device's own Philox draws replayed on the host.

Every case asserts the regime it is named for: the warps per CTA the launch picks (``binary_replay.bin_warps``), more
than one CTA with a partial last one, and the word count of p.  The C ABI is called directly where outputs must be
read despite an error bit; the public classes are checked to raise on it.  The move is checked one generation at a time
from the kernel's own previous row, so each tolerance covers one generation.  Inputs are synthetic and seeded.  The
file takes about 36 s of pytest time on an H100 80GB HBM3 at a 700 W power limit, most of it in the long-double host
replay."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import binary_replay as br  # noqa: E402
from test_binary_replay_host import edgy_proposal, gammas  # noqa: E402

P_SET = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128]
KINDS = ["bic", "bvs", "gprior"]
DKINDS = ["gauss", "ar1", "scaled"]


def host(t):
    return t.detach().cpu().numpy()


def dev(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device="cuda", dtype=dtype)


@pytest.fixture(scope="module")
def ctx():
    from particles_b200.device import context
    return context()


def P(t):
    from particles_b200.device import ptr
    return ptr(t)


def lib_call(ctx, name, *args):
    from particles_b200 import _lib
    _lib.check(getattr(ctx.lib, name)(ctx.handle, *args))


class DevDesc:
    """A binary_replay.Desc on the device: the smcb_vs_desc the kernels take."""

    def __init__(self, d):
        from particles_b200 import _lib
        self.xtx, self.xty = dev(d.xtx), dev(d.xty)
        self.c = _lib.VsDesc(d.p, d.use_ldet, self.xtx.data_ptr(), self.xty.data_ptr(), d.vm2, d.coef_len,
                             d.coef_log, d.coef_in_log, d.gw, d.lq, d.l1q)


def vs_call(ctx, d, gam, kmax, epn):
    """smcb_vs_loglik with every output: ({name: host array}, err)."""
    dd = DevDesc(d)
    g = dev(np.asarray(gam, dtype=bool), torch.bool)
    n = g.shape[0]
    outs = {k: torch.full((n,), 12345.0, dtype=torch.float64, device="cuda")
            for k in ("len_gam", "ldet", "wtw", "lprior", "llik", "lpost")}
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    lib_call(ctx, "smcb_vs_loglik", C.byref(dd.c), P(g), n, int(kmax), d.vm2, float(epn),
             *[P(outs[k]) for k in ("len_gam", "ldet", "wtw", "lprior", "llik", "lpost")], P(err))
    return {k: host(v) for k, v in outs.items()}, int(err.item())


def check_vs(tag, d, gam, got, epn, wpc, want=None):
    """Every output of smcb_vs_loglik against vs_ld; rows whose in_log is within its bound of 0 are left to the
    caller.  Returns the long-double result."""
    want = br.vs_ld(d, gam, epn) if want is None else want
    np.testing.assert_array_equal(got["len_gam"], want["len_gam"], err_msg=tag + " len_gam")
    np.testing.assert_array_equal(got["lprior"], want["lprior"], err_msg=tag + " lprior")
    ok = want["ok"]
    br.assert_close(tag + " ldet", got["ldet"][ok], want["ldet"][ok], want["b_ldet"][ok], wpc=None)
    br.assert_close(tag + " wtw", got["wtw"][ok], want["wtw"][ok], want["b_wtw"][ok])
    f = ok & ~want["near0"]
    idx = np.flatnonzero(f)
    for name in ("llik", "lpost"):
        w = want[name] if name == "llik" else br.post_ld(want["lprior"], want["llik"], want["b_llik"], epn)[0]
        b = want["b_" + name] if name == "llik" else br.post_ld(want["lprior"], want["llik"], want["b_llik"], epn)[1]
        try:
            br.assert_close(f"{tag} {name}", got[name][idx], w[idx], b[idx])
        except AssertionError as e:
            j = int(idx[np.argmax(~(np.abs(got[name][idx] - w[idx].astype(np.float64)) <= b[idx]))])
            raise AssertionError(f"{e} -- particle {j}, CTA {j // wpc}, warp {j % wpc}") from None
    if not epn > 0:
        np.testing.assert_array_equal(got["lpost"], got["lprior"], err_msg=tag + " lpost at epn 0")
    assert not np.isnan(got["llik"][ok & ~want["near0"]]).any()
    return want


# ------------------------------------------------------------------------------------ smcb_vs_loglik
@pytest.mark.parametrize("p", P_SET)
@pytest.mark.parametrize("kind", KINDS)
def test_vs_loglik_word_edges(ctx, kind, p):
    """All three designs (Gaussian, AR(1) rho = 0.995, column scales 10^U(-3, 3)); rows with |gamma| = 0, 1, p - 1, p,
    only the last coordinate, only coordinates >= 96, random densities; epn in {0, 0.37, 1}; q in {0.5, 0.02, 0, 1}."""
    for di, dk in enumerate(DKINDS):
        X, y = br.design(dk, p, seed=100 * p + di)
        gam = gammas(p, 67, p + di)
        kmax = int(gam.sum(axis=1).max())
        assert kmax == p
        wpc = br.bin_warps(kmax)
        n = gam.shape[0]
        assert n > wpc and n % wpc != 0                      # several CTAs, a partial last one
        chol = None
        for qi, q in enumerate((0.5, 0.02, 0.0, 1.0)):
            d = br.model_desc(kind, X, y, q=q)
            chol = br.chol_ld(gam, d.xtx, d.xty, d.vm2) if chol is None else chol
            want = br.vs_ld(d, gam, 0.0, chol=chol)
            for epn in ((0.0, 0.37, 1.0) if qi == 0 else (0.37,)):
                got, err = vs_call(ctx, d, gam, kmax, epn)
                assert err == 0
                check_vs(f"p={p} ({br.words(p)} words, {wpc} warps) {kind}/{dk} q={q} epn={epn}", d, gam, got, epn,
                         wpc, want)
    print(f"p={p}: words {br.words(p)}, {br.bin_warps(p)} warps per CTA")


KMAX_SET = [77, 78, 83, 84, 90, 91, 99, 100, 111, 112, 128]


@pytest.mark.parametrize("kmax", KMAX_SET)
def test_vs_loglik_warp_tiers(ctx, kmax):
    """p = 128: a batch where every warp of every CTA has |gamma| = kmax (adjacent triangles full) and a mixed batch
    whose largest |gamma| is kmax, at the tiers' both sides."""
    p = 128
    wpc = br.bin_warps(kmax)
    X, y = br.design("ar1" if kmax % 2 else "gauss", p, seed=kmax)
    r = np.random.RandomState(kmax)
    full = np.zeros((2 * wpc + 1, p), dtype=bool)
    for i in range(full.shape[0]):
        full[i, r.choice(p, kmax, replace=False)] = True
    mixed = r.rand(3 * wpc + 2, p) < r.uniform(0.05, 0.6, (3 * wpc + 2, 1))
    mixed[:, :] &= np.cumsum(mixed, axis=1) <= kmax
    mixed[1] = False
    mixed[1, r.choice(p, kmax, replace=False)] = True
    for tag, gam in (("full", full), ("mixed", mixed)):
        assert int(gam.sum(axis=1).max()) == kmax and gam.shape[0] % wpc != 0
        for kind in KINDS:
            d = br.model_desc(kind, X, y)
            got, err = vs_call(ctx, d, gam, kmax, 0.37)
            assert err == 0
            check_vs(f"kmax={kmax} ({wpc} warps, {br.bin_smem(kmax, wpc)} B) {tag} {kind}", d, gam, got, 0.37, wpc)
    print(f"kmax={kmax}: {wpc} warps per CTA, {br.bin_smem(kmax, wpc)} bytes of shared memory")


def dup_design(p, d1, d2, seed):
    """A Gaussian design whose column d2 repeats column d1 = +-1 on 16 rows (X^T X's pivot of the pair is 16 and the
    second copy's is 16 - 4^2 = 0 in any precision when no column below d1 is selected); X^T X in long double, so
    the copies' rows and columns are bit-identical."""
    X, y = br.design("gauss", p, seed=seed)
    r = np.random.RandomState(seed)
    X[:, d1] = 0.0
    X[r.choice(X.shape[0], 16, replace=False), d1] = r.choice([-1.0, 1.0], 16)
    X[:, d2] = X[:, d1]
    xtx = (X.T.astype(br.LD) @ X.astype(br.LD)).astype(np.float64)
    xty = (X.T.astype(br.LD) @ y.astype(br.LD)).astype(np.float64)
    assert np.array_equal(xtx[d1], xtx[d2]) and np.array_equal(xtx, xtx.T)
    return X, y, xtx, xty


@pytest.mark.parametrize("kind", ["bic", "gprior"])
@pytest.mark.parametrize("p", [40, 128])
def test_vs_loglik_duplicated_column(ctx, kind, p):
    """A row selecting both copies with nothing below the first gets llik = -inf, NaN ldet / wtw and err bit 1 (and
    the Python layer raises LinAlgError); a row selecting both above other columns has a pivot at rounding level
    (either sign, in any precision): its llik is -inf or finite, never NaN; the other rows are unaffected."""
    d1, d2 = 5, p - 3
    X, y, xtx, xty = dup_design(p, d1, d2, p)
    base = br.model_desc(kind, X, y, lamb=1.0)             # X^T X is singular: no full-model sigma^2
    d = br.Desc(xtx, xty, 0, 0.0, base.coef_len, base.coef_log, base.coef_in_log, base.gw)
    r = np.random.RandomState(p)
    gam = r.rand(50, p) < 0.4
    gam[:10, :d1] = False
    gam[:10, d1] = gam[:10, d2] = True                     # exact zero pivot
    gam[10:20, d1] = gam[10:20, d2] = True                 # rounding-level pivot
    gam[10:20, 0] = True
    gam[20:, d2] = False                                   # positive definite
    got, err = vs_call(ctx, d, gam, int(gam.sum(axis=1).max()), 0.5)
    want = br.vs_ld(d, gam, 0.5)
    assert err & 1 and not err & 2
    assert not want["ok"][:10].any() and want["ok"][20:].all()
    assert np.all(got["llik"][:10] == -np.inf) and np.isnan(got["ldet"][:10]).all() and np.isnan(got["wtw"][:10]).all()
    assert np.all(got["lpost"][:10] == -np.inf)
    assert not np.isnan(got["llik"]).any()
    assert np.all((got["llik"][10:20] == -np.inf) | np.isfinite(got["llik"][10:20]))
    wpc = br.bin_warps(int(gam.sum(axis=1).max()))
    rest = np.arange(20, 50)
    check_vs(f"dup p={p} {kind}", d, gam[rest], {k: v[rest] for k, v in got.items()}, 0.5, wpc)
    from particles_b200 import binary_smc as bs
    with pytest.raises(np.linalg.LinAlgError):
        bs.chol_and_friends(gam[:12], xtx, xty, 0.0)
    print(f"dup p={p} {kind}: rows above other columns give {int(np.sum(got['llik'][10:20] == -np.inf))} of 10 -inf")


def test_vs_loglik_k_above_kmax(ctx):
    """A row with more selected coordinates than kmax: err bit 2, NaN ldet / wtw / llik for it, the others exact;
    the Python layer raises ValueError."""
    p = 65
    X, y = br.design("gauss", p, seed=1)
    d = br.model_desc("bvs", X, y)
    gam = gammas(p, 21, 2)
    k = gam.sum(axis=1)
    kmax = int(k.max()) - 1
    got, err = vs_call(ctx, d, gam, kmax, 0.5)
    assert err == 2
    over = k > kmax
    assert over.any() and (~over).any()
    for name in ("ldet", "wtw", "llik", "lpost"):
        assert np.isnan(got[name][over]).all(), name
    check_vs("k <= kmax rows", d, gam[~over], {n: v[~over] for n, v in got.items()}, 0.5, br.bin_warps(kmax))
    from particles_b200 import binary_smc as bs
    with pytest.raises(ValueError):
        bs._raise_on(torch.full((1,), err, dtype=torch.int32))


@pytest.mark.parametrize("p", [33, 128])
def test_vs_loglik_bic_exact_fit(ctx, p):
    """y in the span of three columns: rows that contain them have in_log = y^T y - w^T w at the rounding level of
    y^T y.  There the kernel returns -(coef_len k + coef_log log(in_log)) of its own rounded in_log, as the reference's
    NumPy does: NaN where it rounds below 0, +inf at 0, else at least -coef_len k - coef_log log(2 b_in).  Pinned;
    every other row is inside the bound."""
    X, _ = br.design("gauss", p, seed=p)
    S = [0, p // 2, p - 1]
    y = X[:, S] @ np.array([1.5, -2.0, 0.75])
    d = br.model_desc("bic", X, y)
    gam = gammas(p, 40, 9)
    gam[:15, S] = True
    got, err = vs_call(ctx, d, gam, int(gam.sum(axis=1).max()), 1.0)
    assert err == 0
    want = br.vs_ld(d, gam, 1.0)
    contains = gam[:, S].all(axis=1)
    assert np.array_equal(want["near0"], contains) and contains.sum() >= 15
    check_vs(f"exact fit p={p}", d, gam, got, 1.0, br.bin_warps(int(gam.sum(axis=1).max())), want)
    ll = got["llik"][contains]
    floor = -(d.coef_len * want["len_gam"][contains] + d.coef_log * np.log(2 * want["b_in"][contains]))
    assert np.all(np.isnan(ll) | (ll == np.inf) | (ll >= floor))
    print(f"exact fit p={p}: {int(np.isnan(ll).sum())} NaN, {int((ll == np.inf).sum())} +inf, "
          f"{int(np.isfinite(ll).sum())} finite of {len(ll)}")


# ------------------------------------------------------------------------------------ smcb_nested_logistic
def nl_call(ctx, c, edgy, n, draw, x=None, u=None):
    cd, ed = dev(c), dev(np.asarray(edgy, np.uint8), torch.uint8)
    xx = dev(np.asarray(x, dtype=bool), torch.bool) if x is not None else torch.empty((n, len(edgy)), dtype=torch.bool,
                                                                                       device="cuda")
    lp = torch.empty(n, dtype=torch.float64, device="cuda")
    ud = None if u is None else dev(u)
    lib_call(ctx, "smcb_nested_logistic", len(edgy), P(cd), P(ed), n, int(draw), P(xx), P(ud), P(lp))
    return host(xx), host(lp)


def check_nl_draw(tag, c, edgy, u, x, lp):
    _, dec, mism = br.nl_replay_draw(c, edgy, u, follow=x)
    if mism.any():
        j, i = np.argwhere(mism)[0]
        raise AssertionError(f"{tag}: particle {j} (CTA {j // br.NL_BLOCK}) coordinate {i}: bit {int(x[j, i])} but "
                             f"u = {u[i, j]!r} decides the other ({int(mism.sum())} bits)")
    _, lo, hi = br.nl_ld(c, edgy, x)
    want, b = br.nl_logpdf(x, lo, hi)
    br.assert_close(tag + " logpdf", lp, want, b)
    return dec


@pytest.mark.parametrize("ckind", ["random", "saturated", "overflow"])
@pytest.mark.parametrize("p", P_SET)
def test_nested_logistic(ctx, p, ckind):
    """Injected uniforms (0, 1 - 2^-53 and u == pr on the edgy coordinates among them), logpdf of arbitrary rows,
    and the device's own draws for calls 0 and 1 after ctx.seed, replayed with the rvs layout."""
    c, edgy = edgy_proposal(p, p, ckind)
    k = 3
    n = 128 * k + 37
    assert -(-n // br.NL_BLOCK) == k + 1                   # a partial last CTA
    r = np.random.RandomState(p)
    u = r.rand(p, n)
    u[:, 0], u[:, 1] = 0.0, 1.0 - 2.0 ** -53
    ei = np.flatnonzero(edgy)
    u[ei, 2] = c[ei, ei]                                   # u == pr exactly: the strict < gives 0
    u[ei, n - 1] = c[ei, ei]
    x, lp = nl_call(ctx, c, edgy, n, True, u=u)
    dec = check_nl_draw(f"p={p} {ckind} injected", c, edgy, u, x, lp)
    assert dec.mean() > 0.99
    assert not x[2, ei].any() and not x[n - 1, ei].any()
    assert not x[0, ei][c[ei, ei] == 0.0].any() and x[1, ei][c[ei, ei] == 1.0].all()
    xa = r.rand(n, p) < 0.5                                 # arbitrary rows, bits of probability 0 included
    _, lpa = nl_call(ctx, c, edgy, n, False, x=xa)
    _, lo, hi = br.nl_ld(c, edgy, xa)
    want, b = br.nl_logpdf(xa, lo, hi)
    br.assert_close(f"p={p} {ckind} logpdf of arbitrary rows", lpa, want, b)
    seed = 0xB1A5 + 7 * p
    ctx.seed(seed)                                          # resets the API call counter: calls 0, 1, ...
    for call in (0, 1):
        xd, lpd = nl_call(ctx, c, edgy, n, True)
        ud = br.rvs_uniforms(n, p, call, seed)
        check_nl_draw(f"p={p} {ckind} device draw, call {call}", c, edgy, ud, xd, lpd)
    print(f"p={p} {ckind}: {br.words(p)} words, {n} particles in {-(-n // br.NL_BLOCK)} CTAs")


# ------------------------------------------------------------------------------------ smcb_binary_wf_move
def move_inputs(ctx, d, c, edgy, M, epn, seed):
    """Start rows drawn from the proposal (injected uniforms), with the kernel's own target values."""
    p = len(edgy)
    u0 = np.random.RandomState(seed).rand(p, M)
    x0, _ = nl_call(ctx, c, edgy, M, True, u=u0)
    got, err = vs_call(ctx, d, x0, max(int(x0.sum(axis=1).max()), 0), epn)
    return x0, got["lprior"], got["llik"], got["lpost"], err


def move_call(ctx, d, c, edgy, M, P_, epn, x0, lpr0, ll0, lp0, up=None, ua=None):
    dd = DevDesc(d)
    p = len(edgy)
    cd, ed = dev(c), dev(np.asarray(edgy, np.uint8), torch.uint8)
    out = {"theta": torch.empty((P_ * M, p), dtype=torch.bool, device="cuda")}
    for k in ("lprior", "llik", "lpost"):
        out[k] = torch.empty(P_ * M, dtype=torch.float64, device="cuda")
    pb = torch.empty((P_ - 1, M), dtype=torch.float64, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    ins = [dev(np.asarray(x0, bool), torch.bool), dev(lpr0), dev(ll0), dev(lp0),   # alive until the launch is read
           None if up is None else dev(up), None if ua is None else dev(ua)]
    lib_call(ctx, "smcb_binary_wf_move", C.byref(dd.c), P(cd), P(ed), M, P_, float(epn), *[P(t) for t in ins],
             P(out["theta"]),
             P(out["lprior"]), P(out["llik"]), P(out["lpost"]), P(pb), P(err))
    o = {k: host(v).reshape((P_, M) + v.shape[1:]) for k, v in out.items()}
    return o, host(pb), int(err.item())


def check_move(tag, d, c, edgy, epn, o, pb, M, P_, wpc, up=None, ua=None, seed=None, call=0, chains=None, steps=None):
    """Replay the generations ``steps`` (default all) for ``chains`` (default: every chain when there are few, else
    the CTA edges, the first 8 and a random 600).  Returns (accepted, undecided, chain-steps checked)."""
    p = len(edgy)
    if chains is None:
        if M * P_ <= 4000:
            chains = np.arange(M)
        else:
            edges = np.arange(0, M, wpc)
            chains = np.unique(np.concatenate([np.arange(min(8, M)), edges, edges - 1, [M - 1],
                                               np.random.RandomState(M).randint(0, M, 600)]))
            chains = chains[(chains >= 0) & (chains < M)]
    steps = range(1, P_) if steps is None else steps
    n_acc = n_und = n = 0
    for s in steps:
        if up is not None:
            us, uas = up[s - 1][:, chains], ua[s - 1][chains]
        else:
            us = br.prop_uniforms(M, p, s, call, seed)[:, chains]
            uas = br.acc_uniforms(M, s, call, seed)[chains]
        prev = {k: o[k][s - 1][chains] for k in ("theta", "lprior", "llik", "lpost")}
        cur = {k: o[k][s][chains] for k in ("theta", "lprior", "llik", "lpost")}
        res = br.check_generation(s, d, c, edgy, epn, prev, cur, pb[s - 1][chains], us, uas, wpc, chains=chains)
        n_acc += int(res["accepted"].sum())
        n_und += res["undecided"]
        n += len(chains)
    return n_acc, n_und, n


MOVE_P = [1, 33, 65, 77, 78, 84, 91, 100, 112, 128]


def move_cases():
    cases = []
    for i, p in enumerate(MOVE_P):
        wpc = br.bin_warps(p)
        cases.append((p, max(wpc - 1, 1), 9, 0.4, "injected"))
        cases.append((p, wpc + 1, 9, (0.0, 1.0)[i % 2], "device"))
        cases.append((p, 1, 2, 1.0, ("injected", "device")[i % 2]))
    cases += [(33, 4097, 9, 0.4, "device"), (128, 4097, 2, 1.0, "injected"), (65, 4097, 2, 0.0, "device")]
    return cases


@pytest.mark.parametrize("p,M,P_,epn,noise", move_cases())
def test_wf_move(ctx, p, M, P_, epn, noise):
    """Every warp tier of the move (3 warps and 198 KB at p >= 112), chains short of a CTA, one past it and 4097."""
    wpc = br.bin_warps(p)
    kind = ("bvs", "gprior", "bic")[p % 3]
    X, y = br.design(("gauss", "ar1", "scaled")[p % 3], p, seed=p)
    d = br.model_desc(kind, X, y)
    c, edgy = edgy_proposal(p, p + 1)
    x0, lpr0, ll0, lp0, err = move_inputs(ctx, d, c, edgy, M, epn, p + M)
    assert err == 0
    up = ua = None
    seed = None
    if noise == "injected":
        r = np.random.RandomState(p + M + P_)
        up, ua = r.rand(P_ - 1, p, M), r.rand(P_ - 1, M)
        o, pb, err = move_call(ctx, d, c, edgy, M, P_, epn, x0, lpr0, ll0, lp0, up, ua)
    else:
        seed = 0x5EED + p * M + P_
        ctx.seed(seed)
        o, pb, err = move_call(ctx, d, c, edgy, M, P_, epn, x0, lpr0, ll0, lp0)
    assert err == 0
    assert np.array_equal(o["theta"][0], x0) and np.array_equal(o["lpost"][0], lp0)
    n_acc, n_und, n = check_move(f"p={p}", d, c, edgy, epn, o, pb, M, P_, wpc, up, ua, seed)
    assert n_und <= 0.01 * n
    print(f"move p={p} ({br.words(p)} words, {wpc} warps, {br.bin_smem(p, wpc)} B) M={M} "
          f"({-(-M // wpc)} CTAs) P={P_} epn={epn} {noise}: {n_acc} of {n} accepted, {n_und} undecided")


@pytest.mark.parametrize("P_,steps", [(257, None), (4099, list(range(1, 24)) + list(range(250, 264))
                                                    + list(range(510, 516)) + list(range(1020, 1030))
                                                    + list(range(4090, 4099)))])
def test_wf_move_long_chains(ctx, P_, steps):
    """p = 33, M = 3, device draws: the step field of the counter runs past 8 bits (and past 12 at P = 4099)."""
    p, M, epn = 33, 3, 0.0
    wpc = br.bin_warps(p)
    X, y = br.design("gauss", p, seed=11)
    d = br.model_desc("bvs", X, y)
    c, edgy = edgy_proposal(p, 12)
    x0, lpr0, ll0, lp0, _ = move_inputs(ctx, d, c, edgy, M, epn, 13)
    seed = 0xC4A1 + P_
    ctx.seed(seed)
    o, pb, err = move_call(ctx, d, c, edgy, M, P_, epn, x0, lpr0, ll0, lp0)
    assert err == 0
    n_acc, n_und, n = check_move(f"P={P_}", d, c, edgy, epn, o, pb, M, P_, wpc, seed=seed, steps=steps)
    assert 0 < n_acc < n and n_und <= 0.01 * n + 1
    print(f"long chain P={P_}: {n} chain-steps checked, {n_acc} accepted, {n_und} undecided")


def test_wf_move_special_rows_and_duplicated_column(ctx):
    """BIC with a duplicated column at coordinates 0 and 1 (a proposal selecting both fails the factorisation: llik
    -inf, pb = 0, rejected, err bit 1, and wf_move raises LinAlgError); start rows with lpost0 = -inf (against a -inf
    proposal: pb NaN, rejected; against a finite one: pb = 1, accepted) and a NaN lpost0 (pb NaN, rejected, every
    step)."""
    p, M, P_, epn = 33, 40, 6, 0.4
    wpc = br.bin_warps(p)
    X, y, xtx, xty = dup_design(p, 0, 1, 21)
    base = br.model_desc("bic", X, y)
    d = br.Desc(xtx, xty, 0, 0.0, base.coef_len, base.coef_log, base.coef_in_log, 1.0)
    c, edgy = edgy_proposal(p, 22)
    c[0, :], c[1, :] = 0.0, 0.0
    c[0, 0], c[1, 1] = 0.5, 0.5
    edgy[0] = edgy[1] = True                               # each copy selected with probability 1/2
    r = np.random.RandomState(23)
    x0 = r.rand(M, p) < 0.3
    x0[:, 1] = False
    got, err = vs_call(ctx, d, x0, int(x0.sum(axis=1).max()), epn)
    assert err == 0
    lpr0, ll0, lp0 = got["lprior"], got["llik"], got["lpost"]
    lp0[0] = lp0[1] = -np.inf
    lp0[2] = np.nan
    up, ua = r.rand(P_ - 1, p, M), r.rand(P_ - 1, M)
    up[0, :2, 0] = 0.0                                     # chain 0, step 1: both copies: a -inf proposal
    up[0, :2, 1] = 0.9                                     # chain 1, step 1: neither: a finite proposal
    o, pb, err = move_call(ctx, d, c, edgy, M, P_, epn, x0, lpr0, ll0, lp0, up, ua)
    assert err & 1
    assert np.isnan(pb[0, 0]) and np.array_equal(o["theta"][1, 0], x0[0])          # -inf vs -inf: rejected
    assert pb[0, 1] == 1.0 and o["lpost"][1, 1] > -np.inf                          # -inf vs finite: accepted
    assert np.isnan(pb[:, 2]).all() and all(np.array_equal(o["theta"][s, 2], x0[2]) for s in range(P_))
    both = up[:, 0, :] < 0.5
    both &= up[:, 1, :] < 0.5
    assert both[:, 3:].any()
    assert np.all(pb[:, 3:][both[:, 3:]] == 0.0)                                   # failed factorisation: rejected
    check_move("dup", d, c, edgy, epn, o, pb, M, P_, wpc, up, ua)
    from particles_b200 import binary_smc as bs, distributions as dists
    from particles_b200.smc_samplers import ThetaParticles
    m = bs.BIC(data=(X, y))
    m.prior = dists.IID(bs.Bernoulli(0.5), p)
    x = ThetaParticles(theta=dev(x0, torch.bool), lprior=dev(lpr0), llik=dev(ll0), lpost=dev(lp0))
    x.shared["proposal"] = bs.NestedLogistic(c, edgy)
    with pytest.raises(np.linalg.LinAlgError):
        m.wf_move(x, epn, P_, noise=(up, ua))


@pytest.mark.parametrize("p", [33, 128])
def test_binary_metropolis_step(ctx, p):
    """BinaryMetropolis.step (the non-fused move) with injected noise: theta where decided, the three scores and the
    mean acceptance inside the bounds."""
    from particles_b200 import binary_smc as bs, distributions as dists
    from particles_b200.smc_samplers import ThetaParticles
    N, epn = 3 * 128 + 5, 0.4
    X, y = br.design("gauss", p, seed=p + 5)
    m = bs.BayesianVS(data=(X, y), prior=dists.IID(bs.Bernoulli(0.5), p))
    d = br.Desc.of_model(m)
    c, edgy = edgy_proposal(p, p + 6)
    r = np.random.RandomState(p)
    x0 = r.rand(N, p) < 0.3
    x = ThetaParticles(theta=dev(x0, torch.bool))
    m.target(x, epn)
    prev = {"theta": x0, "lprior": host(x.lprior).copy(), "llik": host(x.llik).copy(), "lpost": host(x.lpost).copy()}
    x.shared["proposal"] = bs.NestedLogistic(c, edgy)
    up, ua = r.rand(p, N), r.rand(N)
    acc = bs.BinaryMetropolis().step(x, lambda xp: m.target(xp, epn), noise=(up, ua))
    cur = {"theta": host(x.theta), "lprior": host(x.lprior), "llik": host(x.llik), "lpost": host(x.lpost)}
    res = br.check_generation(1, d, c, edgy, epn, prev, cur, None, up, ua, 1)
    assert res["undecided"] == 0 and len(res["known"]) == N
    mean = float(np.mean(res["pb"].astype(np.float64)))
    b = float(np.sum(res["b_pb"])) / N + 4 * br.gamma(N) * mean
    assert abs(float(host(acc)[0]) - mean) <= b, (float(host(acc)[0]), mean, b)
    print(f"BinaryMetropolis.step p={p}: {int(res['accepted'].sum())} of {N} accepted, mean pb {mean:.4f}")
