"""GPU parity tests for the L0 numerics (weights algebra, scan, search, resampling,
distributions) -- all calls go through the C-ABI of libsmcb.so (via the ctypes host
layer).  Checker = the oracle + golden vectors produced by the live reference.

Bars: bit-exact for ancestor indices and anything integer; for fp64 the tolerances
are written next to each assert (transcendentals differ from NumPy's by <= a few ulp).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import cext  # noqa: E402
from oracle import smc_numpy as orc  # noqa: E402
import philox_ref  # noqa: E402

LW_CASES = ["gauss_1000", "equal_257", "dominant_513", "neginf_777", "nan_300", "single_1",
            "wide_4099", "tiny_2"]
RS_CASES = ["dirichlet_1000", "skewed_513", "M_lt_N", "M_gt_N", "zeros_300", "dominant_64",
            "equal_1025", "n7"]
SCHEMES = ["systematic", "stratified", "multinomial", "residual"]


@pytest.fixture(scope="module")
def pb():
    import particles_b200 as pb
    return pb


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def host(t):
    return t.detach().cpu().numpy()


# --------------------------------------------------------------------------- RNG
def test_philox_matches_host_reference(pb):
    """The device generator is Philox4x32-10 with the documented counter layout
    (known-answer vectors are checked on the CPU side in test_host.py)."""
    from particles_b200 import _lib
    from particles_b200.device import context, empty, ptr
    ctx = context()
    ctx.seed(0x1234567890ABCDEF)
    u = empty(1001)
    _lib.check(ctx.lib.smcb_uniform(ctx.handle, ptr(u), 1001))
    ref = philox_ref.uniforms(1001, 0, 0x1234567890ABCDEF, w3=philox_ref.PURPOSE_API)
    assert np.array_equal(host(u), ref)           # integer pipeline + exact scaling: bit-exact
    z = empty(1001)
    _lib.check(ctx.lib.smcb_standard_normal(ctx.handle, ptr(z), 1001))
    refz = philox_ref.normals(1001, 1, 0x1234567890ABCDEF, w3=philox_ref.PURPOSE_API)
    np.testing.assert_allclose(host(z), refz, rtol=1e-13, atol=1e-15)   # log/sincos: few ulp
    big = empty(2_000_000)
    _lib.check(ctx.lib.smcb_standard_normal(ctx.handle, ptr(big), big.shape[0]))
    b = host(big)
    assert abs(b.mean()) < 5 / np.sqrt(b.size) and abs(b.var() - 1) < 5 * np.sqrt(2 / b.size)
    assert abs((b ** 4).mean() - 3) < 0.05


def test_device_math(pb):
    """csrc/smcb_math.cuh (the step kernel's own exp / log / sincos) against NumPy: <= 2 ulp."""
    from particles_b200 import _lib
    from particles_b200.device import context, empty, ptr
    ctx = context()
    r = np.random.RandomState(0)

    def run(fn, x):
        xd, out = dev(x), empty(x.shape[0])
        _lib.check(ctx.lib.smcb_device_math(ctx.handle, fn, ptr(xd), ptr(out), x.shape[0]))
        return host(out)

    x = np.concatenate([r.uniform(-745, 5, 200_000), r.uniform(-2, 2, 200_000),
                        [0.0, -0.0, -708.0, -1e-300, 1e-17, 700.0, -np.inf, -800.0]])
    e = run(0, x)
    ref = np.exp(x)
    ok = x >= -708
    np.testing.assert_allclose(e[ok], ref[ok], rtol=4.5e-16)            # 2 ulp
    assert np.all(e[~ok] == 0.0)                                        # flushed tail < 3e-308
    assert np.isnan(run(0, np.array([np.nan, 1.0]))[0])
    u = np.concatenate([r.rand(300_000), 1 - 2.0 ** -np.arange(1, 54), 2.0 ** -np.arange(1, 55),
                        r.uniform(0, 1e6, 1000)])
    u = u[u > 0]
    np.testing.assert_allclose(run(1, u), np.log(u), rtol=4.5e-16, atol=2.3e-16)
    v = np.concatenate([r.rand(300_000), np.arange(0, 1, 1 / 64), [0.0, 0.25, 0.5, 0.75, 1 - 2.0 ** -53]])
    import mpmath
    # NumPy rounds the argument 2*pi*v first (error up to ~1e-15): loose here, strict vs mpmath below
    np.testing.assert_allclose(run(2, v), np.sin(2 * np.pi * v), atol=2e-15, rtol=0)
    np.testing.assert_allclose(run(3, v), np.cos(2 * np.pi * v), atol=2e-15, rtol=0)
    exact = [float(mpmath.sin(2 * mpmath.pi * mpmath.mpf(float(t)))) for t in v[:2000]]
    np.testing.assert_allclose(run(2, v)[:2000], exact, rtol=0, atol=1e-15)    # <= 4.5 ulp of 1
    # the table-assisted family the step kernels run on (fn 4..8; tables staged into shared memory by TMA)
    e = run(4, x)
    np.testing.assert_allclose(e[ok], ref[ok], rtol=4.5e-16)
    assert np.all(e[~ok] == 0.0) and np.isnan(run(4, np.array([np.nan, 1.0]))[0])
    # NaN with any payload, among them low words of all ones (texp adds to the exponent field of its core's result),
    # and the NaN the device itself makes of -inf - -inf
    nans = np.array([0x7FF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0x7FF0000000000001,
                     0x7FF80000FFFFFFFF], dtype=np.uint64).view(np.float64)
    for fn in (0, 4):
        assert np.isnan(run(fn, nans)).all(), (fn, run(fn, nans))
    made = dev(np.full(4, -np.inf))
    made = made - made                                                  # NaN made by the device
    out = empty(4)
    _lib.check(ctx.lib.smcb_device_math(ctx.handle, 4, ptr(made), ptr(out), 4))
    assert np.isnan(host(out)).all(), host(made).view(np.uint64)
    assert run(4, np.array([710.0, 1.0]))[0] == np.inf
    np.testing.assert_allclose(run(5, u), np.log(u), rtol=7e-16, atol=3e-19)
    np.testing.assert_allclose(run(6, v), np.sin(2 * np.pi * v), atol=2e-15, rtol=0)
    np.testing.assert_allclose(run(7, v), np.cos(2 * np.pi * v), atol=2e-15, rtol=0)
    np.testing.assert_allclose(run(6, v)[:2000], exact, rtol=0, atol=8e-16)     # <= 3.5 ulp of 1
    a = np.concatenate([r.uniform(0, 80, 200_000), 2.0 ** r.uniform(-60, 7, 100_000), [1.0, 4.0, 1e-300]])
    np.testing.assert_allclose(run(8, a), np.sqrt(a), rtol=6e-16)               # rsqrt seed + one third-order step


# ----------------------------------------------------------------------- weights
@pytest.mark.parametrize("name", LW_CASES)
def test_weights_vs_reference(pb, golden, name):
    from particles_b200 import resampling as rs
    lw_in = golden[f"w/{name}/lw_in"]
    lw = dev(lw_in.copy())
    w = rs.Weights(lw=lw)
    ref_stats, ref_W = golden[f"w/{name}/stats"], golden[f"w/{name}/W"]
    assert not np.isnan(host(lw)).any()           # NaN -> -inf in the caller's array (resampling.py:220)
    assert host(w.lw).max() == ref_stats[0]       # max is exact
    # log_mean / ESS: summation order + exp differ -> 1e-13 relative
    np.testing.assert_allclose([w.log_mean, w.ESS], ref_stats[1:], rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(host(w.W), ref_W, rtol=1e-13, atol=1e-300)
    fin = lw_in.copy()
    fin[np.isnan(fin)] = -np.inf
    lse = golden[f"w/{name}/lse"]
    np.testing.assert_allclose([rs.log_sum_exp(dev(fin)), rs.log_mean_exp(dev(fin)), rs.essl(dev(fin))],
                               lse, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(host(rs.exp_and_normalise(dev(fin))),
                               golden[f"w/{name}/exp_and_normalise"], rtol=1e-13, atol=1e-300)
    np.testing.assert_allclose(rs.log_mean_exp(dev(fin), W=dev(golden[f"w/{name}/Wn"])),
                               golden[f"w/{name}/log_mean_exp_W"][0], rtol=1e-13, atol=1e-15)


def test_weights_edge_semantics(pb):
    from particles_b200 import resampling as rs
    w = rs.Weights()
    assert w.N == 0 and not hasattr(w, "W") and not hasattr(w, "ESS") and not hasattr(w, "log_mean")
    w2 = w.add(dev(np.array([0.0, -1.0, -2.0])))
    assert w2.N == 3 and w.lw is None             # add returns a NEW object
    ref = orc.Weights(lw=np.array([0.0, -1.0, -2.0]))
    np.testing.assert_allclose([w2.ESS, w2.log_mean], [ref.ESS, ref.log_mean], rtol=1e-14)
    w3 = w2.add(dev(np.array([1.0, 1.0, 5.0])))
    ref3 = ref.add(np.array([1.0, 1.0, 5.0]))
    np.testing.assert_allclose(host(w3.W), ref3.W, rtol=1e-14)
    # all -inf and +inf inputs: NaN W / ESS / log_mean, no exception (SURVEY.md section 9.3)
    for bad in (np.full(5, -np.inf), np.array([0.0, np.inf, 1.0])):
        wb = rs.Weights(lw=dev(bad.copy()))
        assert np.isnan(wb.ESS) and np.isnan(wb.log_mean)
    # exactly equal weights, ESSrmin = 1.0 -> ESS == N up to rounding, strict < is the caller's test
    we = rs.Weights(lw=dev(np.zeros(4096)))
    assert we.ESS == 4096.0 and we.log_mean == 0.0


def test_weights_large_matches_oracle(pb):
    from particles_b200 import resampling as rs
    r = np.random.RandomState(3)
    lw = r.randn(3_000_001) * 4.0
    ref = orc.Weights(lw=lw.copy())
    w = rs.Weights(lw=dev(lw))
    np.testing.assert_allclose([w.log_mean, w.ESS], [ref.log_mean, ref.ESS], rtol=1e-12)
    np.testing.assert_allclose(host(w.W), ref.W, rtol=1e-12, atol=1e-300)
    mv = rs.wmean_and_var(w.W, dev(lw))
    refmv = orc.wmean_and_var(ref.W, lw)
    np.testing.assert_allclose([mv["mean"], mv["var"]], [refmv["mean"], refmv["var"]], rtol=1e-10)


# -------------------------------------------------------------------------- scan
@pytest.mark.parametrize("n", [1, 7, 2047, 2048, 2049, 65536 + 3, 1_000_003, 10_000_000])
def test_cumsum_monotone_deterministic(pb, n):
    from particles_b200 import resampling as rs
    r = np.random.RandomState(n % 1000)
    W = r.rand(n) ** 8
    W[r.rand(n) < 0.3] = 0.0                       # many exact zeros (ties in the CDF)
    W = W / W.sum()
    Wd = dev(W)
    c1, c2 = host(rs.cumsum(Wd)), host(rs.cumsum(Wd))
    assert np.array_equal(c1, c2)                  # a pure function of the input
    assert np.all(np.diff(c1) >= 0)                # non-decreasing by construction
    # np.cumsum is a sequential fp64 sum (error grows ~ n*eps); judge against extended precision
    ref = np.cumsum(W.astype(np.longdouble)).astype(np.float64)
    np.testing.assert_allclose(c1, ref, rtol=1e-13, atol=1e-16)    # tile prefixes add sequentially
    np.testing.assert_allclose(c1, np.cumsum(W), rtol=1e-15 * max(n, 100), atol=1e-16)
    assert abs(c1[-1] - 1.0) < 1e-13


def test_cumsum_adversarial_tiny_weights(pb):
    """Weights below 1 ulp of the running sum: the clamped scan must stay monotone."""
    from particles_b200 import resampling as rs
    n = 300_000
    W = np.full(n, 1e-25)
    W[::4099] = 1.0
    W /= W.sum()
    c = host(rs.cumsum(dev(W)))
    assert np.all(np.diff(c) >= 0)
    np.testing.assert_allclose(c, np.cumsum(W), rtol=1e-13, atol=1e-16)


# ------------------------------------------------------------------------ search
@pytest.mark.parametrize("name", RS_CASES)
def test_inverse_cdf_vs_reference(pb, golden, name):
    from particles_b200 import resampling as rs
    W, su = golden[f"rs/{name}/W"], golden[f"rs/{name}/su"]
    A = host(rs.inverse_cdf(dev(su), dev(W)))
    assert A.dtype == np.int64
    cdf = host(rs.cumsum(dev(W)))
    assert np.array_equal(A, cext.searchsorted_left(cdf, su))       # bit-exact on the device's CDF
    assert np.array_equal(A, golden[f"rs/{name}/inverse_cdf"])       # and equal to the reference here


@pytest.mark.parametrize("name", RS_CASES)
@pytest.mark.parametrize("scheme", SCHEMES)
def test_resampling_vs_reference_injected_uniforms(pb, golden, name, scheme):
    """Same W, same uniforms (in the reference's draw order) -> same ancestors."""
    from particles_b200 import resampling as rs
    W, M = golden[f"rs/{name}/W"], int(golden[f"rs/{name}/M"][0])
    u = golden[f"rs/{name}/{scheme}/u"]
    A = host(rs.rs_funcs[scheme](dev(W), M=M, u=u))
    ref = golden[f"rs/{name}/{scheme}/A"]
    assert A.shape == ref.shape and A.dtype == np.int64
    if scheme in ("systematic", "stratified"):
        assert np.array_equal(A, ref)
    else:
        # multinomial / residual go through a second scan (cumsum of -log u) whose rounding
        # differs from np.cumsum: a draw that lands within 1e-15 of a CDF value may move by one
        bad = np.flatnonzero(A != ref)
        assert bad.size <= max(1, M // 500) and np.all(np.abs(A[bad] - ref[bad]) <= 1)


@pytest.mark.parametrize("name", RS_CASES)
def test_ssp_killing_iid_vs_reference(pb, golden, golden_rs_extra, name):
    """The schemes outside the fused kernel (resampling.py:560-570, 630-697) with the reference's uniforms."""
    from particles_b200 import resampling as rs
    W, M = golden[f"rs/{name}/W"], int(golden[f"rs/{name}/M"][0])
    n, x = W.shape[0], golden_rs_extra
    A = host(rs.ssp(dev(W), M=M, u=x[f"rs/{name}/ssp/u"]))
    assert A.dtype == np.int64 and np.array_equal(A, x[f"rs/{name}/ssp/A"])     # same recursion, same bits
    A2 = host(rs.resampling("ssp", dev(W), M=M))                                  # device uniforms
    cnt = np.bincount(A2, minlength=n)
    assert A2.shape == (M,) and np.all(np.abs(cnt - M * W) < 1.0 + 1e-9) and np.all(np.diff(A2) >= 0)
    if M == n:
        K = host(rs.killing(dev(W), M=M, u=x[f"rs/{name}/killing/u"], u_multinomial=x[f"rs/{name}/killing/u_multinomial"]))
        ref = x[f"rs/{name}/killing/A"]
        bad = np.flatnonzero(K != ref)      # the multinomial stage's second scan may move a tie by one
        assert bad.size <= max(1, M // 500) and np.all(np.abs(K[bad] - ref[bad]) <= 1)
        kept = x[f"rs/{name}/killing/u"] * W.max() < W
        assert np.array_equal(K[kept], np.arange(n)[kept])
    else:
        with pytest.raises(ValueError) as e:
            rs.killing(dev(W), M=M)
        assert str(e.value) == bytes(x["rs/killing_error"]).decode()
    B = host(rs.multinomial_iid(dev(W), M=M))
    assert B.shape == (M,) and B.min() >= 0 and B.max() < n and np.all(W[B] > 0)
    a = rs.multinomial_once(dev(W), u=0.5)
    assert a == min(int(np.searchsorted(np.cumsum(W), 0.5)), n - 1)
    I = host(rs.idiotic(dev(W), M=M, u=0.5))
    assert np.array_equal(I, np.full(M, a))


def test_ssp_large_and_plugin_path(pb):
    """ssp at N = 2e5 against the oracle's restatement (same uniforms -> identical ancestors), and a filter
    run with resampling='ssp' (plugin path: fused kernels have no ssp branch)."""
    import particles_b200
    from particles_b200 import resampling as rs, state_space_models as ssm
    r = np.random.RandomState(3)
    n = 200_000
    W = orc.exp_and_normalise(r.randn(n) * 2.0)
    u = r.rand(n - 1)
    assert np.array_equal(host(rs.ssp(dev(W), u=u)), orc.ssp(W, n, u=u))
    x, y = ssm.StochVol().simulate(30)
    pf = particles_b200.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=2000, resampling="ssp", seed=3)
    pf.run()
    assert not pf.fused and np.isfinite(pf.logLt) and any(pf.summaries.rs_flags)
    # the observations are shape-(1,) CUDA tensors (StateSpaceModel.simulate): they must broadcast against the (N,)
    # particles exactly as NumPy's data[t] does -- N weights per step, and the likelihood of the fused filter
    assert pf.wgts.N == 2000 and pf.wgts.lw.shape == (2000,)
    lls = []
    for seed in range(4):
        q = particles_b200.SMC(fk=ssm.Bootstrap(ssm=ssm.StochVol(), data=y), N=20000, resampling="ssp", seed=seed)
        q.run()
        lls.append(q.logLt)
    yh = [np.atleast_1d(host(v)) for v in y]
    ref = orc.SMC(orc.Bootstrap(orc.StochVol(), yh), N=20000)
    np.random.seed(5)
    ref.run()
    assert abs(np.mean(lls) - ref.logLt) < 0.25, (lls, ref.logLt)


def test_normal_broadcasts_size_one_arguments(pb):
    """Normal.logpdf / rvs with a shape-(1,) tensor argument (what simulate() returns) against (N,) parameters."""
    from particles_b200 import distributions as dists
    loc = dev(np.linspace(-1, 1, 1000))
    d = dists.Normal(loc=loc, scale=0.5)
    y1 = dev(np.array([0.3]))
    out = host(d.logpdf(y1))
    assert out.shape == (1000,)
    np.testing.assert_allclose(out, orc.Normal(loc=host(loc), scale=0.5).logpdf(0.3), rtol=1e-13)
    with pytest.raises(ValueError):
        d.logpdf(dev(np.zeros(7)))


def test_unknown_scheme_raises(pb, golden):
    from particles_b200 import resampling as rs
    with pytest.raises(ValueError) as e:
        rs.resampling("bogus", dev(golden["rs/n7/W"]))
    assert str(e.value) == bytes(golden["rs/bogus_error"]).decode()


@pytest.mark.parametrize("scheme", ["systematic", "stratified", "multinomial"])
@pytest.mark.parametrize("n,m", [(10_000_000, 10_000_000), (1_000_003, 777_777), (5000, 20_001)])
def test_resampling_bitexact_on_own_cdf_large(pb, scheme, n, m):
    """Full-size property test: ancestors == np.searchsorted(device CDF, device su)."""
    from particles_b200 import resampling as rs
    r = np.random.RandomState(11)
    lw = r.randn(n) * 3.0
    W = orc.exp_and_normalise(lw)
    Wd = dev(W)
    nu = {"systematic": 1, "stratified": m, "multinomial": m + 1}[scheme]
    u = r.rand(nu)
    A, scratch = rs._resample(scheme, Wd, m, u=u, return_scratch=True)
    A = host(A)
    cdf = host(scratch[:n])
    assert np.array_equal(cdf, host(rs.cumsum(Wd)))
    if scheme == "multinomial":
        off = (n + 1) & ~1
        z = host(scratch[off: off + m + 1])
        su = z[:-1] / z[-1]
        np.testing.assert_allclose(z, np.cumsum(-np.log(u)), rtol=1e-12)
    else:
        su = (u + np.arange(m)) / m               # the reference's expression, IEEE-exact on both sides
    ref = np.minimum(np.searchsorted(cdf, su, side="left"), n - 1)
    assert np.array_equal(A, ref)
    assert np.all(np.diff(A) >= 0)                 # sorted output (resampling.py:548-552)
    if scheme == "systematic" and m == n:
        cnt = np.bincount(A, minlength=n)
        assert np.all(np.abs(cnt - n * W) < 1.0 + 1e-6)      # offspring in {floor, ceil}(N W)
        # vs the reference's sequential inverse_cdf on np.cumsum: only 1-ulp CDF ties may differ
        mism = np.count_nonzero(A != orc.inverse_cdf(su, W))
        assert mism <= n * 1e-6


def test_residual_structure_large(pb):
    from particles_b200 import resampling as rs
    r = np.random.RandomState(5)
    n = 200_003
    W = orc.exp_and_normalise(r.randn(n) * 2.0)
    u = r.rand(n + 1)
    A = host(rs.residual(dev(W), u=u))
    ip = np.floor(n * W).astype(np.int64)
    sip = int(ip.sum())
    assert np.array_equal(A[:sip], np.arange(n).repeat(ip))        # deterministic part: exact
    ref = orc.residual(W, n, u=u)
    bad = np.flatnonzero(A != ref)
    assert bad.size <= n // 1000 and np.all(np.abs(A[bad] - ref[bad]) <= 1)
    assert np.all(np.diff(A[sip:]) >= 0)


def test_gather(pb):
    from particles_b200 import _lib
    from particles_b200.device import context, empty, ptr
    ctx = context()
    r = np.random.RandomState(0)
    X = r.randn(3, 1001)
    A = r.randint(0, 1001, size=777).astype(np.int64)
    out = empty((3, 777))
    Xd, Ad = dev(X), dev(A)                      # keep the tensors alive across the launch
    _lib.check(ctx.lib.smcb_gather(ctx.handle, ptr(Xd), 1001, ptr(Ad), 777, 3, ptr(out)))
    assert np.array_equal(host(out), X[:, A])
    Xr = np.ascontiguousarray(X.T)
    Xrd = dev(Xr)
    out2 = empty((777, 3))
    _lib.check(ctx.lib.smcb_gather_rows(ctx.handle, ptr(Xrd), 1001, ptr(Ad), 777, 3, ptr(out2)))
    assert np.array_equal(host(out2), Xr[A])


# ----------------------------------------------------------------- distributions
def test_normal_vs_reference(pb, golden):
    from particles_b200 import distributions as dists
    g = golden
    x, loc, scale = g["d/normal/x"], g["d/normal/loc"], g["d/normal/scale"]
    lp = host(dists.Normal(loc=dev(loc), scale=dev(scale)).logpdf(dev(x)))
    np.testing.assert_allclose(lp, g["d/normal/logpdf"], rtol=1e-14, atol=1e-15)   # 1 log + 1 div
    lp2 = host(dists.Normal(loc=0.3, scale=1.7).logpdf(dev(x)))
    np.testing.assert_allclose(lp2, g["d/normal/logpdf_scalar"], rtol=1e-14, atol=1e-15)
    # rvs with the reference's own normals: loc + scale*z is pure IEEE arithmetic -> bit-exact
    xs = host(dists.Normal(loc=dev(loc), scale=dev(scale)).rvs(size=500, z=g["d/normal/rvs_z"]))
    assert np.array_equal(xs, g["d/normal/rvs"])


def test_mvnormal_vs_reference(pb, golden):
    from particles_b200 import distributions as dists
    g = golden
    cov, locs, xs, sc = g["d/mvn/cov"], g["d/mvn/loc"], g["d/mvn/x"], g["d/mvn/scale"]
    lp = host(dists.MvNormal(loc=dev(locs), cov=cov).logpdf(dev(xs)))
    np.testing.assert_allclose(lp, g["d/mvn/logpdf"], rtol=1e-13)
    lp2 = host(dists.MvNormal(loc=dev(locs), scale=sc, cov=cov).logpdf(dev(xs)))
    np.testing.assert_allclose(lp2, g["d/mvn/logpdf_scaled"], rtol=1e-13)
    rv = host(dists.MvNormal(loc=dev(locs), scale=sc, cov=cov).rvs(size=200, z=g["d/mvn/rvs_z"]))
    np.testing.assert_allclose(rv, g["d/mvn/rvs"], rtol=1e-14, atol=1e-15)   # dot-product order
    with pytest.raises(ValueError):
        dists.MvNormal(loc=np.zeros(2), cov=np.array([[1.0, 2.0], [2.0, 1.0]]))


@pytest.mark.parametrize("d", [9, 16, 32])
def test_mvnormal_large_d_vs_oracle(pb, d):
    """8 < d <= 32 (factor staged in shared memory, one particle per thread) against the oracle's restatement of
    distributions.py:888-982 with scipy's triangular solve: logpdf, rvs with injected normals, and the moments of
    device draws."""
    from particles_b200 import distributions as dists
    r = np.random.RandomState(d)
    B = r.randn(d, d)
    cov = B @ B.T / d + np.eye(d) * 0.3
    n = 3001
    loc, sc = r.randn(n, d), np.exp(r.randn(n, d) * 0.2)
    x = loc + r.randn(n, d)
    ref = orc.MvNormal(loc=loc, scale=sc, cov=cov)
    got = host(dists.MvNormal(loc=dev(loc), scale=dev(sc), cov=cov).logpdf(dev(x)))
    np.testing.assert_allclose(got, ref.logpdf(x), rtol=1e-11)
    ref0 = orc.MvNormal(loc=loc[0], scale=1.0, cov=cov)
    np.testing.assert_allclose(host(dists.MvNormal(loc=loc[0], cov=cov).logpdf(dev(x))), ref0.logpdf(x), rtol=1e-11)
    z = r.standard_normal((n, d))
    rv = host(dists.MvNormal(loc=dev(loc), scale=dev(sc), cov=cov).rvs(size=n, z=z))
    np.testing.assert_allclose(rv, ref.rvs(size=n, z=z), rtol=1e-12, atol=1e-13)
    pb.seed(5)
    dr = host(dists.MvNormal(loc=np.zeros(d), cov=cov).rvs(size=200_000))
    assert dr.shape == (200_000, d)
    assert np.abs(dr.mean(0)).max() < 0.02 and np.abs(np.cov(dr.T) - cov).max() < 0.03
    with pytest.raises(ValueError):
        dists.MvNormal(loc=np.zeros(33), cov=np.eye(33)).rvs(size=4)


def test_more_univariate_distributions_vs_scipy(pb):
    """Student / Gamma / Laplace / Logistic / Categorical / MixMissing (distributions.py:288-433, 598-628, 819-847):
    logpdf against scipy (what the reference calls), scalar and per-particle parameters; rvs moments."""
    from scipy import stats
    from particles_b200 import distributions as dists
    r = np.random.RandomState(0)
    n = 5000
    x, loc, sc = r.randn(n) * 2, r.randn(n), np.exp(r.randn(n) * 0.3)
    np.testing.assert_allclose(host(dists.Student(df=4.5, loc=dev(loc), scale=dev(sc)).logpdf(dev(x))),
                               stats.t.logpdf(x, 4.5, loc=loc, scale=sc), rtol=1e-12)
    np.testing.assert_allclose(host(dists.Student(df=3.0, loc=dev(loc)).logpdf(np.array([0.7]))),
                               stats.t.logpdf(0.7, 3.0, loc=loc), rtol=1e-12)
    xg = np.abs(x) + 0.1
    np.testing.assert_allclose(host(dists.Gamma(a=2.5, b=dev(sc)).logpdf(dev(xg))),
                               stats.gamma.logpdf(xg, 2.5, scale=1.0 / sc), rtol=1e-12)
    assert host(dists.Gamma(a=2.0, b=1.0).logpdf(dev(np.array([-1.0, 1.0]))))[0] == -np.inf
    np.testing.assert_allclose(host(dists.Laplace(loc=dev(loc), scale=0.7).logpdf(dev(x))),
                               stats.laplace.logpdf(x, loc=loc, scale=0.7), rtol=1e-12)
    np.testing.assert_allclose(host(dists.Logistic(loc=dev(loc), scale=dev(sc)).logpdf(dev(x))),
                               stats.logistic.logpdf(x, loc=loc, scale=sc), rtol=1e-11)
    p = r.dirichlet(np.ones(5), size=n)
    k = r.randint(0, 5, n)
    np.testing.assert_allclose(host(dists.Categorical(p=dev(p)).logpdf(dev(k, dtype=torch.int64))),
                               np.log(p[np.arange(n), k]), rtol=1e-13)
    np.testing.assert_allclose(host(dists.Categorical(p=p[0]).logpdf(dev(k, dtype=torch.int64))), np.log(p[0][k]), rtol=1e-13)
    draws = host(dists.Categorical(p=p[0]).rvs(size=200_000))
    np.testing.assert_allclose(np.bincount(draws, minlength=5) / 200_000, p[0], atol=5e-3)
    xm = x.copy()
    xm[::7] = np.nan
    lp = host(dists.MixMissing(pmiss=0.1, base_dist=dists.Normal(loc=dev(loc), scale=0.5)).logpdf(dev(xm)))
    want = stats.norm.logpdf(xm, loc=loc, scale=0.5) + np.log(0.9)
    want[::7] = np.log(0.1)
    np.testing.assert_allclose(lp, want, rtol=1e-12)
    t = host(dists.Student(df=5.0, loc=1.0, scale=2.0).rvs(size=400_000))
    assert abs(t.mean() - 1.0) < 0.02 and abs(t.var() - 4.0 * 5 / 3) < 0.15
    gm = host(dists.Gamma(a=3.0, b=2.0).rvs(size=400_000))
    assert abs(gm.mean() - 1.5) < 0.01 and abs(gm.var() - 0.75) < 0.02


def test_indepprod_dirac_vs_reference(pb, golden):
    from particles_b200 import state_space_models as ssm
    g = golden
    xp = dev(g["d/indep/xp"])
    law = ssm.BearingsOnly().PX(1, xp)
    xn = g["d/indep/rvs"]
    # recover the two columns of normals the reference drew, then replay them
    z = np.stack([(xn[:, 0] - g["d/indep/xp"][:, 0]) / 2e-4, (xn[:, 1] - g["d/indep/xp"][:, 1]) / 2e-4], 1)
    out = host(law.rvs(size=50, z=z))
    np.testing.assert_allclose(out, xn, rtol=1e-12, atol=1e-15)
    assert np.array_equal(out[:, 2:], xn[:, 2:])                     # Dirac components: exact
    np.testing.assert_allclose(host(law.logpdf(dev(xn))), g["d/indep/logpdf"], rtol=1e-13)
    lpy = host(ssm.BearingsOnly().PY(1, xp, dev(xn)).logpdf(np.array([0.7])))
    np.testing.assert_allclose(lpy, g["d/indep/bearing_logpdf"], rtol=1e-12)


@pytest.mark.gpu
def test_mvstochvol_plugin_path(pb):
    """MVStochVol (state_space_models.py:633-654) on the plugin path: MvNormal kernels with a per-particle scale.
    (1) its closures against the oracle's on the same particles; (2) logLt of bootstrap filters at N = 2000 within
    3 sigma of 30 runs of the live reference (tests/golden/golden_mvsv.npz)."""
    import os
    import particles_b200
    from particles_b200 import state_space_models as ssm
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_mvsv.npz"))
    kw = dict(mu=g["mu"], covX=g["covX"], corY=g["corY"], F=g["F"])
    m, mo = ssm.MVStochVol(**kw), orc.MVStochVol(**kw)
    r = np.random.RandomState(4)
    xp, x = r.randn(500, 3) * 0.5 - 0.4, r.randn(500, 3) * 0.5 - 0.4
    np.testing.assert_allclose(host(m.PX(3, dev(xp)).logpdf(dev(x))), mo.PX(3, xp).logpdf(x), rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(host(m.PY(3, dev(xp), dev(x)).logpdf(dev(g["y"][3]))), mo.PY(3, xp, x).logpdf(g["y"][3]),
                               rtol=1e-11, atol=1e-11)
    z = r.randn(500, 3)
    np.testing.assert_allclose(host(m.PX(3, dev(xp)).rvs(size=500, z=dev(z))), mo.PX(3, xp).rvs(500, z=z), rtol=1e-12, atol=1e-13)
    data = [row.reshape(1, -1) for row in g["y"]]
    lls = []
    for seed in range(6):
        pf = particles_b200.SMC(fk=ssm.Bootstrap(ssm=m, data=data), N=2000, seed=seed)
        pf.run()
        assert not pf.fused and pf.wgts.N == 2000
        lls.append(pf.logLt)
    ref = g["stat_logLt_N2000"]
    sd = ref.std(ddof=1)
    assert abs(np.mean(lls) - ref.mean()) < 3 * sd * np.sqrt(1 / 6 + 1 / len(ref)), (lls, ref.mean(), sd)
