"""High-precision reference of the sampler kernels of ``csrc/smcb_sampler.cu`` (TEST INFRASTRUCTURE).

Everything here is NumPy in fp64 and ``np.longdouble`` (x87 extended precision: unit roundoff 2^-64, 2048 times
smaller than fp64's, so the long-double values stand in for exact ones and every bound below counts fp64 roundings
only):

* the tempered logistic target (``lprior``, ``llik``, ``lpost`` over the data rows [0, n_rows)), the per-row
  softplus in long double with ``np.logaddexp(0, v)`` semantics and NaN -> -inf after the row sum, as the reference's
  ``StaticModel.loglik`` does;
* the two-pass weighted mean and covariance, a Cholesky backward-error check and the ESS of ``delta * lw``;
* replays of the sampler's Philox counter layouts (built on ``philox_ref._ctr``), Box-Muller in long double;
* the launch geometry the kernels choose (``tier``, ``tile_rows``, grids), so a test can assert the branch it reaches;
* ``check_generation``: one generation of the fused waste-free move replayed from the kernel's own previous row.

Each bound is written next to the operation it covers: ``gamma(k) = k u / (1 - k u)`` (u = 2^-53) is the usual bound
on the relative error of k chained fp64 roundings (Higham, Accuracy and Stability of Numerical Algorithms, 3.1).
The checks raise ``AssertionError`` naming the first chain / entry where the two sides disagree.
"""
import numpy as np

import philox_ref

LD = np.longdouble
U = np.finfo(np.float64).eps / 2                     # fp64 unit roundoff
EPS = np.finfo(np.float64).eps
LOG2PI_HALF = LD("0.918938533204672741780329736405617639861397473637783412817")
PI = LD("3.14159265358979323846264338327950288419716939937510582097")

# launch geometry of csrc/smcb_sampler.cu
SAMP_BLOCK = 128                                     # k_logistic_target (two particles per thread), k_rw_propose, k_mh_accept
WF_BLOCK, WF_LANES = 512, 16                         # k_logistic_wf_move: 16 lanes per chain, 32 chains per CTA
SMEM_BUDGET = 200 * 1024                             # launch_wf's shared-memory budget
TIERS = (4, 8, 12, 16, 20, 24, 32)
CTL_BLOCK, CTL_GRID = 256, 2 * 132                   # k_ctl_*: 256 threads, at most two CTAs per SM of an H100 SXM
ROOT_WAYS, ROOT_PASSES = 16, 11
WS_PARTIALS = 65536                                  # block partials of k_mh_accept in the context's workspace


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def tier(d):
    """The padded size D the kernels are instantiated for (the dispatch of smcb_logistic_target / wf_move)."""
    return next(D for D in TIERS if d <= D)


def tile_rows(D):
    """Data rows launch_wf stages per tile: (200 KiB - 8 D^2) / (8 D)."""
    return (SMEM_BUDGET - 8 * D * D) // (8 * D)


def wf_resident(d, n_rows):
    """True when the whole data set sits in shared memory (k_logistic_wf_move's ``tile_rows >= n_data``)."""
    return tile_rows(tier(d)) >= n_rows


def wf_grid(M):
    return -(-M // (WF_BLOCK // WF_LANES))


def target_grid(n):
    return -(-((n + 1) // 2) // SAMP_BLOCK)


def ctl_grid_root(n):
    return min(-(-n // CTL_BLOCK), CTL_GRID)


def ctl_grid_wcov(n):
    return min(-(-n // 8), CTL_GRID)


# ----------------------------------------------------------------------------------------- the logistic target
def lognorm(d, scale):
    return LD(d) * np.log(LD(scale)) + LD(d) * LOG2PI_HALF


def lprior_ld(theta, scale):
    th = np.asarray(theta, dtype=np.float64).astype(LD) / LD(scale)
    with np.errstate(invalid="ignore", over="ignore"):
        return -0.5 * np.sum(th * th, axis=1) - lognorm(theta.shape[1], scale)


def lprior_bound(theta, scale, D):
    """z = th / s (1 rounding), z^2 (1), a chain of D additions, -0.5 q (exact) minus the fp64 lognorm (its own
    d log s + d log(2 pi)/2: 4 roundings of terms <= |lognorm|) and 1 rounding of the result."""
    q = np.sum((np.asarray(theta, np.float64) / scale) ** 2, axis=1)
    ln = abs(float(lognorm(theta.shape[1], scale)))
    return gamma(D + 2) * 0.5 * q + gamma(4) * ln + U * (0.5 * q + ln)


def softplus_rows(theta, data):
    """g_r(theta) = -logaddexp(0, -theta . x_r) for every (particle, row), long double; also |theta_j x_rj| summed."""
    th = np.asarray(theta, np.float64).astype(LD)
    x = np.asarray(data, np.float64).astype(LD)
    with np.errstate(invalid="ignore", over="ignore"):
        lin = th @ x.T
        v = -lin
        g = -(np.maximum(v, 0) + np.log1p(np.exp(-np.abs(v))))
    with np.errstate(invalid="ignore", over="ignore"):
        absdot = np.abs(np.asarray(theta, np.float64)) @ np.abs(np.asarray(data, np.float64)).T
    return g, absdot


def llik_ld(theta, data):
    return llik_from_rows(softplus_rows(theta, data)[0])


def llik_from_rows(g):
    with np.errstate(invalid="ignore"):
        ll = g.sum(axis=1)
    ll[np.isnan(ll)] = -np.inf
    return ll


def llik_bound(g, absdot, dot_depth, sum_depth):
    """Error of the kernel's log-likelihood: per row, the dot product (``dot_depth`` chained fma / add roundings of
    terms bounded by sum_j |theta_j x_rj|, and the softplus' slope is at most 1), plus the softplus itself: exp of a
    non-positive argument and log of 1 + e (1.5 ulp each of values <= 1 and <= log 2), the rounding of 1 + e (one ulp of
    1) and of the final sum -- 4 ulp of 1 + |g_r| per row, generously; then the row sum in any order of depth
    ``sum_depth``: gamma(sum_depth) sum_r |g_r|.  ``g``, ``absdot``: what softplus_rows returns."""
    with np.errstate(invalid="ignore"):
        ag = np.abs(g).astype(np.float64)
        per_row = gamma(dot_depth) * absdot + 4 * EPS * (1.0 + ag)
        return per_row.sum(axis=1) + gamma(sum_depth) * ag.sum(axis=1)


def target_ld(theta, data, scale, epn):
    """(lprior, llik, lpost) in long double; lpost = lprior when epn == 0 (smc_samplers.py:840-843)."""
    lp = lprior_ld(theta, scale)
    ll = llik_ld(theta, data)
    with np.errstate(invalid="ignore"):
        post = lp + LD(epn) * ll if epn > 0 else lp.copy()
    return lp, ll, post


def target_bounds(theta, data, scale, epn, D, dot_depth, sum_depth):
    """(lprior, llik, lpost) in long double and their error bounds; lpost adds epn * llik's error and the rounding of
    epn * llik and of the sum."""
    bp = lprior_bound(theta, scale, D)
    g, absdot = softplus_rows(theta, data)
    bl = llik_bound(g, absdot, dot_depth, sum_depth)
    lp = lprior_ld(theta, scale)
    ll = llik_from_rows(g)
    with np.errstate(invalid="ignore"):
        post = lp + LD(epn) * ll if epn > 0 else lp.copy()
        bpost = bp + (epn * bl + U * (abs(epn) * np.abs(ll.astype(np.float64)) + np.abs(post.astype(np.float64)))
                      if epn > 0 else 0.0)
    return (lp, ll, post), (bp, bl, bpost)


def assert_close(what, got, want, bound, where="entry"):
    """|got - want| <= bound entry by entry; equal infinities and NaN on both sides count as equal."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want)
    with np.errstate(invalid="ignore"):
        diff = np.abs(got.astype(LD) - want.astype(LD)).astype(np.float64)
        same = (got == want.astype(np.float64)) | (np.isnan(got) & np.isnan(want.astype(np.float64)))
        bad = ~same & ~(diff <= bound)
    if bad.any():
        k = np.unravel_index(int(np.flatnonzero(bad)[0]), bad.shape)
        b = np.broadcast_to(bound, bad.shape)[k]
        raise AssertionError(f"{what}: {where} {k}: {got[k]!r} vs {float(want[k])!r} (|diff| {diff[k]:.3e} > "
                             f"bound {b:.3e}; {int(bad.sum())} of {bad.size} entries)")


# ----------------------------------------------------------------------------------------- Philox replays
def box_muller_ld(r):
    """Box-Muller of one Philox block in long double (the device's box_muller_fast is within 4 ulp of it: flog_pos
    and the sin/cos polynomials are <= 1.5 ulp, then sqrt, the halving of the log's error and the product: 3.25)."""
    u1 = philox_ref.u53_open(r[0], r[1]).astype(LD)
    u2 = philox_ref.u53(r[2], r[3]).astype(LD)
    rad = np.sqrt(-2 * np.log(u1))
    ang = 2 * PI * u2
    return rad * np.cos(ang), rad * np.sin(ang)


Z_REL = 4 * EPS                                      # the device normal's relative error against box_muller_ld


def rw_propose_normals(n, d, call, seed):
    """z (n, d) of k_rw_propose: pair i, word ((call >> 32) << 16) | ((j >> 1) << 8) | PURPOSE_API, t = (u32) call."""
    z = np.empty((n, d), dtype=LD)
    for j in range(0, d, 2):
        w3 = (((call >> 32) & 0xFFFF) << 16) | ((j >> 1) << 8) | philox_ref.PURPOSE_API
        r = philox_ref._ctr(np.arange(n), call & 0xFFFFFFFF, w3, seed)
        a, b = box_muller_ld(r)
        z[:, j] = a
        if j + 1 < d:
            z[:, j + 1] = b
    return z


def mh_accept_uniforms(n, call, seed):
    """u (n,) of k_mh_accept: pair i, word ((call >> 32) << 8) | PURPOSE_API, the first uniform of the block."""
    w3 = (((call >> 32) & 0xFFFFFF) << 8) | philox_ref.PURPOSE_API
    r = philox_ref._ctr(np.arange(n), call & 0xFFFFFFFF, w3, seed)
    return philox_ref.u53(r[0], r[1])


def wf_normals(M, d, s, call, seed):
    """z (M, d) of generation s of k_logistic_wf_move: pair = chain c, word (s << 16) | ((j >> 1) << 8) | NORMAL."""
    z = np.empty((M, d), dtype=LD)
    for j in range(0, d, 2):
        r = philox_ref._ctr(np.arange(M), call & 0xFFFFFFFF, (s << 16) | ((j >> 1) << 8) | philox_ref.PURPOSE_NORMAL,
                            seed)
        a, b = box_muller_ld(r)
        z[:, j] = a
        if j + 1 < d:
            z[:, j + 1] = b
    return z


def wf_uniforms(M, s, call, seed):
    """u (M,) of generation s: pair = chain c, word (s << 16) | PURPOSE_UNIFORM, the first uniform."""
    r = philox_ref._ctr(np.arange(M), call & 0xFFFFFFFF, (s << 16) | philox_ref.PURPOSE_UNIFORM, seed)
    return philox_ref.u53(r[0], r[1])


# ----------------------------------------------------------------------------------------- random-walk proposal
def propose_ld(theta, z, L):
    """theta + z @ L.T in long double, and the bound on the kernel's fp64 value: coordinate a is theta_a plus a chain of
    a + 1 products added in order (a + 2 roundings of terms bounded by |theta_a| + sum_b |z_b L_ab|), plus the
    device normals' own error when they are drawn on the device (``z_rel``)."""
    th = np.asarray(theta, np.float64)
    Lf = np.asarray(L, np.float64)
    zl = np.asarray(z).astype(LD)
    with np.errstate(invalid="ignore", over="ignore"):
        prop = th.astype(LD) + zl @ Lf.astype(LD).T
        zabs = np.abs(zl.astype(np.float64))
        terms = zabs @ np.abs(Lf).T
        d = th.shape[1]
        bound = gamma(np.arange(d) + 2)[None, :] * (np.abs(th) + terms)
    return prop, bound


def propose_bound_z(z, L, z_rel):
    with np.errstate(invalid="ignore", over="ignore"):
        return z_rel * (np.abs(np.asarray(z).astype(np.float64)) @ np.abs(np.asarray(L, np.float64)).T)


# ----------------------------------------------------------------------------------------- Metropolis decision
def pb_ld(lp_acc):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.exp(np.minimum(lp_acc, 0))


def decisions(u, lp_acc, tol):
    """(accept, decided): accept = log u < lp_acc (u < exp(min(lp_acc, 0))); ``decided`` marks the draws whose margin
    |log u - min(lp_acc, 0)| exceeds ``tol`` -- the others may fall either way within the kernel's rounding."""
    u = np.asarray(u, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        lu = np.log(u.astype(LD))
        la = np.minimum(lp_acc, 0)
        acc = lu < la
        margin = np.abs(lu - la).astype(np.float64)
        decided = np.isnan(la) | np.isneginf(la) | (margin > tol)
    return acc, decided


# ----------------------------------------------------------------------------------------- weighted mean / covariance
def wsums_ld(W, theta, mean=None):
    """Pass 0: (sum w x_j, sum w); pass 1 (``mean`` given): the lower triangle (row-major) of
    sum w (x - mean)(x - mean)^T -- all in long double."""
    w = np.asarray(W, np.float64).astype(LD)
    x = np.asarray(theta, np.float64).astype(LD)
    if mean is None:
        return (w[:, None] * x).sum(axis=0), w.sum()
    dev = x - np.asarray(mean, np.float64).astype(LD)[None, :]
    C = (w[:, None] * dev).T @ dev
    a, b = np.tril_indices(x.shape[1])
    return C[a, b]


def wcov_depth(n, slices=1):
    """Depth of the wcov kernels' sums: one warp's rows in order, then the 8 warps of a CTA, then the CTAs in order
    (and the caller's sum over ``slices``)."""
    g = ctl_grid_wcov(n)
    return -(-n // (8 * g)) + 8 + g + slices


def wsums_bounds(W, theta, mean=None, depth=None, extra=0):
    """Bounds of the device sums: pass 0 one product per term, pass 1 two subtractions and two products per term, then
    the sum of depth ``depth`` (``extra``: further roundings per term, e.g. a per-shard normalisation and share)."""
    w = np.abs(np.asarray(W, np.float64))
    x = np.asarray(theta, np.float64)
    n = x.shape[0]
    depth = wcov_depth(n) if depth is None else depth
    if mean is None:
        return gamma(depth + 1 + extra) * (w[:, None] * np.abs(x)).sum(axis=0), gamma(depth + extra) * w.sum()
    dev = np.abs(x - np.asarray(mean, np.float64)[None, :])
    C = (w[:, None] * dev).T @ dev
    a, b = np.tril_indices(x.shape[1])
    return gamma(depth + 4 + extra) * C[a, b]


def check_wcov(W, theta, s0, tri, depth=None, extra=0):
    """The device's pass-0 sums ``s0`` (d + 1) and pass-1 triangle ``tri`` (taken about the device's own mean
    s0[:d] / s0[d]) against long double, and the mean and covariance derived from them."""
    d = np.asarray(theta).shape[1]
    s0 = np.asarray(s0, np.float64)
    sx, sw = wsums_ld(W, theta)
    bx, bw = wsums_bounds(W, theta, None, depth, extra)
    assert_close("sum w x", s0[:d], sx, bx)
    assert_close("sum w", s0[d:], np.array([sw]), np.array([bw]))
    mean = s0[:d] / s0[d]
    tri_ld = wsums_ld(W, theta, mean)
    btri = wsums_bounds(W, theta, mean, depth, extra)
    assert_close("sum w (x - m)(x - m)^T", tri, tri_ld, btri)
    # the mean: sums' error over sum w, and sum w's own relative error, one rounding of the quotient
    m_ld = sx / sw
    assert_close("mean", mean, m_ld, (bx + np.abs(m_ld.astype(np.float64)) * bw) / float(sw) +
                 U * np.abs(m_ld.astype(np.float64)))
    return mean, unpack_tri(np.asarray(tri, np.float64), d) / s0[d]


def check_mean_cov(W, theta, mean, cov, depth=None, extra=0):
    """A weighted mean and covariance (any two-pass evaluation in fp64 whose sums have depth ``depth``) against long
    double: the mean as in check_wcov, the covariance about the given mean -- the sums' bound over sum w, plus sum w's
    relative error and two roundings of the quotient (a division, or a multiplication by 1 / sum w)."""
    d = np.asarray(theta).shape[1]
    sx, sw = wsums_ld(W, theta)
    bx, bw = wsums_bounds(W, theta, None, depth, extra)
    m_ld = sx / sw
    am = np.abs(m_ld.astype(np.float64))
    assert_close("mean", mean, m_ld, (bx + am * bw) / float(sw) + U * am)
    tri_ld = wsums_ld(W, theta, mean)
    btri = wsums_bounds(W, theta, mean, depth, extra)
    cov_ld = unpack_tri(tri_ld, d) / sw
    bound = unpack_tri(btri, d) / float(sw) + np.abs(cov_ld.astype(np.float64)) * (bw / float(sw) + 2 * U)
    assert_close("covariance", cov, cov_ld, bound)


def unpack_tri(tri, d):
    C = np.zeros((d, d), dtype=np.asarray(tri).dtype)
    a, b = np.tril_indices(d)
    C[a, b] = tri
    C[b, a] = tri
    return C


def chol_backward_check(A, L):
    """|L L^T - A| <= gamma(d + 1) |L| |L|^T elementwise (Higham, Theorem 10.3) for the fp64 matrix A the kernel
    factored and its factor L (unscaled), evaluated in long double; L must be lower-triangular."""
    A = np.asarray(A, np.float64)
    L = np.asarray(L, np.float64)
    d = A.shape[0]
    assert np.all(np.triu(L, 1) == 0.0), "factor not lower-triangular"
    Ll = L.astype(LD)
    resid = np.abs(Ll @ Ll.T - A.astype(LD)).astype(np.float64)
    bound = gamma(d + 1) * (np.abs(L) @ np.abs(L).T)
    bad = ~(resid <= bound)
    if bad.any():
        k = np.unravel_index(int(np.flatnonzero(bad)[0]), bad.shape)
        raise AssertionError(f"Cholesky backward error at {k}: {resid[k]:.3e} > {bound[k]:.3e}")


# ----------------------------------------------------------------------------------------- ESS and the root-find
def ess_ld(delta, lw):
    """ESS(delta * lw) = (sum w)^2 / sum w^2 with w = exp(delta (lw - max lw)), long double; N at delta <= 0."""
    lw = np.asarray(lw, np.float64)
    if delta <= 0:
        return LD(lw.shape[0])
    a = lw.astype(LD) - LD(lw.max())
    with np.errstate(invalid="ignore"):
        e = np.exp(LD(delta) * a)
    e[np.isnan(e)] = 0                                 # -inf entries carry no weight
    return e.sum() ** 2 / (e * e).sum()


def ess_slope_ld(delta, lw):
    """d ESS / d delta at delta, long double."""
    lw = np.asarray(lw, np.float64)
    a = lw.astype(LD) - LD(lw.max())
    fin = np.isfinite(a)
    a = a[fin]
    e = np.exp(LD(delta) * a)
    S, Q = e.sum(), (e * e).sum()
    dS, dQ = (a * e).sum(), 2 * (a * e * e).sum()
    return (2 * S * dS * Q - S * S * dQ) / (Q * Q)


def ess_err(delta, lw):
    """Bound on the device's relative ESS error at delta: every term exp(delta (lw_i - M)) carries the roundings of
    lw_i - M and of the product (relative u |delta a_i| each) and fexp_neg's 1.5 ulp; the sums have the depth of the
    root pass (a thread's entries in order, 5 shuffle levels, 8 warps, the CTAs in order); ESS = s^2 / q doubles s's
    error and adds q's and 2 roundings."""
    lw = np.asarray(lw, np.float64)
    n = lw.shape[0]
    g = ctl_grid_root(n)
    depth = -(-n // (g * CTL_BLOCK)) + 5 + 8 + g
    a = lw - lw.max()
    fin = np.isfinite(a)
    a = a[fin]
    e = np.exp(delta * a)
    eps_i = U * (2 * np.abs(delta * a) + 3)
    s, q = e.sum(), (e * e).sum()
    ds = (e * eps_i).sum() + gamma(depth) * s
    dq = 2 * (e * e * eps_i).sum() + gamma(depth + 1) * q
    return 2 * ds / s + dq / q + 2 * U


def root_ld(lw, epn, alpha, tol=LD(2) ** -60):
    """The exponent at which ESS((e - epn) lw) = alpha N, by bisection in long double (1.0 when the full step keeps
    ESS >= alpha N, as next_annealing_epn returns)."""
    n = np.asarray(lw).shape[0]
    target = LD(alpha) * n
    hi = LD(1) - LD(epn)
    if ess_ld(float(hi), lw) >= target:
        return 1.0
    lo = LD(0)
    while hi - lo > tol * max(hi, LD(1e-30)):
        mid = (lo + hi) / 2
        if mid == lo or mid == hi:
            break
        if ess_ld(float(mid), lw) >= target:      # float(mid): ess_ld multiplies in long double again
            lo = mid
        else:
            hi = mid
    return float(LD(epn) + (lo + hi) / 2)


def final_bracket(epn):
    """Width of the device root-find's last bracket: (1 - epn) 16^-11; its result is that bracket's midpoint."""
    return (1.0 - epn) * float(ROOT_WAYS) ** -ROOT_PASSES


def check_root(lw, epn, alpha, got):
    """Accept the device's exponent ``got`` when ESS_ld(delta - w) >= alpha N >= ESS_ld(delta + w), delta = got - epn:
    the exact root lies within half a final bracket of the midpoint the device returns, and a grid point whose ESS is
    within the device's rounding of alpha N may fall into the neighbouring bracket -- that moves the root by at most the
    ESS error over the ESS slope.  A result of 1.0 needs ESS(1 - epn) >= alpha N up to the same rounding."""
    lw = np.asarray(lw, np.float64)
    n = lw.shape[0]
    target = alpha * n
    hi = 1.0 - epn
    e_hi = ess_ld(hi, lw)
    if got == 1.0:
        rel = ess_err(hi, lw) if np.isfinite(lw).any() and hi > 0 else 0.0
        assert float(e_hi) * (1 + rel) >= target, f"returned 1.0 but ESS(1 - epn) = {float(e_hi)!r} < {target!r}"
        return
    assert epn <= got < 1.0, f"exponent {got!r} outside [{epn!r}, 1)"
    delta = got - epn
    rel = ess_err(delta, lw)
    slope = abs(float(ess_slope_ld(delta, lw)))
    shift = rel * float(ess_ld(delta, lw)) / slope if slope > 0 else np.inf
    # the device returns epn + delta rounded to fp64: half an ulp of the exponent (1e-16 near 1, far more than the
    # last bracket when epn is close to 1), taken twice
    w = 0.5 * final_bracket(epn) + shift + 2 * U * got
    lo_e = ess_ld(max(delta - w, 0.0), lw)
    hi_e = ess_ld(min(delta + w, hi), lw)
    assert lo_e >= target >= hi_e, (f"exponent {got!r}: ESS(delta - w) = {float(lo_e)!r}, ESS(delta + w) = "
                                    f"{float(hi_e)!r}, alpha N = {target!r}, w = {w:.3e}")


# ----------------------------------------------------------------------------------------- one waste-free generation
def check_generation(s, prev, out, pb, z, u, L, data, scale, epn, d, z_rel=0.0):
    """Generation s of k_logistic_wf_move from the kernel's own row s - 1.

    ``prev`` / ``out``: dicts of theta (M, d), lprior, llik, lpost (rows s - 1 and s of the kernel's output); ``pb``:
    the kernel's pb_out row s - 1; ``z`` (M, d) and ``u`` (M,): the draws of generation s (long-double normals when
    replayed from the device's Philox stream, with ``z_rel`` their relative error on the device); ``L``: the factor;
    ``data``: the rows the target uses.  Checks that a rejected chain's row is a bit-for-bit copy of row s - 1, that an
    accepted chain's row is the long-double proposal and its target values, that every decision whose margin exceeds
    the tolerance agrees with the long-double one, and pb.  Returns (accepted, decided) masks."""
    D = tier(d)
    M = prev["theta"].shape[0]
    prop, bprop = propose_ld(prev["theta"], z, L)
    bprop = bprop + propose_bound_z(z, L, z_rel)
    propf = prop.astype(np.float64)
    # target of the long-double proposal, bounds for the kernel's own: dot products in two fma chains of D / 2 and
    # one add; rows split over 16 lanes, summed in tiles and a 4-level butterfly: any order of depth n_rows + 4
    (lp, ll, post), (bp, bl, bpost) = target_bounds(propf, data, scale, epn, D, D // 2 + 1, data.shape[0] + 4)
    # the kernel evaluates its own rounded proposal: add the target's slope times the proposal error
    # (prior: |theta| / s^2 per coordinate; likelihood: sum_r |x_rj| per coordinate -- the softplus' slope is <= 1)
    absx = np.abs(np.asarray(data, np.float64)).sum(axis=0)
    with np.errstate(invalid="ignore", over="ignore"):
        gp = ((np.abs(propf) + bprop) / scale ** 2 * bprop).sum(axis=1)
        gl = (absx[None, :] * bprop).sum(axis=1)
        bp, bl = bp + gp, bl + gl
        bpost = bpost + gp + (epn * gl if epn > 0 else 0.0)
        lp_acc = post - np.asarray(prev["lpost"], np.float64).astype(LD)
        # the kernel's lp_acc: its lpost's error, one rounding of the difference; pb = exp: 1 more ulp
        tol = bpost + U * np.abs(lp_acc.astype(np.float64)) + 2 * EPS
    tol = np.where(np.isfinite(tol), tol, np.inf)
    acc, decided = decisions(u, lp_acc, tol)

    same = np.all(out["theta"] == prev["theta"], axis=1) | np.all(
        np.isnan(out["theta"]) & np.isnan(prev["theta"]), axis=1)
    dev_acc = ~same
    for k in ("lprior", "llik", "lpost"):               # a rejected chain's row s: row s - 1, bit for bit
        a, b = np.asarray(out[k], np.float64), np.asarray(prev[k], np.float64)
        eq = (a.view(np.int64) == b.view(np.int64))
        bad = same & ~eq
        if bad.any():
            c = int(np.flatnonzero(bad)[0])
            raise AssertionError(f"generation {s}: rejected chain {c} (CTA {c // (WF_BLOCK // WF_LANES)}): {k} not "
                                 f"bit-identical to row s - 1: {a[c]!r} vs {b[c]!r}")
    flip = decided & (acc != dev_acc)
    if flip.any():
        c = int(np.flatnonzero(flip)[0])
        raise AssertionError(f"generation {s}: chain {c} (CTA {c // (WF_BLOCK // WF_LANES)}) "
                             f"{'accepted' if dev_acc[c] else 'rejected'} but u = {float(u[c])!r}, "
                             f"lp_acc = {float(lp_acc[c])!r} +- {tol[c]:.3e} ({int(flip.sum())} of {M} decisions)")
    A = dev_acc
    if A.any():
        assert_close(f"generation {s}: accepted theta", out["theta"][A], prop[A], bprop[A], "chain")
        assert_close(f"generation {s}: accepted lprior", out["lprior"][A], lp[A], bp[A], "chain")
        assert_close(f"generation {s}: accepted llik", out["llik"][A], ll[A], bl[A], "chain")
        assert_close(f"generation {s}: accepted lpost", out["lpost"][A], post[A], bpost[A], "chain")
    # pb = exp(min(lp_acc, 0)): relative error exp(tol) - 1 of the long-double value, NaN where lp_acc is NaN
    want = pb_ld(lp_acc)
    with np.errstate(invalid="ignore", over="ignore"):
        bpb = np.abs(want.astype(np.float64)) * np.expm1(np.minimum(tol, 700.0)) + EPS
    assert_close(f"generation {s}: pb", pb, want, bpb, "chain")
    return dev_acc, decided
