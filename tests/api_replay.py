"""Long-double replay of the stand-alone kernels of ``csrc/smcb_api.cu`` (TEST INFRASTRUCTURE).

The weights algebra (``k_lse``, ``k_max_sum``, ``k_exp_normalise``), ``wmean_and_var`` (``k_wmoments``), the CDF scans
and inverse-CDF searches behind every resampling scheme, and the log-densities and draws of ``distributions.py``, each
restated in NumPy fp64 and ``np.longdouble``.  Every bound is ``SAFETY`` times an operation count written beside it,
in units of the fp64 unit round-off, applied to the magnitudes the operation touches, so a subtly wrong kernel (an
element read twice or skipped, one slot or one counter word off, a CDF entry off by one ulp where a grid point sits on
it) fails, while the fp64 rounding of a correct kernel passes at every size.

Ancestors are judged twice: bit for bit against ``searchsorted`` on the kernel's own CDF and grid points (where the
scratch that holds them is readable), and against the long-double CDF, exactly wherever the derived bounds decide the
draw and otherwise within the bracket of the knots the bounds cannot separate.
"""
import numpy as np

import philox_ref
from step_replay import EPS, LD, fix_nan, lse_stats

SAFETY = 4.0
BLOCK = 256
N_SM = 132
MAX_GRID = N_SM * 8                 # grid_for's cap (smcb_common.cuh)
SEARCH_TILE = BLOCK * 4             # outputs per k_search tile
SEARCH_STAGE = 4096                 # CDF entries a tile stages in shared memory
SCAN_TILE = BLOCK * 8               # values per scan tile
WMOM_GRID = 592                     # k_wmoments' CTA cap
WMOM_MAX_D = 32
PI_LD = LD("3.14159265358979323846264338327950288")
HALFLOG2PI_LD = LD(0.5) * np.log(LD(2) * PI_LD)
HALFLOG2PI = 0.91893853320467274178                     # the constant the kernels use (kHalfLog2Pi)


def grid_for(n, per):
    return int(max(1, min(-(-int(n) // per), MAX_GRID)))


def _ld(a):
    return np.asarray(a, dtype=np.float64).astype(LD)


def within(what, got, want, bound, where=None):
    """``got`` (fp64) within ``bound`` of ``want`` (long double) elementwise; equal infinities and NaN on both sides
    pass.  Raises with the first offending index."""
    got, want, bound = np.atleast_1d(got), np.atleast_1d(want), np.broadcast_to(np.atleast_1d(bound), np.shape(want))
    g = got.astype(LD)
    same = (g == want) | (np.isnan(got) & np.isnan(want.astype(np.float64)))
    with np.errstate(invalid="ignore"):
        ok = same | (np.abs(g - want) <= bound)
    if not ok.all():
        k = int(np.flatnonzero(~ok)[0])
        tag = "" if where is None else f" ({where})"
        raise AssertionError(f"{what}: differs first at {k}{tag}: {got[k]!r} vs {float(want[k])!r} "
                             f"(bound {float(bound[k]):.3e}; {int((~ok).sum())} of {ok.size})")


# ------------------------------------------------------------------------------------------------- weights
def weights_ref(lw):
    """Weights.__init__ (resampling.py:217-226) on the NaN -> -inf rewritten lw: max (exact), log_mean, ESS, sum, W,
    each in long double, with the bound of the kernels' fp64 values.

    The kernels' sum: every term exp(v - m) is one fp64 subtraction (|v - m| eps / 2) and one exponential (2 ulp);
    it then passes through at most (per-thread batches + 5 warp + 3 block + 8 grid merges) rescalings, each one more
    exponential of a difference that telescopes to |v - m|, and through as many additions, one rounding each.  So
    |ds| <= eps sum_i e_i (3 |v_i - m| + 2 + 3 (k + 16)), with k the values one thread adds."""
    v = fix_nan(lw)
    n = v.size
    grid = grid_for(n, BLOCK * 4)
    k = -(-n // (grid * BLOCK))
    m = v.max()
    out = {"m": m, "n": n}
    if not np.isfinite(m):
        out.update(log_mean=LD(np.nan), ess=LD(np.nan), s=LD(np.nan), W=np.full(n, LD(np.nan)),
                   b_log_mean=LD(0), b_ess=LD(0), b_s=LD(0), b_W=np.zeros(n, dtype=LD))
        return out
    _, s, q, e = lse_stats(v)
    with np.errstate(invalid="ignore"):
        d = np.where(np.isfinite(v), np.abs(v - m), 0.0).astype(LD)
    c = LD(2 + 3 * (k + 16))
    rs = SAFETY * LD(EPS) * (e * (3 * d + c)).sum() / s               # relative bound on s
    rq = SAFETY * LD(EPS) * (e * e * (6 * d + 2 * c)).sum() / q       # q = sum e^2: twice the relative error per term
    lm = LD(m) + np.log(s / LD(n))
    out.update(s=s, q=q, log_mean=lm, ess=s * s / q, W=e / s,
               b_s=rs * s, b_log_mean=rs + SAFETY * LD(EPS) * (abs(lm) + 2),
               b_ess=(2 * rs + rq + SAFETY * 2 * LD(EPS)) * (s * s / q))
    # W = fexp(lw - m) / s: one subtraction, one 2-ulp exponential, one correctly rounded quotient, and s itself; the
    # exponential flushes to 0 below exp(-708) (smcb_math.cuh), so W may be 0 where the exact value is below that / s
    out["b_W"] = (e / s) * (rs + SAFETY * LD(EPS) * (d / 2 + 3)) + LD(3.4e-308) / s + LD(2.0 ** -1070)
    return out


def check_weights(lw_in, lw_after, stats, W=None):
    """``smcb_normalise``'s stats {m, log_mean, ESS, s} and W, and the in-place NaN -> -inf rewrite of lw."""
    lw_in = np.asarray(lw_in, dtype=np.float64)
    fixed = fix_nan(lw_in)
    assert np.array_equal(np.asarray(lw_after), fixed), "the NaN -> -inf rewrite of lw"
    r = weights_ref(lw_in)
    if np.isfinite(r["m"]):
        assert stats[0] == r["m"], f"max {stats[0]!r} vs {r['m']!r}"
    else:
        assert stats[0] == r["m"] or np.isnan(stats[0]), stats[0]
    within("log_mean", stats[1], np.atleast_1d(r["log_mean"]), r["b_log_mean"])
    within("ESS", stats[2], np.atleast_1d(r["ess"]), r["b_ess"])
    within("sum", stats[3], np.atleast_1d(r["s"]), r["b_s"])
    if W is not None:
        within("W", W, r["W"], r["b_W"])
    return r


def lse_ref(v, mode, W=None):
    """log_sum_exp / log_mean_exp / essl (resampling.py:166-188, 247-317) as the reference evaluates them, in long
    double, and the bound of the kernel's value.  The reference's rules at the edges: any NaN, any +inf or every entry
    -inf makes ``m + log(sum(exp(v - m)))`` NaN (inf - inf); a weighted mean of the same is NaN as well."""
    v = np.asarray(v, dtype=np.float64)
    n = v.size
    m = v.max()
    if not np.isfinite(m):
        return LD(np.nan), LD(0)
    grid = grid_for(n, BLOCK * 4)
    k = -(-n // (grid * BLOCK))
    e = np.exp(_ld(v) - LD(m))
    with np.errstate(invalid="ignore"):
        d = np.where(np.isfinite(v), np.abs(v - m), 0.0).astype(LD)
    c = LD(2 + 3 * (k + 16))
    if mode == "sum" or mode == "mean":
        s = e.sum()
        r = SAFETY * LD(EPS) * (e * (3 * d + c)).sum() / s
        val = LD(m) + np.log(s if mode == "sum" else s / LD(n))
        return val, r + SAFETY * LD(EPS) * (abs(val) + 2)
    if mode == "essl":
        s, q = e.sum(), (e * e).sum()
        r = SAFETY * LD(EPS) * (e * (3 * d + c)).sum() / s
        rq = SAFETY * LD(EPS) * (e * e * (6 * d + 2 * c)).sum() / q
        return s * s / q, (2 * r + rq + SAFETY * 2 * LD(EPS)) * s * s / q
    # weighted: m + log(sum W e / sum W); the sums of w e and of W: one product more per term, n terms in order
    w = _ld(W)
    sw, s = w.sum(), (w * e).sum()
    r = SAFETY * LD(EPS) * ((w * e * (3 * d + c + 1)).sum() / s + c)
    val = LD(m) + np.log(s / sw)
    return val, r + SAFETY * LD(EPS) * (abs(val) + 2)


def exp_normalise_ref(lw):
    """exp_and_normalise (resampling.py:138-163, no NaN rewrite): NaN everywhere when the max is not finite or any
    entry is NaN, as NumPy gives; else weights_ref's W."""
    lw = np.asarray(lw, dtype=np.float64)
    if np.isnan(lw).any() or not np.isfinite(lw.max()):
        return np.full(lw.size, LD(np.nan)), np.zeros(lw.size, dtype=LD)
    r = weights_ref(lw)
    return r["W"], r["b_W"]


# ------------------------------------------------------------------------------------------------- moments
def wmoments_geometry(n):
    """(CTAs, values one thread adds in sequence) of k_wmoments."""
    grid = min(grid_for(n, BLOCK * 4), WMOM_GRID)
    return grid, -(-n // (grid * BLOCK))


def wmoments_ref(W, x):
    """wmean_and_var (resampling.py:320-338): mean = sum W x / sum W, var = m2 - mean^2 with m2 = sum W x^2 / sum W,
    the reference's own formula (so offset data cancels in var exactly as it does there).  x is (n,) or (n, d).

    The kernel's three sums run through D = k (one thread, in sequence) + 5 (warp) + 8 (block) + grid (in sequence)
    additions, one rounding each, and one or two roundings per product: |dS0| <= D eps S0, |dS1| <= (D + 1) eps
    sum W|x|, |dS2| <= (D + 2) eps sum W x^2.  mean and m2 add one division each, var one product and one
    subtraction; the bound carries |dmean| through mean^2."""
    W = np.asarray(W, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    x2 = x.reshape(W.size, -1)
    grid, k = wmoments_geometry(W.size)
    D = LD(k + 5 + 8 + grid)
    w, xl = _ld(W)[:, None], x2.astype(LD)
    S0, S1, S2 = w.sum(), (w * xl).sum(0), (w * xl * xl).sum(0)
    A1 = (np.abs(w) * np.abs(xl)).sum(0)
    mean, m2 = S1 / S0, S2 / S0
    var = m2 - mean * mean
    e = SAFETY * LD(EPS)
    d0 = e * D * np.abs(w).sum() / abs(S0)
    dmean = e * (D + 1) * A1 / abs(S0) + np.abs(mean) * (d0 + e)
    dm2 = e * (D + 2) * S2 / abs(S0) + np.abs(m2) * (d0 + e)
    dvar = dm2 + 2 * np.abs(mean) * dmean + dmean * dmean + e * (mean * mean + np.abs(var))
    return mean, var, dmean, dvar


def check_wmoments(W, x, out):
    """``out`` = the kernel's {mean[d], var[d]} against wmoments_ref."""
    mean, var, dmean, dvar = wmoments_ref(W, x)
    d = mean.size
    out = np.asarray(out, dtype=np.float64)
    assert out.size == 2 * d, (out.size, d)
    within("wmean", out[:d], mean, dmean)
    within("wvar", out[d:], var, dvar)


# -------------------------------------------------------------------------------------------- CDF / search
def scan_depth(n):
    """Roundings on the path of one prefix of run_scan: 8 in the thread, 5 in the warp, 3 across the block, one
    per earlier tile of the chunk (at most ceil(tiles / 132): at least one chunk per SM), 10 + 3 in the CTA-wide scan
    of the chunk sums, and 2 to add the bases."""
    tiles = -(-int(n) // SCAN_TILE)
    return 8 + 5 + 3 + -(-tiles // N_SM) + 13 + 2


def cdf_ref(w):
    """Long-double inclusive prefix sum of the fp64 values ``w`` (>= 0) and the bound of run_scan's value."""
    w = np.asarray(w, dtype=np.float64)
    C = np.cumsum(_ld(w))
    return C, SAFETY * LD(EPS) * scan_depth(w.size) * C


def check_cdf(what, cdf, w, ref=None):
    C, b = cdf_ref(w) if ref is None else ref
    cdf = np.asarray(cdf, dtype=np.float64)
    assert np.all(np.diff(cdf) >= 0), f"{what}: decreases at {int(np.flatnonzero(np.diff(cdf) < 0)[0])}"
    within(what, cdf, C, b)
    return C, b


def spacings_ref(u):
    """z = cumsum(-log u) (resampling.py:536) in long double, and the bound of the kernel's: each -log u is one
    1-ulp logarithm, then the scan's roundings on the running sum."""
    u = np.asarray(u, dtype=np.float64)
    t = -np.log(_ld(u))
    z = np.cumsum(t)
    return z, SAFETY * LD(EPS) * (np.cumsum(t) * scan_depth(u.size) + np.cumsum(t))


def grid_bound(z, bz, M):
    """su_k = z[k] / z[M] and its bound from those of z: relative errors add, plus one division."""
    su = z[:M] / z[M]
    return su, bz[:M] / z[M] + su * (bz[M] / z[M]) + su * LD(EPS) * SAFETY


def bracket(C, bC, su, bsu):
    """[lo, hi] of the ancestors the bounds allow for each grid point: lo = the first knot that can lie at or above
    su, hi = the first knot that surely does (searchsorted 'left' on the bounded knots), clipped to N - 1."""
    n = C.size
    su = np.asarray(su, dtype=LD)
    lo = np.searchsorted(C + bC, su - bsu, side="left")
    hi = np.searchsorted(C - bC, su + bsu, side="left")
    return np.minimum(lo, n - 1), np.minimum(hi, n - 1)


def check_ancestors(what, A, C, bC, su, bsu, W):
    """Every ancestor within its bracket (exact where lo == hi); a positive grid point never draws a zero-weight
    entry.  Returns the number of draws the bounds decide exactly."""
    A = np.asarray(A)
    su = np.asarray(su, dtype=LD)
    lo, hi = bracket(C, bC, su, bsu)
    bad = (A < lo) | (A > hi)
    if bad.any():
        k = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: ancestor {A[k]} outside [{lo[k]}, {hi[k]}] first at output {k} "
                             f"(su {float(su[k])!r}; {int(bad.sum())} of {A.size})")
    drawn = (su > 0) & (np.searchsorted(C, su, side="left") < C.size)
    zero = drawn & ~(np.asarray(W)[A] > 0)
    assert not zero.any(), f"{what}: output {int(np.flatnonzero(zero)[0])} draws a zero-weight entry"
    return int((lo == hi).sum())


def check_search_exact(what, A, cdf, su):
    """Bit for bit: A = minimum(searchsorted(cdf, su, 'left'), N - 1) on the kernel's own CDF and grid points."""
    ref = np.minimum(np.searchsorted(np.asarray(cdf), np.asarray(su), side="left"), len(cdf) - 1)
    A = np.asarray(A)
    if not np.array_equal(A, ref):
        k = int(np.flatnonzero(A != ref)[0])
        raise AssertionError(f"{what}: ancestor {A[k]} vs searchsorted {ref[k]} first at output {k} "
                             f"({int((A != ref).sum())} of {A.size} differ)")


def search_branches(cdf, su):
    """Per k_search tile, True where it staged its CDF slice in shared memory and False where it bisected in global
    memory: the slice [bnd[t], bnd[t + 1]] (+1) of k_search_bounds, against kSearchStage entries."""
    cdf, su = np.asarray(cdf), np.asarray(su)
    n, m = cdf.size, su.size
    nt = -(-m // SEARCH_TILE)
    keys = np.concatenate([su[np.arange(nt) * SEARCH_TILE], su[m - 1:m]])
    bnd = np.searchsorted(cdf, keys, side="left")
    hi1 = np.minimum(bnd[1:] + 1, n)
    return (hi1 - bnd[:-1]) <= SEARCH_STAGE


def su_of(scheme, u, M):
    """The reference's grid points (resampling.py:602, 609) as IEEE expressions."""
    u = np.asarray(u, dtype=np.float64).reshape(-1)
    if scheme == "systematic":
        return (u[0] + np.arange(M)) / M
    return (u[:M] + np.arange(M)) / M


def check_inverse_cdf(scheme, W, M, u, A, cdf=None, z=None, ref=None):
    """systematic / stratified / multinomial: the kernel's CDF (when given) against the long-double one, the
    ancestors bit for bit on it, and against the long-double CDF within the bounds.  ``u``: the uniforms the scheme
    consumed; ``z``: multinomial's spacings from the scratch; ``ref``: cdf_ref(W), when the caller holds it."""
    W = np.asarray(W, dtype=np.float64)
    C, bC = cdf_ref(W) if ref is None else ref
    if cdf is not None:
        check_cdf(f"{scheme} CDF", cdf, W, ref=(C, bC))
    if scheme == "multinomial":
        zr, bz = spacings_ref(np.asarray(u)[:M + 1])
        if z is not None:
            within("multinomial spacings", z, zr, bz)
            if cdf is not None:
                check_search_exact(scheme, A, cdf, np.asarray(z)[:M] / np.asarray(z)[M])
        su, bsu = grid_bound(zr, bz, M)
    else:
        su = su_of(scheme, u, M)
        bsu = np.zeros(M, dtype=LD)
        if cdf is not None:
            check_search_exact(scheme, A, cdf, su)
    return check_ancestors(scheme, A, C, bC, su, bsu, W)


def residual_parts(W, M):
    """floor(M W), sip and res / sres as the reference and the kernel compute them: M W is one rounding and the rest
    is exact, so these are the same fp64 values on both sides."""
    W = np.asarray(W, dtype=np.float64)
    MW = M * W
    ip = np.floor(MW).astype(np.int64)
    sip = int(ip.sum())
    sres = M - sip
    with np.errstate(invalid="ignore", divide="ignore"):
        res = (MW - ip) / sres
    return ip, sip, sres, res


def check_residual(W, M, u, A, cdf=None, z=None):
    """A[:sip] = arange(N).repeat(floor(M W)) bit for bit; the sres stochastic draws as multinomial on res / sres
    over the first sres + 1 uniforms."""
    W = np.asarray(W, dtype=np.float64)
    A = np.asarray(A)
    ip, sip, sres, res = residual_parts(W, M)
    assert A.size == M
    assert np.array_equal(A[:sip], np.arange(W.size).repeat(ip)), "residual: deterministic part"
    if sres == 0:
        return 0
    C, bC = cdf_ref(res)
    zr, bz = spacings_ref(np.asarray(u)[:sres + 1])
    if cdf is not None:
        check_cdf("residual CDF", cdf, res)
    if z is not None:
        within("residual spacings", np.asarray(z)[:sres + 1], zr, bz)
        if cdf is not None:
            check_search_exact("residual", A[sip:], cdf, np.asarray(z)[:sres] / np.asarray(z)[sres])
    su, bsu = grid_bound(zr, bz, sres)
    return check_ancestors("residual", A[sip:], C, bC, su, bsu, res)


def check_killing(W, u, u_mult, A):
    """Particle i survives iff not u_i max(W) >= W_i (IEEE, exact); the killed slots, in order, hold a multinomial
    draw of nkilled over u_mult."""
    W = np.asarray(W, dtype=np.float64)
    A = np.asarray(A)
    killed = np.asarray(u) * W.max() >= W
    n = W.size
    assert np.array_equal(A[~killed], np.arange(n)[~killed]), "killing: a survivor moved"
    nk = int(killed.sum())
    if nk == 0:
        return 0, 0
    return nk, check_inverse_cdf("multinomial", W, nk, u_mult, A[killed])


# ------------------------------------------------------------------------------------------- distributions
def _lsbounds(x, loc, scale):
    x, loc, scale = (np.asarray(v, dtype=np.float64) for v in (x, loc, scale))
    z = (_ld(x) - _ld(loc)) / _ld(scale)
    return z, scale.astype(LD)


def normal_logpdf_ref(x, loc, scale):
    """scipy.stats.norm.logpdf's -z^2 / 2 - log(2 pi) / 2 - log(scale): z is two roundings (|z| eps), z^2 / 2 three
    more, the constant is the kernel's fp64 one, log one ulp, two additions."""
    z, s = _lsbounds(x, loc, scale)
    with np.errstate(invalid="ignore", over="ignore"):
        r = -z * z / 2 - LD(HALFLOG2PI) - np.log(s)
        b = SAFETY * LD(EPS) * (3 * z * z + 2 * np.abs(np.log(s)) + 2 + np.abs(r))
    return _overflow_rule(r, x, loc, scale), b


def _overflow_rule(r, x, loc, scale):
    """-inf wherever z^2 overflows in fp64 for a finite z, as it does in scipy's formula and in the kernel's."""
    with np.errstate(invalid="ignore", over="ignore"):
        z64 = (np.asarray(x, dtype=np.float64) - loc) / scale
        over = np.isinf(z64 * z64) & np.isfinite(z64)
    return np.where(over, LD(-np.inf), r)


def student_logpdf_ref(x, df, c0, loc, scale):
    """scipy.stats.t.logpdf with the kernel's host constant c0: c0 - (df + 1) / 2 log1p(z^2 / df) - log(scale).
    y = z^2 / df carries 5 roundings of y (so log1p's argument error moves its value by <= 5 eps y / (1 + y) <= 5 eps),
    log1p one ulp, (df + 1) / 2 and the product two, log one, two additions.  z^2 overflows in fp64 exactly where
    scipy's does: -inf there."""
    z, s = _lsbounds(x, loc, scale)
    df = LD(df)
    with np.errstate(invalid="ignore", over="ignore"):
        t1 = (df + 1) / 2 * np.log1p(z * z / df)
        r = LD(c0) - t1 - np.log(s)
        b = SAFETY * LD(EPS) * (3 * np.abs(t1) + 6 * (df + 1) / 2 + 2 * np.abs(np.log(s)) + np.abs(r) + abs(LD(c0)))
    return _overflow_rule(r, x, loc, scale), b


def gamma_logpdf_ref(x, a, c0, b):
    """scipy.stats.gamma.logpdf(x, a, scale=1/b) with the kernel's c0 = -gammaln(a): a log b + c0 + xlogy(a - 1, x)
    - b x, with xlogy's rules: (a - 1) log x is 0 when a == 1, at x = 0 as at x = +inf; x < 0 gives -inf, NaN gives NaN,
    and +inf gives -inf for a <= 1 and NaN (inf - inf) for a > 1.  Two roundings per term, three additions."""
    x = np.asarray(x, dtype=np.float64)
    b = np.broadcast_to(np.asarray(b, dtype=np.float64), x.shape)
    xl, bl, al = _ld(x), _ld(b), LD(a)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        t1 = al * np.log(bl)
        t2 = LD(0) * xl if a == 1.0 else (al - 1) * np.log(np.where(x < 0, np.nan, xl))
        t2 = np.where(a == 1.0, LD(0), t2)
        t3 = bl * xl
        r = t1 + LD(c0) + t2 - t3
        bound = SAFETY * LD(EPS) * (2 * (np.abs(t1) + np.abs(t2) + np.abs(t3) + abs(LD(c0))) + np.abs(r))
    r = np.where(x < 0, LD(-np.inf), r)
    r = np.where(np.isnan(x), LD(np.nan), r)
    return r, bound


def laplace_logpdf_ref(x, loc, scale):
    """-log(2 scale) - |x - loc| / scale, the log of the density.  scipy.stats.laplace.logpdf takes log(pdf) and so
    gives -inf once the density underflows (|z| > ~745); the kernel keeps the finite value.  Two roundings per term,
    one addition."""
    z, s = _lsbounds(x, loc, scale)
    with np.errstate(invalid="ignore"):
        r = -np.log(2 * s) - np.abs(z)
        b = SAFETY * LD(EPS) * (2 * np.abs(np.log(2 * s)) + 2 * np.abs(z) + np.abs(r))
    return r, b


def logistic_logpdf_ref(x, loc, scale):
    """scipy.stats.logistic.logpdf: y - 2 log1p(exp(y)) - log(scale) with y = -|z| (symmetric, no overflow).  y has
    |z| eps, exp one ulp more and (|z| eps) through its argument, log1p one ulp; log one; two additions."""
    z, s = _lsbounds(x, loc, scale)
    y = -np.abs(z)
    with np.errstate(invalid="ignore"):
        r = y - 2 * np.log1p(np.exp(y)) - np.log(s)
        b = SAFETY * LD(EPS) * (2 * np.abs(z) + 6 + 2 * np.abs(np.log(s)) + np.abs(r))
    return r, b


def logistic_logpdf_overflowing(x, loc, scale):
    """The form -z - 2 log1p(exp(-z)) - log(scale): exp(-z) overflows for z < -709.78 and gives -inf there."""
    x, loc, scale = (np.asarray(v, dtype=np.float64) for v in (x, loc, scale))
    with np.errstate(over="ignore", invalid="ignore"):
        z = (x - loc) / scale
        return -z - 2.0 * np.log1p(np.exp(-z)) - np.log(scale)


def _mvn_cols(v, d, n, default):
    """(d, n) long-double parameter from a (d,) host vector or a (d, n) SoA array."""
    if v is None:
        return np.full((d, n), LD(default))
    a = np.asarray(v, dtype=np.float64)
    return np.broadcast_to(_ld(a).reshape(d, -1), (d, n)) if a.ndim == 1 else _ld(a)


def mvn_logpdf_ref(L, x, loc=None, scale=None):
    """MvNormal.logpdf (distributions.py:949-959) on SoA x (d, n): b = (x - loc) / scale, z = L^{-1} b by forward
    substitution in long double on the fp64 factor the kernel receives, -|z|^2 / 2 - sum log scale - sum log L_aa -
    d log(2 pi) / 2.  The kernel's forward substitution solves (L + dL) z = b with |dL| <= (d + 1) eps |L|
    (componentwise), and b carries two roundings, so |dz| <= |L^{-1}| ((d + 1) eps |L| |z| + 2 eps |b|): the bound
    grows with the factor's Skeel condition number.  ss adds 2 |z| |dz| per component plus d roundings, the log sums
    one ulp per term."""
    L = np.asarray(L, dtype=np.float64)
    d = L.shape[0]
    x = np.asarray(x, dtype=np.float64).reshape(d, -1)
    n = x.shape[1]
    Ll = _ld(L)
    lo, sc = _mvn_cols(loc, d, n, 0.0), _mvn_cols(scale, d, n, 1.0)
    bvec = (_ld(x) - lo) / sc
    z = np.empty_like(bvec)
    for a in range(d):
        z[a] = (bvec[a] - (Ll[a, :a, None] * z[:a]).sum(0)) / Ll[a, a]
    Linv = np.abs(np.linalg.inv(L)).astype(LD)
    e = SAFETY * LD(EPS)
    dz = Linv @ ((d + 1) * e * (np.abs(Ll) @ np.abs(z)) + 2 * e * np.abs(bvec))
    ss = (z * z).sum(0)
    logs = np.log(sc)
    hl = np.log(np.diag(Ll)).sum()
    r = -ss / 2 - logs.sum(0) - hl - d * HALFLOG2PI_LD
    b = (2 * np.abs(z) * dz + dz * dz).sum(0) / 2 + e * d * ss + e * (np.abs(logs).sum(0) + np.abs(hl) + d) * 2 \
        + e * (d + 2) * np.abs(r)
    return r, b


def mvn_rvs_ref(L, zs, loc=None, scale=None, dz=None):
    """MvNormal.rvs (distributions.py:946-947, 961-969) on SoA normals zs (d, n): loc + scale * (L z), in long
    double.  The kernel's row a sums a + 1 products in order (a + 2 roundings on sum |L_ab z_b|), then one product
    and one addition; ``dz``, the bound of the normals themselves, enters through |scale| |L| dz."""
    L = np.asarray(L, dtype=np.float64)
    d = L.shape[0]
    zl = np.asarray(zs, dtype=LD).reshape(d, -1)
    n = zl.shape[1]
    Ll = _ld(L)
    lo, sc = _mvn_cols(loc, d, n, 0.0), _mvn_cols(scale, d, n, 1.0)
    acc = Ll @ zl
    r = lo + sc * acc
    e = SAFETY * LD(EPS)
    ab = np.abs(Ll) @ np.abs(zl)
    b = np.abs(sc) * ab * e * (np.arange(d, dtype=LD)[:, None] + 3) + e * np.abs(r)
    if dz is not None:
        b = b + np.abs(sc) * (np.abs(Ll) @ np.asarray(dz, dtype=LD).reshape(d, -1))
    return r, b


# -------------------------------------------------------------------------------------------------- draws
API = philox_ref.PURPOSE_API


def w3_api(call, field=0, wide=False):
    """Word 3 of an API draw's counter: (call >> 32) above the purpose byte, or above a 8-bit ``field`` (a
    component, or a component pair) in the MvNormal kernels."""
    hi = call >> 32
    return (((hi << 16) | (field << 8)) if wide else (hi << 8)) | API


def api_uniforms(n, call, seed):
    """k_uniform: u[2p], u[2p + 1] from counter (p, call, w3) -- exact bits."""
    return philox_ref.uniforms(n, call & 0xFFFFFFFF, seed, w3=w3_api(call))


def _bm_ld(r):
    """Box-Muller on Philox words in long double: (z0, z1, rad)."""
    u1 = philox_ref.u53_open(r[0], r[1]).astype(LD)
    u2 = philox_ref.u53(r[2], r[3]).astype(LD)
    rad = np.sqrt(-2 * np.log(u1))
    return rad * np.cos(2 * PI_LD * u2), rad * np.sin(2 * PI_LD * u2), rad


def normal_bound(rad):
    """The kernels' box_muller: log (1 ulp), the product by -2 (exact) and sqrt (half an ulp) make rad's relative
    error <= 1 eps; sincospi is within 1 ulp of 1 and the product rounds once: |dz| <= 3 eps rad."""
    return SAFETY * 3 * LD(EPS) * rad


def api_normals(n, call, seed, field=None, wide=False):
    """k_std_normal / k_normal_rvs (field None) and k_mvn_rvs (field = component k, wide): pair p of the counter
    (p, call, w3) gives values 2p and 2p + 1.  Returns (z, bound) in long double."""
    npairs = (n + 1) // 2
    r = philox_ref._ctr(np.arange(npairs), call & 0xFFFFFFFF, w3_api(call, field or 0, wide), seed)
    z0, z1, rad = _bm_ld(r)
    z = np.empty(2 * npairs, dtype=LD)
    z[0::2], z[1::2] = z0, z1
    b = np.repeat(normal_bound(rad), 2)
    return z[:n], b[:n]


def mvn_small_normals(n, d, call, seed):
    """k_mvn_rvs (d <= 8): component k of particles 2p, 2p + 1 from counter (p, call, (k << 8) | purpose)."""
    zs, bs = zip(*[api_normals(n, call, seed, field=k, wide=True) for k in range(d)])
    return np.stack(zs), np.stack(bs)


def mvn_big_normals(n, d, call, seed):
    """k_mvn_big<false> (8 < d <= 32): one counter per particle i, components 2j and 2j + 1 from (i, call,
    (j << 8) | purpose)."""
    z = np.empty((d + 1, n), dtype=LD)
    b = np.empty((d + 1, n), dtype=LD)
    for j in range((d + 1) // 2):
        r = philox_ref._ctr(np.arange(n), call & 0xFFFFFFFF, w3_api(call, j, True), seed)
        z0, z1, rad = _bm_ld(r)
        z[2 * j], z[2 * j + 1] = z0, z1
        b[2 * j] = b[2 * j + 1] = normal_bound(rad)
    return z[:d], b[:d]
