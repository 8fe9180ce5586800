"""High-precision reference of the binary-space kernels of ``csrc/smcb_binary.cu`` (TEST INFRASTRUCTURE).

NumPy in fp64 and ``np.longdouble`` (x87 extended precision, unit roundoff 2^-64), as ``sampler_replay`` does: the
long-double values stand in for exact ones and every bound counts the kernels' fp64 roundings only.

* the launch geometry (``bin_warps`` / ``bin_smem``, particle -> (CTA, warp)), so a test can assert the tier it reaches;
* ``chol_ld``: ``chol_and_friends`` of the gammas in long double, grouped by |gamma| so that the factorisation is
  vectorised over the particles, with a per-particle bound on the kernel's ldet and wtw from the Cholesky backward
  error; ``vs_ld``: the three models' llik and the IID(Bernoulli(q), p) prior from a descriptor's constants;
* ``nl_ld``: the nested-logistic probabilities coordinate by coordinate, conditioned on the kernel's own bits, with
  the interval each fp64 probability lies in, the bits that interval decides and the logpdf bound;
* ``check_generation``: one generation of the fused waste-free move replayed from the kernel's own previous row;
* the Philox counter layouts of ``bin_uniform`` (built on ``philox_ref._ctr``).

``gamma(k) = k u / (1 - k u)`` bounds the relative error of k chained fp64 roundings (Higham, Accuracy and Stability
of Numerical Algorithms, 3.1).  Every bound below is its first-order sum of terms times ``SAFETY``.  The library is
built with ``-fmad=false``, so no product is contracted into an fma behind the bounds' back.
"""
import numpy as np

import philox_ref

LD = np.longdouble
U = np.finfo(np.float64).eps / 2                     # fp64 unit roundoff
EPS = np.finfo(np.float64).eps
SAFETY = 4.0                                         # the one factor every bound carries (first-order terms, |L| of
                                                     # the long-double factor standing in for the kernel's)
LOG_CLIP = 1e-300                                    # log_no_warn's floor

# launch geometry of csrc/smcb_binary.cu
MAX_P = 128                                          # kBinMaxP
SMEM_BUDGET = 200 * 1024                             # kBinSmemBudget
WARP_CAP = 8
NL_BLOCK = 128                                       # k_nested_logistic: one thread per particle
PURPOSE_PROP, PURPOSE_ACC, PURPOSE_RVS = 4, 5, 6


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def tri(a):
    return a * (a + 1) // 2


def bin_warps(k):
    """Warps per CTA for a per-warp triangle of tri(k + 1) doubles plus kBinMaxP ints of indices."""
    return min(SMEM_BUDGET // (tri(k + 1) * 8 + MAX_P * 4), WARP_CAP)


def bin_smem(k, wpc):
    return wpc * (tri(k + 1) * 8 + MAX_P * 4)


def cta_warp(i, wpc):
    """(CTA, warp) of particle / chain i in a launch of ``wpc`` warps per CTA."""
    return int(i) // wpc, int(i) % wpc


def words(p):
    """32-bit words of a p-bit row."""
    return -(-p // 32)


# ----------------------------------------------------------------------------------------- chol_and_friends
def _chol_group(A, B):
    """Long-double Cholesky of the (m, k, k) batch A and w = L^-1 B: (L, w, ok) with ok = every pivot > 0."""
    m, k, _ = A.shape
    L = np.zeros((m, k, k), dtype=LD)
    w = np.zeros((m, k), dtype=LD)
    ok = np.ones(m, dtype=bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        for j in range(k):
            lj = L[:, j, :j]
            piv = A[:, j, j] - np.sum(lj * lj, axis=1)
            ok &= piv > 0
            piv = np.where(ok, piv, LD(np.nan))
            L[:, j, j] = np.sqrt(piv)
            w[:, j] = (B[:, j] - np.sum(lj * w[:, :j], axis=1)) / L[:, j, j]
            if j + 1 < k:
                L[:, j + 1:, j] = (A[:, j + 1:, j] - np.matmul(L[:, j + 1:, :j], lj[:, :, None])[:, :, 0]) \
                    / L[:, j, j][:, None]
    return L, w, ok


def chol_ld(gam, xtx, xty, vm2, chunk=192):
    """chol_and_friends of the (N, p) bool ``gam`` in long double: dict of len_gam (exact), ldet, wtw (long double;
    NaN where a pivot is not positive, ``ok`` False), and the bounds ``b_ldet``, ``b_wtw`` on the kernel's values.

    The kernel factors the augmented (k + 1)-row matrix [A b; b^T .] (A = X^T X[gamma, gamma] + vm2 I, b = X^T y[gamma])
    right-looking, so its factor [L 0; w^T .] satisfies [L 0; w^T .][L 0; w^T .]^T = [A + dA, b + db; ...] with
    |[dA db]| <= gamma(k + 2) |L_aug| |L_aug|^T (Higham Theorem 10.3 on k + 1 rows, plus the rounding of A_ii + vm2).
    Linearised:
      ldet = sum log l_jj = log det (A + dA) / 2:       1/2 |A^-1| : |dA|
                 k logs, each within 1 ulp:             + 2 u sum |log l_jj|
                 their sum in order:                    + gamma(k) sum |log l_jj|
      wtw = (b + db)^T (A + dA)^-1 (b + db), v = A^-1 b: |v~|^T |dA_aug| |v~| with v~ = (v, -1)
                                                        (= |v|^T |dA| |v| + 2 |v|^T |db|: the forward substitution)
                 the sum of squares (a lane's ceil(k / 32) terms in order, 5 butterfly levels, the squares):
                                                        + gamma(ceil(k / 32) + 6) sum w^2
    """
    gam = np.asarray(gam, dtype=bool)
    N = gam.shape[0]
    kk = gam.sum(axis=1)
    out = {"len_gam": kk.astype(np.float64), "ldet": np.zeros(N, LD), "wtw": np.zeros(N, LD),
           "b_ldet": np.zeros(N), "b_wtw": np.zeros(N), "ok": np.ones(N, dtype=bool)}
    X = np.asarray(xtx, np.float64).astype(LD)
    b = np.asarray(xty, np.float64).astype(LD)
    for k in np.unique(kk):
        if k == 0:
            continue
        rows_all = np.flatnonzero(kk == k)
        for c0 in range(0, len(rows_all), chunk):
            rows = rows_all[c0:c0 + chunk]
            m = len(rows)
            idx = np.nonzero(gam[rows])[1].reshape(m, k)          # ascending, as boolean indexing takes them
            A = X[idx[:, :, None], idx[:, None, :]] + LD(vm2) * np.eye(k, dtype=LD)[None]
            B = b[idx]
            L, w, ok = _chol_group(A, B)
            with np.errstate(invalid="ignore", divide="ignore"):
                dg = np.diagonal(L, axis1=1, axis2=2)
                logs = np.log(dg)
                ldet = logs.sum(axis=1)
                wtw = (w * w).sum(axis=1)
            out["ldet"][rows] = np.where(ok, ldet, LD(np.nan))
            out["wtw"][rows] = np.where(ok, wtw, LD(np.nan))
            out["ok"][rows] = ok
            bl = np.full(m, np.nan)
            bw = np.full(m, np.nan)
            g = ok
            if g.any():
                Lf = L[g].astype(np.float64)
                wf = w[g].astype(np.float64)
                Laug = np.zeros((Lf.shape[0], k + 1, k + 1))
                Laug[:, :k, :k] = Lf
                Laug[:, k, :k] = wf
                G = gamma(k + 2) * np.abs(Laug) @ np.abs(Laug).transpose(0, 2, 1)       # |dA_aug| bound
                Linv = np.linalg.inv(Lf)
                Ainv = Linv.transpose(0, 2, 1) @ Linv
                v = (Ainv @ np.asarray(B[g], np.float64)[:, :, None])[:, :, 0]
                vt = np.abs(np.concatenate([v, -np.ones((v.shape[0], 1))], axis=1))
                la = np.abs(logs[g].astype(np.float64)).sum(axis=1)
                bl[g] = 0.5 * np.sum(np.abs(Ainv) * G[:, :k, :k], axis=(1, 2)) + (2 * U + gamma(k)) * la
                bw[g] = np.einsum("mi,mij,mj->m", vt, G, vt) + gamma(-(-k // 32) + 6) * wtw[g].astype(np.float64)
            out["b_ldet"][rows] = SAFETY * bl
            out["b_wtw"][rows] = SAFETY * bw
    return out


def iid_prior(gam, lq, l1q):
    """IID(Bernoulli(q), p).logpdf as the kernels add it: p terms in coordinate order, in fp64 -- exact."""
    gam = np.asarray(gam, dtype=bool)
    lp = np.zeros(gam.shape[0])
    for i in range(gam.shape[1]):
        lp = lp + np.where(gam[:, i], lq, l1q)
    return lp


class Desc:
    """The constants of an smcb_vs_desc (fp64, as the kernels receive them) and the design's X^T X, X^T y."""

    def __init__(self, xtx, xty, use_ldet=0, vm2=0.0, coef_len=0.0, coef_log=0.0, coef_in_log=1.0, gw=1.0, q=0.5):
        self.xtx = np.ascontiguousarray(xtx, dtype=np.float64)
        self.xty = np.ascontiguousarray(xty, dtype=np.float64)
        self.p = self.xtx.shape[0]
        self.use_ldet, self.vm2 = int(use_ldet), float(vm2)
        self.coef_len, self.coef_log, self.coef_in_log, self.gw = (float(coef_len), float(coef_log),
                                                                   float(coef_in_log), float(gw))
        with np.errstate(divide="ignore"):
            self.lq = float(np.log(np.clip(q, LOG_CLIP, None)))
            self.l1q = float(np.log(np.clip(1.0 - q, LOG_CLIP, None)))

    @classmethod
    def of_model(cls, m, q=0.5):
        """The descriptor a particles_b200.binary_smc model builds (VariableSelection._desc)."""
        return cls(m.xtx, m.xty, m.use_ldet, m.iv2, m.coef_len, m.coef_log, m.coef_in_log, m._gw(), q)


def vs_ld(desc, gam, epn=0.0, chol=None):
    """All outputs of smcb_vs_loglik in long double with their bounds: dict of len_gam, ldet, wtw, lprior (fp64,
    exact), in_log, llik, lpost and b_ldet, b_wtw, b_in, b_llik, b_lpost; ``ok`` (every pivot > 0) and ``near0``
    (the long-double in_log within its bound of 0, where log(in_log) is not determined by the kernel's rounding).

      in_log = coef_in_log - gw wtw:     |gw| b_wtw + u |gw wtw| (the product) + u |in_log| (the difference)
      log(in_log):                       b_in / in_log (first order) + 2 u |log in_log| (1 ulp)
      llik = -(coef_len k [+ ldet] + coef_log log(in_log)):
                                         [b_ldet] + |coef_log| b_log + u |coef_len k| + u |coef_log log|
                                         + 2 u (|lead| [+ |ldet|] + |coef_log log|) (two additions)
      lpost = lprior + epn llik:         epn b_llik + u |epn llik| + u |lpost|; lprior itself when epn == 0
    The ldet / wtw bounds already carry SAFETY; the roundings added here are multiplied by it too.  ``chol``: a
    chol_ld result for the same gammas, X^T X, X^T y and vm2, to reuse."""
    c = dict(chol_ld(gam, desc.xtx, desc.xty, desc.vm2) if chol is None else chol)
    k = c["len_gam"]
    lpr = iid_prior(gam, desc.lq, desc.l1q)
    with np.errstate(invalid="ignore", divide="ignore"):
        gw = LD(desc.gw)
        in_log = LD(desc.coef_in_log) - gw * c["wtw"]
        b_in = abs(desc.gw) * c["b_wtw"] + SAFETY * U * (np.abs(np.float64(desc.gw) * c["wtw"].astype(np.float64))
                                                          + np.abs(in_log.astype(np.float64)))
        near0 = c["ok"] & ~(np.abs(in_log.astype(np.float64)) > b_in)
        lg = np.log(in_log)
        b_log = b_in / np.abs(in_log.astype(np.float64)) + SAFETY * 2 * U * np.abs(lg.astype(np.float64))
        lead = LD(desc.coef_len) * LD(1) * k.astype(LD)
        term = LD(desc.coef_log) * lg
        s = lead + term + (c["ldet"] if desc.use_ldet else LD(0))
        llik = -s
        al, at, ad = (np.abs(lead.astype(np.float64)), np.abs(term.astype(np.float64)),
                      np.abs(c["ldet"].astype(np.float64)) if desc.use_ldet else 0.0)
        b_ll = (c["b_ldet"] if desc.use_ldet else 0.0) + abs(desc.coef_log) * b_log + \
            SAFETY * U * (al + at + 2 * (al + ad + at))
    llik = np.where(c["ok"], llik, LD(-np.inf))
    b_ll = np.where(c["ok"], b_ll, 0.0)
    b_ll = np.where(near0, np.inf, b_ll)
    c.update(lprior=lpr, in_log=in_log, b_in=b_in, llik=llik, b_llik=b_ll, near0=near0)
    c["lpost"], c["b_lpost"] = post_ld(lpr, llik, b_ll, epn)
    return c


def post_ld(lpr, llik, b_ll, epn):
    if not epn > 0:
        return lpr.astype(LD), np.zeros(len(lpr))
    with np.errstate(invalid="ignore"):
        post = lpr.astype(LD) + LD(epn) * llik
        b = epn * b_ll + SAFETY * U * (np.abs(epn * llik.astype(np.float64)) + np.abs(post.astype(np.float64)))
    b = np.where(np.isinf(llik), 0.0, b)
    return post, b


def assert_close(what, got, want, bound, where="particle", wpc=None):
    """|got - want| <= bound entry by entry; equal infinities and NaN on both sides count as equal.  The failure
    names the first bad entry and, given ``wpc``, its CTA and warp."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), got.shape)
    with np.errstate(invalid="ignore"):
        diff = np.abs(got.astype(LD) - want.astype(LD)).astype(np.float64)
        wf = want.astype(np.float64)
        same = (got == wf) | (np.isnan(got) & np.isnan(wf))
        bad = ~same & ~(diff <= bound)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        at = f" (CTA {i // wpc}, warp {i % wpc})" if wpc else ""
        raise AssertionError(f"{what}: {where} {i}{at}: {got[i]!r} vs {float(want[i])!r} (|diff| {diff[i]:.3e} > "
                             f"bound {bound[i]:.3e}; {int(bad.sum())} of {bad.size} entries)")


# ----------------------------------------------------------------------------------------- nested logistic
def _pr_interval(z, dz):
    """pr = 1 / (1 + exp(-z)) in long double for the long-double logits z with the kernel's logit error dz, and the
    interval [lo, hi] that holds the kernel's fp64 pr: exp within 1 ulp, then 1 + e and the quotient give
    dpr = pr (1 - pr) (dz + 2 u) + 2 u pr.  Two cases are exact whatever the rounding: exp(-z) <= 2^-53 makes
    1 + e == 1 and pr == 1 (a saturated logit: the reference's 1 - pr is then 0 and hits the clip too), and exp(-z)
    beyond fp64's range makes pr == 0.  Between them, exp(-z) > 2^-53 for sure keeps pr <= 1 - 2^-52: near 1 the
    fp64 1 - pr is quantised to 2^-53, so log(1 - pr) is known to O(1) there -- in the reference's fp64 too."""
    with np.errstate(over="ignore", invalid="ignore"):
        pr = 1 / (1 + np.exp(-z))
        prf = pr.astype(np.float64)
        dpr = SAFETY * (prf * (1 - prf) * (dz + 2 * U) + 2 * U * prf)
        lo, hi = np.maximum(prf - dpr, 0.0), np.minimum(prf + dpr, 1.0)
        zf = z.astype(np.float64)
        one = np.exp(-zf + dz) * (1 + 8 * U) <= 2.0 ** -53
        zero = -zf - dz > 709.8
        # exp(-z) > 2^-53 for sure: 1 + e >= 1 + 2^-52, so pr <= fl(1 / (1 + 2^-52)) = 1 - 2^-52
        below = np.exp(-zf - dz) * (1 - 8 * U) > 2.0 ** -53
    hi = np.where(below, np.minimum(hi, 1.0 - 2.0 ** -52), hi)
    lo = np.minimum(lo, hi)
    lo, hi = np.where(one, 1.0, np.where(zero, 0.0, lo)), np.where(one, 1.0, np.where(zero, 0.0, hi))
    return np.where(one, LD(1), np.where(zero, LD(0), pr)), lo, hi


def nl_ld(coeffs, edgy, x):
    """NestedLogistic.predict_prob for every coordinate of the (n, p) bool rows ``x`` (each coordinate conditioned
    on the bits before it in x -- the kernel's own bits), in long double: (pr, lo, hi) with [lo, hi] an interval that
    holds the kernel's fp64 probability.

    Edgy coordinates: coeffs[i, i] exactly.  Otherwise z = c_ii + sum_{j<i} c_ij x_j, a sum with at most i + 7
    roundings along any path (a thread adds in order; a warp adds 4 words per lane and 5 butterfly levels):
    dz = gamma(i + 7) (|c_ii| + sum |c_ij| x_j); then ``_pr_interval``."""
    c = np.asarray(coeffs, np.float64)
    edgy = np.asarray(edgy, dtype=bool)
    x = np.asarray(x, dtype=bool)
    n, p = x.shape
    cl = np.tril(c, -1)
    diag = np.diag(c)
    with np.errstate(over="ignore", invalid="ignore"):
        z = diag.astype(LD)[None, :] + x.astype(LD) @ cl.astype(LD).T
        dz = SAFETY * gamma(np.arange(p) + 7)[None, :] * (np.abs(diag)[None, :] + x.astype(np.float64) @ np.abs(cl).T)
    pr, lo, hi = _pr_interval(z, dz)
    ed = np.broadcast_to(edgy[None, :], (n, p))
    return (np.where(ed, diag.astype(LD)[None, :], pr), np.where(ed, diag[None, :], lo),
            np.where(ed, diag[None, :], hi))


def nl_bits(u, lo, hi):
    """The kernel's bit ``u < pr`` (strict, Bernoulli.rvs) where [lo, hi] decides it: (bit, decided)."""
    u = np.asarray(u, np.float64)
    return u < lo, (u < lo) | (u >= hi)


def nl_logpdf(x, lo, hi):
    """The logpdf of the rows x from the probability intervals: (long-double midpoint, bound).  Each term is
    log_no_warn of pr or of 1 - pr over the interval (exact where both ends sit at the 1e-300 clip), plus the log's
    ulp and one rounding of 1 - pr (u, absolute after the log); the p terms are added in order: gamma(p) sum |term|."""
    x = np.asarray(x, dtype=bool)
    a = np.where(x, lo, 1.0 - hi).astype(LD)
    b = np.where(x, hi, 1.0 - lo).astype(LD)
    with np.errstate(divide="ignore"):
        la = np.log(np.maximum(a, LD(LOG_CLIP)))
        lb = np.log(np.maximum(b, LD(LOG_CLIP)))
    mid = (la + lb) / 2
    hw = ((lb - la) / 2).astype(np.float64)
    am = np.abs(mid.astype(np.float64))
    p = x.shape[1]
    bound = hw.sum(axis=1) + SAFETY * (U + 2 * U * am).sum(axis=1) + SAFETY * gamma(p) * am.sum(axis=1)
    return mid.sum(axis=1), bound


def nl_replay_draw(coeffs, edgy, u, follow=None):
    """Replay NestedLogistic.rvs from the uniforms ``u`` (p, n) coordinate by coordinate, with the probability
    intervals of ``nl_ld``.  Where a bit is undecided the replay takes ``follow``'s bit (the kernel's own) when given,
    so that later coordinates are conditioned on what the kernel drew.  Returns (bits (n, p), decided (n, p),
    mismatch (n, p): decided bits that differ from ``follow``)."""
    c = np.asarray(coeffs, np.float64)
    edgy = np.asarray(edgy, dtype=bool)
    u = np.asarray(u, np.float64)
    p, n = u.shape
    x = np.zeros((n, p), dtype=bool)
    dec = np.zeros((n, p), dtype=bool)
    mism = np.zeros((n, p), dtype=bool)
    for i in range(p):
        if edgy[i]:
            lo = hi = np.full(n, c[i, i])
        else:
            with np.errstate(over="ignore", invalid="ignore"):
                z = LD(c[i, i]) + x[:, :i].astype(LD) @ c[i, :i].astype(LD)
                dz = SAFETY * gamma(i + 7) * (abs(c[i, i]) + x[:, :i].astype(np.float64) @ np.abs(c[i, :i]))
            _, lo, hi = _pr_interval(z, dz)
        b, d = nl_bits(u[i], lo, hi)
        dec[:, i] = d
        if follow is not None:
            f = np.asarray(follow[:, i], dtype=bool)
            mism[:, i] = d & (b != f)
            b = np.where(d, b, f)
        x[:, i] = b
    return x, dec, mism


# ----------------------------------------------------------------------------------------- Philox layouts
def _u(chains, call, w3, seed):
    r = philox_ref._ctr(np.asarray(chains, dtype=np.uint64), int(call) & 0xFFFFFFFF, int(w3) & 0xFFFFFFFF, seed)
    return philox_ref.u53(r[0], r[1])


def rvs_uniforms(n, p, call, seed):
    """u (p, n) of k_nested_logistic: counter (particle, call, (i << 8) | 6)."""
    return np.stack([_u(np.arange(n), call, (i << 8) | PURPOSE_RVS, seed) for i in range(p)])


def prop_uniforms(M, p, s, call, seed):
    """u (p, M) of step s of k_binary_wf_move's proposal: counter (chain, call, (s << 16) | (i << 8) | 4)."""
    return np.stack([_u(np.arange(M), call, (s << 16) | (i << 8) | PURPOSE_PROP, seed) for i in range(p)])


def acc_uniforms(M, s, call, seed):
    """u (M,) of step s's acceptance: counter (chain, call, (s << 16) | 5)."""
    return _u(np.arange(M), call, (s << 16) | PURPOSE_ACC, seed)


# ----------------------------------------------------------------------------------------- one waste-free generation
def check_generation(s, desc, coeffs, edgy, epn, prev, out, pb, u_prop, u_acc, wpc, chains=None):
    """Generation s of k_binary_wf_move from the kernel's own row s - 1.

    ``prev`` / ``out``: dicts of theta (m, p) bool, lprior, llik, lpost (rows s - 1 and s of the kernel's output, for
    the chains ``chains``, default 0..m-1); ``pb``: its pb_out row s - 1; ``u_prop`` (p, m), ``u_acc`` (m,): the
    draws of step s.  The proposal does not depend on the state, so it is replayed from the uniforms, following the
    kernel's bits where the kernel accepted.  Checks:
      a rejected chain's row is a bit copy of row s - 1 and its three scores (that is how a rejection is recognised);
      an accepted chain's row is the proposal at every decided bit, its lprior is exact and llik / lpost lie inside
      the target's bounds;
      the decision and pb agree with long double wherever the margin |u - pb| exceeds the bound from lp_acc:
        lp_acc = (lpost' - lpost) + (lq_cur - lq_prop): lpost' and both logpdfs' bounds, then three roundings.
    A chain-step is undecided when a proposal bit is undecided and the kernel rejected: its proposal is not known.
    ``pb`` None skips the per-chain pb check (BinaryMetropolis.step returns only the mean).  Returns a dict:
    accepted, undecided (chain-steps), inside (decisions within the bound), known (the chains whose proposal is
    known) and pb, b_pb (long-double pb and its bound for those)."""
    th0 = np.asarray(prev["theta"], dtype=bool)
    th1 = np.asarray(out["theta"], dtype=bool)
    m = th0.shape[0]
    chains = np.arange(m) if chains is None else np.asarray(chains)
    where = lambda j: f"chain {int(chains[j])} (CTA {int(chains[j]) // wpc}, warp {int(chains[j]) % wpc})"
    same = np.all(th1 == th0, axis=1)
    sc_same = np.ones(m, dtype=bool)
    for k in ("lprior", "llik", "lpost"):
        a, b = np.asarray(out[k], np.float64), np.asarray(prev[k], np.float64)
        sc_same &= a.view(np.int64) == b.view(np.int64)
    dev_acc = ~(same & sc_same)
    prop, dec, mism = nl_replay_draw(coeffs, edgy, u_prop, follow=th1)
    bad = mism & dev_acc[:, None]
    if bad.any():
        j = int(np.flatnonzero(bad.any(axis=1))[0])
        i = int(np.flatnonzero(bad[j])[0])
        raise AssertionError(f"generation {s}: {where(j)} accepted a proposal with coordinate {i} = {int(th1[j, i])}, "
                             f"but u = {float(u_prop[i, j])!r} decides the other bit ({int(bad.sum())} bits)")
    undecided = ~dev_acc & ~dec.all(axis=1)
    known = ~undecided
    kn = np.flatnonzero(known)
    t = vs_ld(desc, prop[kn], epn)
    _, lo1, hi1 = nl_ld(coeffs, edgy, prop[kn])
    lq_p, b_qp = nl_logpdf(prop[kn], lo1, hi1)
    _, lo0, hi0 = nl_ld(coeffs, edgy, th0[kn])
    lq_c, b_qc = nl_logpdf(th0[kn], lo0, hi0)
    lp = np.asarray(prev["lpost"], np.float64)[kn]
    with np.errstate(invalid="ignore", over="ignore"):
        d1 = t["lpost"] - lp.astype(LD)
        dq = lq_c - lq_p
        lp_acc = d1 + dq
        # three roundings, of terms no larger than |lpost'| + |lpost| + |dq| in either order of the sums (the fused
        # move adds (lpost' - lpost) + dq, BinaryMetropolis.step (lpost' + dq) - lpost)
        tol = t["b_lpost"] + b_qp + b_qc + SAFETY * U * 3 * (np.abs(t["lpost"].astype(np.float64)) + np.abs(lp)
                                                              + np.abs(dq.astype(np.float64)))
        tol = np.where(np.isfinite(tol), tol, np.inf)
        tol = np.where(np.isfinite(lp_acc.astype(np.float64)), tol, 0.0)     # -inf / +inf / NaN are exact
        want_pb = np.exp(np.minimum(lp_acc, 0))
        wpb = want_pb.astype(np.float64)
        # plus one subnormal ulp: below 2^-1022 exp's error is absolute (pb = 0 where long double gives 5e-324)
        b_pb = wpb * np.expm1(np.minimum(tol, 700.0)) + SAFETY * 2 * U * wpb + SAFETY * 2.0 ** -1074
        b_pb = np.where(lp_acc.astype(np.float64) - tol > 0, 0.0, b_pb)          # lp_acc > 0 for sure: pb == 1
        u = np.asarray(u_acc, np.float64)[kn]
        want_acc = u < wpb
        decided = np.isnan(wpb) | (b_pb == 0) | (np.abs(u - wpb) > b_pb)
    acc_k = dev_acc[kn]
    # an accepted proposal equal to the state is indistinguishable from a rejection
    flip = decided & (want_acc != acc_k) & ~(want_acc & np.all(prop[kn] == th0[kn], axis=1))
    if flip.any():
        j = int(np.flatnonzero(flip)[0])
        raise AssertionError(f"generation {s}: {where(kn[j])} {'accepted' if acc_k[j] else 'rejected'} but "
                             f"u = {u[j]!r}, pb = {wpb[j]!r} +- {b_pb[j]:.3e} (lp_acc = {float(lp_acc[j])!r}, "
                             f"lpost0 = {lp[j]!r}; {int(flip.sum())} of {len(kn)} decisions)")
    if pb is not None:
        assert_close(f"generation {s}: pb", np.asarray(pb, np.float64)[kn], want_pb, b_pb, "chain (known)")
    A = acc_k
    if A.any():
        rows = kn[A]
        np.testing.assert_array_equal(np.asarray(out["lprior"], np.float64)[rows], t["lprior"][A],
                                      err_msg=f"generation {s}: accepted lprior")
        assert_close(f"generation {s}: accepted llik", np.asarray(out["llik"], np.float64)[rows], t["llik"][A],
                     t["b_llik"][A], "accepted chain")
        assert_close(f"generation {s}: accepted lpost", np.asarray(out["lpost"], np.float64)[rows], t["lpost"][A],
                     t["b_lpost"][A], "accepted chain")
    return {"accepted": dev_acc, "undecided": int(undecided.sum()), "inside": int((~decided).sum()), "known": kn,
            "pb": want_pb, "b_pb": b_pb}


# ----------------------------------------------------------------------------------------- synthetic designs
def design(kind, p, seed=0, n=None):
    """(X, y) with n = 2 p + 17 rows: ``gauss`` (iid N(0, 1) columns), ``ar1`` (columns an AR(1) with rho = 0.995:
    the correlation matrix's condition number is about 400), ``scaled`` (gauss columns scaled by 10^U(-3, 3)).
    y is a sparse linear model on a few columns plus noise."""
    r = np.random.RandomState(seed)
    n = 2 * p + 17 if n is None else n
    X = r.standard_normal((n, p))
    if kind == "ar1":
        rho = 0.995
        for j in range(1, p):
            X[:, j] = rho * X[:, j - 1] + np.sqrt(1 - rho * rho) * X[:, j]
    elif kind == "scaled":
        X = X * 10.0 ** r.uniform(-3, 3, p)
    beta = np.zeros(p)
    act = r.choice(p, min(p, 5), replace=False)
    beta[act] = r.choice([-1.0, 1.0], len(act)) / np.maximum(X[:, act].std(axis=0), 1e-300)
    y = X @ beta + r.standard_normal(n)
    return X, y


def model_desc(kind, X, y, q=0.5, lamb=None):
    """The descriptor of BIC / BayesianVS / BayesianVS_gprior (binary_smc.py's constants, as binary_oracle.VS and
    particles_b200.binary_smc compute them; ``lamb`` None: the full model's sigma^2)."""
    import binary_oracle as bo
    o = bo.VS(kind, X, y, lamb=lamb)
    if kind == "bic":
        return Desc(o.xtx, o.xty, 0, 0.0, o.coef_len, o.coef_log, o.coef_in_log, 1.0, q)
    if kind == "bvs":
        return Desc(o.xtx, o.xty, 1, o.iv2, o.coef_len, o.coef_log, float(np.reshape(o.coef_in_log, -1)[0]), 1.0, q)
    return Desc(o.xtx, o.xty, 0, 0.0, o.coef_len, o.coef_log, float(np.reshape(o.coef_in_log, -1)[0]), o.gogp1, q)
