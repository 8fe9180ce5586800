"""Per-time-step replay of the smoothing kernels (TEST INFRASTRUCTURE): csrc/smcb_smooth.cu (FFBS: ON2, MCMC,
hybrid reject), csrc/smcb_online.cu (PaRIS draws, ON2 backward weights, the Phi updates) and csrc/smcb_twofilter.cu
(ON2_ROWS, ON_LOGW), in NumPy fp64 and ``np.longdouble``.

``Trans`` is the transition log-density ``PX(t, xp).logpdf(x)`` of each device model (the ``transition_spec`` of
``particles_b200.state_space_models``), evaluated in long double from the same fp64 inputs and constants the kernel
reads, together with a per-pair bound on the kernel's fp64 error.  Each bound is an operation count written beside the
code (u = 2^-53, one rounding of a correctly rounded operation) times the one safety factor ``SAFETY``.

Every check starts from the kernel's own output at t + 1 (its ``idx[t + 1]``, its previous generation), so a bound
covers one step and the two sides cannot drift apart at a near-tie.  Where a decision lies inside its bound the
replay does not guess: it reports the draw as undecided and the caller checks that such draws are rare.

The randomness the kernels draw themselves is restated here: ``smooth_uniforms`` (Philox counter (m, t, call,
(trial << 8) | purpose), u0 from words 0-1, u1 from words 2-3, both ``u53_open``) with the context's key, and
PaRIS's key ``seed ^ kOnlineSeedMix`` with m = n * Np + i, t-field 0 and call = t.
"""
import numpy as np

from philox_ref import philox4x32_10, u53_open

LD = np.longdouble
U = 2.0 ** -53                  # unit roundoff of fp64
EXP_ULP = 1.5                   # fexp_neg / texp_neg / mexp, ulp of the result (asserted in tests/test_math_host.py)
SAFETY = 4.0                    # the one factor every bound carries over its first-order operation count
TINY = 2.0 ** -1022             # exp's error is absolute below the normal range (fexp_neg / texp_neg flush there)
H2PI_SCIPY = float.fromhex("0x1.d67f1c864beb4p-1")    # kHalfLog2PiScipy: np.log(np.sqrt(2 pi))
H2PI = 0.91893853320467274178                         # kHalfLog2Pi (smcb_common.cuh)
PURPOSE_SMOOTH, PURPOSE_EXACT = 4, 5                  # kPurposeSmooth / kPurposeSmoothExact (smcb_smooth.cuh)
ONLINE_SEED_MIX = 0x9E3779B97F4A7C15                  # kOnlineSeedMix (smcb_online.cu)
SM_BLOCK = 256                                        # kSmBlock: trajectories per CTA and particles per ON2 tile

# model codes of include/smcb.h (particles_b200._lib), kept here so that the replay needs no built library
STOCHVOL, LINGAUSS, GORDON, THETALOGISTIC, BEARINGS, MVLINGAUSS, DISCRETECOX, STOCHVOLLEV = range(8)


def f64(a):
    return np.asarray(a, dtype=np.float64)


# ---------------------------------------------------------------------------------------------------- randomness
def smooth_uniforms(seed, call, m, t, trial, purpose):
    """(u0, u1) of smooth_uniforms(key_of(seed), call, m, t, trial, purpose), vectorised over m / t / trial."""
    m, t, trial = np.broadcast_arrays(np.asarray(m, dtype=np.int64), np.asarray(t, dtype=np.int64),
                                      np.asarray(trial, dtype=np.int64))
    w3 = ((trial.astype(np.uint64) << np.uint64(8)) | np.uint64(purpose)).astype(np.uint32)
    r = philox4x32_10(m.astype(np.uint32), t.astype(np.uint32), np.full(m.shape, call & 0xFFFFFFFF, np.uint32), w3,
                      seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return u53_open(r[0], r[1]), u53_open(r[2], r[3])


def paris_seed(seed):
    """The key of the PaRIS draws of a run seeded ``seed``."""
    return (int(seed) ^ ONLINE_SEED_MIX) & (2 ** 64 - 1)


def draw_cdf(cdf, u):
    """draw_cdf (smcb_smooth.cuh): the first j with cdf[j] >= u * cdf[N - 1], at most N - 1."""
    cdf = np.asarray(cdf, dtype=np.float64)
    v = np.asarray(u, dtype=np.float64) * cdf[-1]
    return np.minimum(np.searchsorted(cdf, v, side="left"), cdf.shape[0] - 1).astype(np.int64)


# ------------------------------------------------------------------------------------------ transition density
class Trans:
    """PX(t, xp).logpdf(x) of one device model.  ``spec``: a ``transition_spec`` dict (model, params, dim,
    step_consts).  ``lpdf(t, xp, x)`` broadcasts xp (..., D) against x (..., D) and returns the long-double value
    and the fp64 bound of the kernel's value, per pair."""

    def __init__(self, spec):
        self.model, self.dim = int(spec["model"]), int(spec["dim"])
        self.p = np.asarray(spec["params"], dtype=np.float64)
        sc = spec.get("step_consts")
        self.sc = None if sc is None else np.asarray(sc, dtype=np.float64)
        p = self.p
        if self.model == MVLINGAUSS:
            D = self.dim
            o = 1
            self.F = p[o:o + D * D].reshape(D, D); o += D * D + 4 * D
            self.L = p[o:o + D * D].reshape(D, D); o += D * D
            self.hld = p[o]
        elif self.model == BEARINGS:
            self.s, self.ls = p[0], p[7]
        else:
            # the constant scale of PX and its log: params of smcb_models.cuh, as TransDensity::init reads them
            i, j = {STOCHVOL: (2, 5), STOCHVOLLEV: (2, 5), LINGAUSS: (1, 4), GORDON: (3, 4), THETALOGISTIC: (3, 5),
                    DISCRETECOX: (1, 4)}[self.model]
            self.s, self.ls = p[i], p[j]

    def step_const(self, t):
        return 0.0 if self.sc is None else float(self.sc[t])

    def loc1(self, t, xp):
        """1-D models: the location of PX(t, xp) in long double, and the bound of the kernel's fp64 location."""
        p, x = self.p, np.asarray(xp, dtype=np.float64)
        xl = x.astype(LD)
        if self.model == LINGAUSS:                          # rho * xp: 1 rounding
            loc = LD(p[0]) * xl
            return loc, U * np.abs(f64(loc))
        if self.model in (STOCHVOL, STOCHVOLLEV):           # c0 + rho * xp: 2 roundings (1 if contracted)
            loc = LD(p[4]) + LD(p[1]) * xl
            return loc, 2 * U * (abs(p[4]) + np.abs(p[1] * x))
        if self.model == DISCRETECOX:                       # mu + phi * (xp - mu): 3 roundings
            loc = LD(p[0]) + LD(p[2]) * (xl - LD(p[0]))
            return loc, 3 * U * (abs(p[0]) + np.abs(p[2] * (x - p[0])) + np.abs(x))
        if self.model == GORDON:                            # b xp + c xp / (1 + xp^2) + sc[t]
            sc = LD(self.step_const(t))
            q = LD(p[2]) * xl / (1 + xl * xl)               # xp*xp, 1+, c*xp, /: 4 roundings of q
            loc = LD(p[1]) * xl + q + sc                    # b*xp: 1, two adds: 2 of the sum
            a = np.abs(p[1] * x) + np.abs(f64(q)) + abs(float(sc))
            return loc, 4 * U * np.abs(f64(q)) + U * np.abs(p[1] * x) + 2 * U * a
        if self.model == THETALOGISTIC:                     # xp + tau0 - tau1 * mexp(tau2 * xp)
            a = LD(p[2]) * xl
            E = np.exp(a)
            loc = xl + LD(p[0]) - LD(p[1]) * E
            # tau2 * xp: u|a| of the argument, i.e. u|a| relative on E; mexp: EXP_ULP; tau1 * E: 1; xp + tau0 and
            # the subtraction: 2 roundings of their operands
            tE = np.abs(f64(LD(p[1]) * E))
            b = tE * (U * np.abs(f64(a)) + (EXP_ULP + 1) * U) + 2 * U * (np.abs(x) + abs(p[0]) + tE)
            return loc, b
        raise ValueError(f"no 1-D location for model {self.model}")

    def lpdf(self, t, xp, x):
        xp, x = np.asarray(xp, dtype=np.float64), np.asarray(x, dtype=np.float64)
        if self.model == MVLINGAUSS:
            return self._mvlg(xp, x)
        if self.model == BEARINGS:
            return self._bearings(xp, x)
        if xp.ndim and xp.shape[-1:] == (1,):
            xp = xp[..., 0]
        if x.ndim and x.shape[-1:] == (1,):
            x = x[..., 0]
        loc, dloc = self.loc1(t, xp)
        return self._normal(x, loc, dloc, self.s, self.ls, H2PI_SCIPY)

    @staticmethod
    def _normal(x, loc, dloc, s, ls, c):
        """-z^2/2 - c - ls, z = (x - loc) / s: the kernel's d = x - loc (1 rounding), div_rn (correctly rounded),
        z * z (1), then three subtractions / halvings (2 roundings of the running sum)."""
        d = np.asarray(x, dtype=np.float64).astype(LD) - loc
        z = d / LD(s)
        v = -z * z / 2 - LD(c) - LD(ls)
        az, ad = np.abs(f64(z)), np.abs(f64(d))
        dz = (dloc + U * ad) / s + U * az
        b = az * dz + 0.5 * dz * dz + U * az * az / 2 + 2 * U * (az * az / 2 + c + abs(ls))
        return v, SAFETY * b

    def _bearings(self, xp, x):
        """IndepProd(N(xp0, sX), N(xp1, sX), Dirac(xp0 + xp2), Dirac(xp1 + xp3)): the Dirac locations are one IEEE
        add each, computed here in fp64 exactly as the kernel does, so the Dirac test is exact."""
        xp, x = np.broadcast_arrays(xp, x)
        zero = np.zeros(xp.shape[:-1])
        a, ba = self._normal(x[..., 0], xp[..., 0].astype(LD), zero, self.s, self.ls, H2PI_SCIPY)
        b, bb = self._normal(x[..., 1], xp[..., 1].astype(LD), zero, self.s, self.ls, H2PI_SCIPY)
        dirac = (x[..., 2] == xp[..., 0] + xp[..., 2]) & (x[..., 3] == xp[..., 1] + xp[..., 3])
        v = np.where(dirac, a + b, LD(-np.inf))
        return v, ba + bb + SAFETY * U * np.abs(f64(a + b))

    def _mvlg(self, xp, x):
        """MvNormal(F xp, covX).logpdf(x) with the fp64 Cholesky factor L the kernel reads: F xp as D fmas per
        component, then the fma forward substitution, each zz_i correctly rounded by div_const, ss by D fmas."""
        D, F, L = self.dim, self.F, self.L
        xp, x = np.broadcast_arrays(xp, x)
        FL, LL = F.astype(LD), L.astype(LD)
        loc = np.einsum("...j,ij->...i", xp.astype(LD), FL)
        dloc = D * U * np.einsum("...j,ij->...i", np.abs(xp), np.abs(F))
        d = x.astype(LD) - loc
        zz = np.empty(d.shape, dtype=LD)
        ezz = np.empty(d.shape)
        for i in range(D):
            acc = d[..., i] - (np.einsum("...j,j->...", zz[..., :i], LL[i, :i]) if i else 0)
            mag = np.abs(f64(d[..., i])) + (np.einsum("...j,j->...", np.abs(f64(zz[..., :i])),
                                                              np.abs(L[i, :i])) if i else 0)
            prop = np.einsum("...j,j->...", ezz[..., :i], np.abs(L[i, :i])) if i else 0
            zz[..., i] = acc / LL[i, i]
            # d_i: dloc + 1 rounding; i fmas of the running sum; the quotient: 1 rounding
            eacc = dloc[..., i] + U * np.abs(f64(d[..., i])) + prop + (i + 1) * U * mag
            ezz[..., i] = eacc / abs(L[i, i]) + U * np.abs(f64(zz[..., i]))
        ss = (zz * zz).sum(-1)
        v = -ss / 2 - LD(self.hld) - LD(D) * LD(H2PI)
        azz = np.abs(f64(zz))
        ess = (2 * azz * ezz + ezz * ezz).sum(-1) + D * U * (azz * azz).sum(-1)
        fs = f64(ss)
        b = 0.5 * ess + 3 * U * (fs / 2 + abs(self.hld) + D * H2PI)          # D * c, - hld, - : 3 roundings
        return v, SAFETY * b


def as_rows(X):
    """(N,) or (N, D) particles -> (N, D) fp64 (a host copy of a history generation)."""
    X = np.asarray(X, dtype=np.float64)
    return X.reshape(X.shape[0], -1)


def row_values(trans, t, Xp, lw, xs):
    """v[k, n] = lw[n] + logpt(t, Xp[n], xs[k]) in long double, and the bound of the kernel's fp64 value (the
    addition of lw: 1 rounding).  NaN (a NaN state or log-weight) is kept: see ``exact_draw_check``."""
    Xp, xs = as_rows(Xp), as_rows(xs)
    lp, b = trans.lpdf(t, Xp[None, :, :], xs[:, None, :])
    v = LD(1) * np.asarray(lw, dtype=np.float64)[None, :] + lp
    return v, b + SAFETY * U * np.abs(f64(v))


# ------------------------------------------------------------------------------------------------- exact draws
def row_sums(v, b):
    """Per row: (max, e = exp(v - max), S = sum e, tau), v NaN and -inf weighing zero (the kernels' rule), and tau the
    bound of the kernel's running sums and of its e_n (per-element bound times e_n, EXP_ULP, 2N + 4 roundings of
    the online sums, the absolute floor of exp)."""
    v = np.where(np.isnan(v), LD(-np.inf), v)
    b = np.where(np.isfinite(v), b, 0.0)                   # a term of weight zero carries no error
    mx = v.max(axis=1)
    fin = np.isfinite(mx)
    e = np.where(np.isfinite(v), np.exp(v - np.where(fin, mx, 0)[:, None]), LD(0))
    S = e.sum(axis=1)
    bmx = np.where(fin, np.take_along_axis(b, np.argmax(np.where(np.isnan(v), -np.inf, v), axis=1)[:, None], 1)[:, 0],
                   0)
    N = v.shape[1]
    ef = f64(e)
    tau = (ef * (b + bmx[:, None])).sum(1) + (EXP_ULP + 2 * N + 4) * U * f64(S) + N * TINY
    return mx, e, S, SAFETY * tau


def exact_draw_check(v, b, u, got):
    """The exact draws (k_bs_on2, warp_exact_draw): for each row k, ``got[k]`` must be a particle of positive weight
    whose cumulative bracket [C[n-1], C[n]] holds u * S within tau; a row of zero weight everywhere must give 0.
    Returns (number of draws whose target lay within tau of a bracket edge, number of all-zero rows)."""
    got = np.asarray(got, dtype=np.int64)
    mx, e, S, tau = row_sums(v, b)
    zero = S == 0
    assert np.all(got[zero] == 0), ("all-zero row", np.flatnonzero(zero & (got != 0))[:8], got[zero][:8])
    k = np.flatnonzero(~zero)
    if k.size == 0:
        return 0, int(zero.sum())
    C = np.cumsum(e[k], axis=1)
    n = got[k]
    assert np.all((n >= 0) & (n < v.shape[1])), "index out of range"
    en = e[k, n]
    assert np.all(en > 0), ("zero-weight particle drawn", k[en == 0][:8], n[en == 0][:8])
    hi = C[np.arange(k.size), n]
    lo = np.where(n > 0, C[np.arange(k.size), np.maximum(n - 1, 0)], LD(0))
    target = LD(1) * np.asarray(u, dtype=np.float64)[k] * S[k]
    t_ = LD(1) * tau[k]
    ok = (target > lo - t_) & (target <= hi + t_)
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, ("draw outside its bracket", k[bad][:8], n[bad][:8], f64(target[bad][:8]),
                           f64(lo[bad][:8]), f64(hi[bad][:8]))
    near = (np.abs(target - lo) <= t_) | (np.abs(target - hi) <= t_)
    return int(near.sum()), int(zero.sum())


# -------------------------------------------------------------------------------------------- MCMC and reject
def accept(lu, lp, blp, shift):
    """The kernels' ``lu < lp - shift`` with its decision margin: (decision, decided).  lp's bound, the fp64
    subtraction and the log of the uniform (1 ulp on either side): 2 roundings of |lu| + |lp - shift|."""
    lu = np.asarray(lu, dtype=np.float64)
    rhs = lp - LD(1) * np.asarray(shift, dtype=np.float64)
    margin = blp + SAFETY * 2 * U * (np.abs(lu) + np.abs(f64(rhs)))
    diff = f64(rhs - lu)
    return diff > 0, np.abs(diff) > margin


def mcmc_step(trans, t, Xt, xn, start, props, lus):
    """Independent Metropolis from ``start`` (M,) towards xn (M, D) at time t (density logpt(t + 1, ...)), with
    proposals props (S, M) and log-uniforms lus (S, M).  Returns (final index, decided mask)."""
    Xt = as_rows(Xt)
    cur = np.array(start, dtype=np.int64)
    lc, bc = trans.lpdf(t + 1, Xt[cur], xn)
    decided = np.ones(cur.shape, dtype=bool)
    for i in range(props.shape[0]):
        lp, bp = trans.lpdf(t + 1, Xt[props[i]], xn)
        acc, sure = accept(lus[i], lp - lc, bp + bc, 0.0)     # lu < lprop - lcur, both densities' bounds
        decided &= sure
        cur = np.where(acc, props[i], cur)
        lc, bc = np.where(acc, lp, lc), np.where(acc, bp, bc)
    return cur, decided


def reject_trials(trans, t_dens, Xp, xn, props, lus, bound):
    """The hybrid sampler's trials of one step: props / lus (K, mt) for K draws targeting xn (K, D); trial k accepts
    when lu < logpt(t_dens, Xp[prop], xn) - bound.  Returns (winning trial or -1, its proposal, decided mask): the
    winner is the first accepted trial in trial order, undecided when a trial up to it lies within its margin."""
    Xp = as_rows(Xp)
    K, mt = props.shape
    if mt == 0:
        return np.full(K, -1), np.zeros(K, dtype=np.int64), np.ones(K, dtype=bool)
    lp, bp = trans.lpdf(t_dens, Xp[props], as_rows(xn)[:, None, :])
    acc, sure = accept(lus, lp, bp, bound)
    first = np.where(acc.any(1), np.argmax(acc, axis=1), -1)
    upto = np.where(first >= 0, first, mt - 1)
    decided = np.array([sure[k, :upto[k] + 1].all() for k in range(K)])
    choice = np.where(first >= 0, props[np.arange(K), np.maximum(first, 0)], 0)
    return first, choice, decided


def device_trials(seed, call, js, t_field, mt, cdf):
    """Proposals and log-uniforms of trials 0..mt-1 drawn by the kernel itself: smooth_uniforms(key, call, j,
    t_field, trial, kPurposeSmooth), the proposal by draw_cdf on ``cdf`` (the caller's CDF bits), lu = log(u1)."""
    js = np.asarray(js, dtype=np.int64)
    trial = np.arange(mt, dtype=np.int64)[None, :]
    u0, u1 = smooth_uniforms(seed, call, js[:, None], t_field, trial, PURPOSE_SMOOTH)
    return draw_cdf(cdf, u0), np.log(u1)


# ------------------------------------------------------------------------------------------- on-line smoothing
def on2_weights_check(trans, t, Xp, lwp, xs, omega):
    """omega[r, i] = exp_and_normalise(lw_{t-1} + logpt(t, X_{t-1}, xs[r])) against long double.  Returns the
    largest error in units of its bound."""
    v, b = row_values(trans, t, Xp, lwp, xs)
    mx, e, S, tau = row_sums(v, b)
    ref = e / S[:, None]
    ef = f64(e)
    # e_n's own bound relative to S, plus S's (tau / S), plus the reciprocal and the product: 2 roundings
    tol = (f64(ref) * (tau / f64(S))[:, None] + SAFETY * ef / f64(S)[:, None]
           * (b + 2 * U * EXP_ULP) + 2 * SAFETY * U * f64(ref) + TINY)
    err = np.abs(f64(LD(1) * omega - ref))
    assert np.all(err <= tol), ("omega", np.unravel_index(np.argmax(err - tol), err.shape), float((err / tol).max()))
    rs_ = f64((LD(1) * omega).sum(1))
    assert np.all(np.abs(rs_ - 1) <= (v.shape[1] + 2) * SAFETY * U + tau / f64(S) * 2)
    return float((err / tol).max())


def phi_on2_check(omega, phi_prev, psi, phi):
    """PHI_ON2: phi[r] = sum_i w[r, i] (phi_prev[i] + psi[r, i]) / sum_i w[r, i], on the kernel's own omega; the
    lane-strided sums: N / 32 + 5 roundings of each partial, 1 of each term and the division."""
    w = LD(1) * omega
    terms = w[:, :, None] * (LD(1) * phi_prev[None, :, :] + psi)
    ref = terms.sum(1) / w.sum(1)[:, None]
    N = omega.shape[1]
    k = N // 32 + 8
    tol = SAFETY * k * U * (f64(np.abs(terms).sum(1)) / f64(w.sum(1))[:, None] + np.abs(f64(ref)))
    err = np.abs(f64(LD(1) * phi - ref))
    assert np.all(err <= tol + TINY), ("phi_on2", float((err / (tol + TINY)).max()))


def phi_paris_check(B, Np, phi_prev, psi, phi):
    """PHI_PARIS: phi[n] = mean_i (phi_prev[B[n Np + i]] + psi[n Np + i]), Np terms in i order then / Np."""
    N = B.shape[0] // Np
    terms = LD(1) * phi_prev[B] + psi
    ref = terms.reshape(N, Np, -1).sum(1) / Np
    tol = SAFETY * (2 * Np + 2) * U * f64(np.abs(terms).reshape(N, Np, -1).sum(1)) / Np
    err = np.abs(f64(LD(1) * phi - ref))
    assert np.all(err <= tol + TINY), ("phi_paris", float((err / (tol + TINY)).max()))


# ---------------------------------------------------------------------------------------------------- two-filter
def on_logw_check(trans, t, X, Xinfo, I, J, mf, mi, log_omega):
    """ON_LOGW: logpt(t + 1, X[J], Xinfo[I]) - mf[J] - mi[I] (forward modifier first), 2 more roundings."""
    X, Xinfo = as_rows(X), as_rows(Xinfo)
    v, b = trans.lpdf(t + 1, X[J], Xinfo[I])
    a = np.abs(f64(v))
    if mf is not None:
        v = v - LD(1) * mf[J]
        a = a + np.abs(mf[J])
    if mi is not None:
        v = v - LD(1) * mi[I]
        a = a + np.abs(mi[I])
    tol = b + SAFETY * 2 * U * a
    err = np.abs(f64(LD(1) * log_omega - v))
    assert np.all(err <= tol), ("log_omega", int(np.argmax(err - tol)), float((err / tol).max()))


def on2_rows_check(trans, t, X, lw, Xinfo, psi, L, S):
    """ON2_ROWS: per row m, L[m] = log sum_n exp(lw[n] + logpt(t + 1, X[n], Xinfo[m])) and S[m] the omega-weighted
    mean of psi[m, :]; a row with no positive weight gives (-inf, 0)."""
    v, b = row_values(trans, t + 1, X, lw, Xinfo)
    mx, e, Ssum, tau = row_sums(v, b)
    zero = Ssum == 0
    assert np.all(np.isneginf(L[zero])) and np.all(S[zero] == 0), "row without positive weight"
    k = ~zero
    Lref = mx[k] + np.log(Ssum[k])
    rel = tau[k] / f64(Ssum[k])
    tolL = rel + SAFETY * 2 * U * np.abs(f64(Lref)) + SAFETY * U
    errL = np.abs(f64(LD(1) * L[k] - Lref))
    assert np.all(errL <= tolL), ("L", float((errL / tolL).max()))
    A = (e[k] * psi[k]).sum(1)
    Sref = A / Ssum[k]
    ef = f64(e[k])
    # each term's bound and exp's, S's own bound (tau, which also covers the max) carried by |S|, the online sums
    aerr = ((ef * np.abs(psi[k]) * (b[k] + 2 * U * EXP_ULP)).sum(1) * SAFETY + tau[k] * np.abs(f64(Sref))
            + SAFETY * (2 * v.shape[1] + 4) * U * (ef * np.abs(psi[k])).sum(1))
    tolS = aerr / f64(Ssum[k]) + SAFETY * U * np.abs(f64(Sref)) + TINY
    errS = np.abs(f64(LD(1) * S[k] - Sref))
    assert np.all(errS <= tolS), ("S", float((errS / tolS).max()))
