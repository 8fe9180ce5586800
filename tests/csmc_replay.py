"""Per-step replay of the conditional SMC kernel (TEST INFRASTRUCTURE): ``k_csmc`` of csrc/smcb_pmcmc.cu, the state
update of ``mcmc.CSMC`` and ``ParticleGibbs``, in NumPy fp64 and ``np.longdouble``.

The kernel keeps every generation (X, lw, A of shape (T, ld) per chain) and its summary rows, so each step t is
replayed from the kernel's own generation t - 1 and each bound covers one step.  ``CsmcReplay.check_chain`` checks:

1. summary row t - 1 (ESS, logLt, rs, log-mean) with ``StepReplay.check_summary``, and the decision of step t
   (``ESS < N ESSrmin`` on the reported ESS, bit for bit; against the long-double ESS unless within 1e-12 of the
   threshold, where it is counted);
2. on a resampling step, every ancestor: a positive-weight index whose bracket of the long-double CDF holds the grid
   point su_k / su_N of the long-double spacings ``cumsum(-log u)`` within a derived bound (``bracket``); away from
   the bound the ancestor is required exactly, within it the draw is counted as undecided.  A spacing uniform of 0
   makes su_N infinite: every grid point is 0 or NaN and the reference's inverse-CDF loop returns 0 for all of them.
   On a non-resampling step A is ``arange``;
3. the particles ``M(t, Xp, z)`` and log-weights ``fix_nan(base + logG(t, Xp, X))``, with the pinned slot x*[t] bit
   for bit, ancestor 0 and weight ``(rs ? 0 : lw[t-1, 0]) + logG(t, x*[t-1], x*[t])`` (``logG(0, -, x*[0])`` at 0);
4. the trajectory: the final index an exact draw on W_{T-1} with ud[T-1]; then either the traced ancestors or, in
   backward mode, an exact draw on ``lw_t + logpt(t + 1, X_t, traj[t + 1])`` with ud[t] (``exact_draw_check``); each
   traj[t] the kernel's own X[t, idx] bit for bit;
5. logLt equal to the last summary row's logLt bit for bit.

``device_noise`` restates the kernel's own draws from the chain's key: the normals of step t (slot 0 consumes its
normal when pinned, so the other slots keep the counters of the bank filter), the N + 1 spacing uniforms and the
trajectory uniform (purpose ``PURPOSE_TRAJ``).
"""
import numpy as np

import philox_ref
from oracle import smc_numpy as orc
from smoothing_replay import EXP_ULP, SAFETY, TINY, U, Trans, exact_draw_check, row_values
from step_replay import LD, StepReplay, fix_nan, lse_stats

PURPOSE_TRAJ = 6                # kPurposeTraj (csrc/smcb_pmcmc.cu)


def device_noise(N, T, key):
    """(z (T, N), u (T, N + 1), ud (T,)) the kernel draws under the Philox key ``key`` (a Python int)."""
    key = int(key) & (2 ** 64 - 1)
    z = np.stack([philox_ref.normals(N, t, key) for t in range(T)])
    u = np.stack([philox_ref.uniforms(N + 1, t, key) for t in range(T)])
    ud = np.array([philox_ref.uniforms(1, t, key, w3=PURPOSE_TRAJ)[0] for t in range(T)])
    return z, u, ud


def counters(N, T):
    """The Philox counters (c0, c1, c2, c3) of each purpose a chain of N particles and T steps uses."""
    npairs = (N + 1) // 2
    sp = (N + 2) // 2
    ts = range(T)
    normals = {(p, 0, t, philox_ref.PURPOSE_NORMAL) for t in ts for p in range(npairs)}
    spacings = {(p, 0, t, philox_ref.PURPOSE_UNIFORM) for t in ts for p in range(sp)}
    traj = {(0, 0, t, PURPOSE_TRAJ) for t in ts}
    return {"normals": normals, "spacings": spacings, "traj": traj}


def chain_objects(tmap, rows, guided, data=None):
    """Per parameter row r of ``tmap`` (a ``bank.ThetaMap``): (the oracle Feynman-Kac object on the chain's data row,
    its ``Trans``).  ``data``: (R, T) per-chain data rows, or None for the map's own row."""
    cols = tmap.columns(rows)
    params = tmap.params(rows)
    sc = tmap.step_consts(rows)
    out = []
    for r in range(params.shape[0]):
        model = getattr(orc, tmap.name)(**{k: float(v[r]) for k, v in cols.items()})
        y = tmap.data if data is None else np.asarray(data[r], dtype=np.float64)
        fk = (orc.GuidedPF if guided else orc.Bootstrap)(model, y)
        # the transition density carries no step constant except Gordon_etal's location term
        spec = {"model": tmap.model, "params": params[r], "dim": 1, "step_consts": None if sc is None else sc[r]}
        out.append((fk, Trans(spec)))
    return out


def oracle_summaries(o):
    """The (T, 4) summary table (ESS, logLt, rs, log-mean) of an oracle run ``o`` (``pmcmc_numpy.CSMC``)."""
    with np.errstate(all="ignore"):
        lm = [orc.Weights(np.array(s["lw"], copy=True)).log_mean for s in o.trace]
    return np.stack([o.ESSs, o.logLts, np.asarray(o.rs_flags, dtype=np.float64), lm], axis=1)


def _same(a, b):
    """Bit equality of fp64 arrays (a NaN equals a NaN with the same bits only)."""
    return np.asarray(a, dtype=np.float64).view(np.uint64) == np.asarray(b, dtype=np.float64).view(np.uint64)


def bracket(lw, g, scale_n):
    """The long-double CDF of exp(lw) and the bound of the kernel's comparison of a grid point g in [0, 1] with its
    fp64 CDF.  The CDF side: exp(lw - m) (the subtraction: u |lw - m|, exp: EXP_ULP), the product by 1 / s and s
    itself (a sum of N terms), the blocked scan: at most 2N + 4 roundings of the running sum.  The grid side: g is a
    ratio of two scanned sums of ``scale_n`` terms -log u (1 ulp each): 2 scale_n + 8 roundings.  Returns (e, S,
    C, tau) with tau in units of S."""
    lw = np.asarray(lw, dtype=np.float64)
    N = lw.shape[0]
    m, S, _, e = lse_stats(lw)
    C = np.cumsum(e)
    with np.errstate(invalid="ignore"):
        sh = np.where(np.isfinite(lw), np.abs(lw - m), 0.0)
    ef = np.asarray(e, dtype=np.float64)
    tau = (SAFETY * U * (float((ef * sh).sum()) + (EXP_ULP + 2 * N + 6) * float(S))
           + SAFETY * U * (2 * scale_n + 8) * float(S) * np.asarray(g, dtype=np.float64) + N * TINY)
    return e, S, C, tau


class CsmcReplay:
    """One kernel configuration: ``fk`` the chain's oracle Feynman-Kac object, ``trans`` its ``smoothing_replay.Trans``
    (backward draws only), ``draw`` 'genealogy' or 'backward'.  Counters: ``n_rs`` resampling steps, ``n_near``
    decisions within 1e-12 of the threshold, ``n_und`` undecided ancestors and trajectory indices, ``n_draws`` all
    ancestors and indices checked, ``n_zero`` trajectory rows with no positive weight, ``n_u0`` steps whose spacings
    hold an infinite term."""

    def __init__(self, N, essrmin, pin, draw, x_rtol=1e-13, x_atol=1e-14, x_exact=False):
        self.N, self.essrmin, self.pin, self.draw = int(N), float(essrmin), bool(pin), draw
        self.tol = dict(x_rtol=x_rtol, x_atol=x_atol, x_exact=x_exact)
        self.n_rs = self.n_near = self.n_und = self.n_draws = self.n_zero = self.n_u0 = 0

    # ---------------------------------------------------------------- ancestors
    def check_ancestors(self, t, lw_prev, u, A):
        N, k0 = self.N, int(self.pin)
        A = np.asarray(A, dtype=np.int64)
        assert np.all((A >= 0) & (A < N)), f"step {t}: ancestor out of range"
        with np.errstate(divide="ignore"):
            su = np.cumsum(-np.log(np.asarray(u, dtype=np.float64)[:N + 1].astype(LD)))
        if not np.isfinite(su[-1]):
            # the reference's inverse_cdf loop: every grid point is 0 (before the zero) or NaN (after), A = 0
            self.n_u0 += 1
            assert np.all(A == 0), f"step {t}: a zero spacing uniform, ancestors {A[A != 0][:8]} (all must be 0)"
            return
        g = su[:N] / su[N]
        e, S, C, tau = bracket(lw_prev, g, N + 1)
        assert S > 0, f"step {t}: resampling from weights that are all zero"
        target = g * S
        hi = C[A]
        lo = np.where(A > 0, C[np.maximum(A - 1, 0)], LD(0))
        pos = e[A] > 0
        t_ = LD(1) * tau
        # the clamp: a grid point above the kernel's last CDF entry takes N - 1, as the reference's does
        clamp = (A == N - 1) & (target > C[-1] - t_)
        ok = (pos & (target > lo - t_) & (target <= hi + t_)) | clamp
        ok[:k0] = True                                   # the pinned slot's ancestor is 0, checked by the caller
        if not ok.all():
            k = int(np.flatnonzero(~ok)[0])
            j = int(min(np.searchsorted(C, target[k], side="left"), N - 1))
            raise AssertionError(f"step {t}: ancestor {A[k]} of output {k} (weight {float(e[A[k]] / S)!r}) does not hold "
                                 f"su {float(g[k])!r}; the long-double search gives {j} "
                                 f"({int((~ok).sum())} of {N} outputs)")
        near = (np.abs(target - lo) <= t_) | (np.abs(target - hi) <= t_) | clamp
        self.n_und += int(near[k0:].sum())
        self.n_draws += N - k0

    # ---------------------------------------------------------------- one chain
    def check_chain(self, fk, X, lw, A, summ, logLt, z, u, xstar=None, traj=None, ud=None, trans=None):
        """X, lw, A (T, N) of one chain (host copies without padding), summ (T, 4), logLt (scalar), z (T, N) and
        u (T, N + 1) the step noise, xstar (T,) the pinned path, traj (T,) and ud (T,) the trajectory and its
        uniforms.  Returns the indices of the trajectory."""
        N, T = self.N, X.shape[0]
        rep = StepReplay(fk, N, "multinomial", self.essrmin, **self.tol)
        pin = self.pin
        # step 0
        with np.errstate(all="ignore"):
            Xr = fk.M0(N, z[0])
        if pin:
            assert _same(X[0, 0], xstar[0]), f"step 0: pinned particle {X[0, 0]!r} vs x* {xstar[0]!r}"
            Xr = np.array(Xr, copy=True)
            Xr[0] = X[0, 0]
        rep._check_x(0, X[0], Xr)
        with np.errstate(all="ignore"):
            lr = fix_nan(fk.logG(0, None, X[0]))
        rep._close(0, "lw", lw[0], lr, 1e-12, 1e-12)
        thr = N * self.essrmin
        for t in range(1, T):
            rep.check_summary(t - 1, X[t - 1], lw[t - 1], summ)
            rs = bool(summ[t, 2] != 0)
            assert rs == bool(summ[t - 1, 0] < thr), \
                f"step {t}: rs {rs} but reported ESS {summ[t - 1, 0]!r}, N ESSrmin {thr}"
            with np.errstate(invalid="ignore"):
                _, S, Q, _ = lse_stats(lw[t - 1])
                ess = float(S * S / Q)
            if abs(ess - thr) <= 1e-12 * thr:
                self.n_near += 1
            else:
                assert rs == (ess < thr), f"step {t}: rs {rs} but the long-double ESS is {ess!r}, N ESSrmin {thr}"
            if rs:
                self.n_rs += 1
                self.check_ancestors(t, lw[t - 1], u[t], A[t])
                Xp, base = X[t - 1][A[t]], np.zeros(N)
            else:
                if not np.array_equal(A[t], np.arange(N)):
                    k = int(np.flatnonzero(A[t] != np.arange(N))[0])
                    raise AssertionError(f"step {t}: no resampling but A[{k}] = {A[t, k]}")
                Xp, base = X[t - 1], lw[t - 1]
            if pin:
                assert A[t, 0] == 0, f"step {t}: pinned ancestor {A[t, 0]}"
                assert _same(X[t, 0], xstar[t]), f"step {t}: pinned particle {X[t, 0]!r} vs x* {xstar[t]!r}"
            with np.errstate(all="ignore"):
                Xr = np.array(fk.M(t, Xp, z[t]), copy=True)
                if pin:
                    Xr[0] = X[t, 0]
                rep._check_x(t, X[t], Xr)
                lr = fix_nan(base + fk.logG(t, Xp, X[t]))
                if pin:
                    b0 = 0.0 if rs else lw[t - 1, 0]
                    lr[0] = fix_nan(b0 + fk.logG(t, xstar[t - 1:t], xstar[t:t + 1]))[0]
            rep._close(t, "lw", lw[t], lr, 1e-12, 1e-12)
        rep.check_last(T, X[T - 1], lw[T - 1], summ)
        assert _same(logLt, summ[T - 1, 1]), f"logLt {logLt!r} vs the last summary row {summ[T - 1, 1]!r}"
        if traj is None:
            return None
        return self.check_traj(X, lw, A, traj, ud, trans)

    # ---------------------------------------------------------------- trajectory
    def _draw(self, t, v, b, u, cands):
        """The exact draw of one row: one of the candidate indices (those whose particle has the trajectory's bits)
        must pass ``exact_draw_check``; u = 0 searches for 0 in a non-decreasing CDF and takes index 0, as the
        reference does.  Returns the index."""
        if u == 0:
            assert 0 in cands, f"trajectory at step {t}: u = 0 but the drawn particle is not X[{t}, 0]"
            self.n_draws += 1
            return 0
        err = None
        for c in cands:
            try:
                near, zero = exact_draw_check(v[None, :], b[None, :], np.array([u]), np.array([c]))
            except AssertionError as ex:
                err = ex
                continue
            self.n_und += near
            self.n_zero += zero
            self.n_draws += 1
            return int(c)
        raise AssertionError(f"trajectory at step {t}: no index with the drawn particle's bits passes its draw "
                             f"(candidates {list(cands)[:8]}): {err}")

    def check_traj(self, X, lw, A, traj, ud, trans):
        N, T = self.N, X.shape[0]
        idx = np.empty(T, dtype=np.int64)

        def cands(t):
            c = np.flatnonzero(_same(X[t], traj[t]))
            assert c.size, f"trajectory at step {t}: {traj[t]!r} is not a particle of generation {t}"
            return c

        # the final index: multinomial_once on W_{T-1} (the kernel compares u with its CDF normalised by its sum)
        last = np.asarray(lw[T - 1], dtype=np.float64)
        with np.errstate(invalid="ignore"):
            m = last.max()
            b = np.where(np.isfinite(last), U * np.abs(last - m), 0.0) if np.isfinite(m) else np.zeros(N)
        idx[T - 1] = self._draw(T - 1, LD(1) * last, b, ud[T - 1], cands(T - 1))
        for t in range(T - 2, -1, -1):
            if self.draw == "genealogy":
                n = int(A[t + 1, idx[t + 1]])
                assert _same(X[t, n], traj[t]), f"trajectory at step {t}: {traj[t]!r} vs X[{t}, {n}] {X[t, n]!r}"
                idx[t] = n
            else:
                v, b = row_values(trans, t + 1, X[t], lw[t], np.array([traj[t + 1]]))
                idx[t] = self._draw(t, v[0], b[0], ud[t], cands(t))
        return idx
