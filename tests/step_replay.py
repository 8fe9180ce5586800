"""Per-step replay of the fused filter (TEST INFRASTRUCTURE).

``StepReplay.check_step`` takes the state a filter left after step t - 1 (its particles and log-weights and its
summary table), the noise of step t and the outputs of step t, and checks step t against plain NumPy in fp64 and
``np.longdouble``, using the Feynman-Kac objects of ``oracle/smc_numpy.py`` (``M0, M, logG, logeta``):

1. the summaries of step t - 1 (log-mean, ESS, logLt), recomputed from the filter's own log-weights with a
   long-double max-shifted sum, and the resampling decision of step t (``ESS_aux < N * ESSrmin``);
2. on a resampling step, the filter's CDF: non-decreasing, last entry 1, and equal to the long-double cumulative sum
   of the normalised (auxiliary) weights;
3. the ancestors, bit for bit: ``minimum(searchsorted(cdf, su, 'left'), N - 1)`` on the filter's own CDF, with the
   grid points ``su`` formed by the reference's IEEE expressions (multinomial: the filter's spacings, themselves held
   to a long-double ``cumsum(-log u)``);
4. every ancestor drawn by a positive grid point has a positive weight;
5. the particles ``M(t, Xp, z)`` with ``Xp = X_{t-1}[A]`` (or ``X_{t-1}``), and the log-weights ``base + logG`` from
   the filter's own particles.

Every prediction starts from the filter's own state, so each tolerance covers one step: errors do not accumulate
over T, and the two sides cannot drift apart at a tie.  The checks raise ``AssertionError`` with the first step,
output index and CTA range where the two disagree.
"""
import numpy as np

from oracle import smc_numpy as orc

LD = np.longdouble
EPS = np.finfo(np.float64).eps


def fix_nan(v):
    v = np.array(v, dtype=np.float64, copy=True)
    v[np.isnan(v)] = -np.inf                    # Weights.__init__, resampling.py:220
    return v


def lse_stats(v):
    """(max, sum exp(v - max), sum exp(v - max)^2, exp(v - max)) of fp64 log-weights, the sums in long double."""
    v = np.asarray(v, dtype=np.float64)
    m = v.max()
    e = np.exp(v.astype(LD) - LD(m))
    return m, e.sum(), (e * e).sum(), e


def step_grid(N, n_sm):
    """(CTAs, pairs per CTA) of the fused step kernel for N particles on a device with n_sm SMs: one CTA per SM, at
    most 256, at least one pair per thread of a 512-thread CTA, contiguous ranges of pairs (smcb_filter.cu)."""
    npairs = (N + 1) // 2
    g = max(1, min(n_sm, 256, -(-npairs // 512)))
    chunk = -(-npairs // g)
    return -(-npairs // chunk), chunk


class StepReplay:
    """One fused filter's step-by-step reference.  ``fk``: an oracle Feynman-Kac object; ``chunk``: pairs of
    particles per CTA of the kernel under test (only used to name the CTA in a failure message)."""

    def __init__(self, fk, N, scheme, essrmin, chunk=None, x_rtol=1e-13, x_atol=1e-14, x_exact=False):
        self.fk, self.N, self.scheme, self.essrmin = fk, int(N), scheme, float(essrmin)
        self.chunk = chunk
        self.x_rtol, self.x_atol, self.x_exact = x_rtol, x_atol, x_exact
        self.apf = bool(getattr(fk, "isAPF", False))
        self.n_rs = 0                # resampling steps checked
        self.n_near = 0              # decisions skipped: the ESS within 1e-12 of the threshold

    # ---------------------------------------------------------------- helpers
    def _where(self, k):
        if self.chunk is None:
            return f"output {k}"
        return f"output {k} (CTA {(k // 2) // self.chunk}, pairs [{((k // 2) // self.chunk) * self.chunk}, " \
               f"{((k // 2) // self.chunk + 1) * self.chunk}))"

    def _close(self, t, what, got, want, rtol, atol):
        got, want = np.asarray(got), np.asarray(want)
        assert got.shape == want.shape, (t, what, got.shape, want.shape)
        same_inf = (got == want) | (np.isnan(got) & np.isnan(want))
        bad = ~same_inf & ~(np.abs(got - want) <= atol + rtol * np.abs(want))
        if bad.any():
            k = int(np.flatnonzero(bad.reshape(bad.shape[0], -1).any(axis=1))[0]) if bad.ndim else 0
            raise AssertionError(f"step {t}: {what} differs first at {self._where(k)}: {got[k]!r} vs {want[k]!r} "
                                 f"({int(bad.reshape(bad.shape[0], -1).any(axis=1).sum())} of {len(got)})")

    def _aux(self, t, X, lw):
        """Auxiliary log-weights of the resampling at step t + 1 and logeta_t(X) (None unless an APF)."""
        if not self.apf:
            return lw, None
        with np.errstate(all="ignore"):
            eta = np.asarray(self.fk.logeta(t, X), dtype=np.float64)
            return fix_nan(lw + eta), eta

    # -------------------------------------------------------------- summaries
    def check_summary(self, s, X, lw, summ):
        """Row s of the summary table (ESS, logLt, rs, log-mean) against the filter's log-weights of step s.  Weights
        that are all -inf give NaN for all three, as NumPy does (and every later logLt is NaN)."""
        with np.errstate(invalid="ignore"):
            m, S, Q, _ = lse_stats(lw)
            lm = float(LD(m) + np.log(S / LD(self.N)))
            ess = float(S * S / Q)
        row = summ[s]

        def near(got, want, tol):
            return (np.isnan(got) and np.isnan(want)) or abs(got - want) <= tol

        assert near(row[3], lm, 1e-12 * (1 + abs(lm))), f"step {s}: log-mean {row[3]!r} vs {lm!r}"
        assert near(row[0], ess, 1e-12 * ess), f"step {s}: ESS {row[0]!r} vs {ess!r}"
        loglt = lm if (s == 0 or row[2] != 0) else lm - summ[s - 1, 3]
        logLt = (0.0 if s == 0 else summ[s - 1, 1]) + loglt
        assert near(row[1], logLt, 1e-12 * (1 + abs(logLt))), f"step {s}: logLt {row[1]!r} vs {logLt!r}"
        return lm, ess

    # ---------------------------------------------------------------- step 0
    def check_init(self, z, X, lw, summ=None):
        """Step 0: X = M0(N, z), lw = logG(0, None, X)."""
        with np.errstate(all="ignore"):
            Xr = self.fk.M0(self.N, z)
        self._check_x(0, X, Xr)
        with np.errstate(all="ignore"):
            lr = fix_nan(self.fk.logG(0, None, X))
        self._close(0, "lw", lw, lr, 1e-12, 1e-12)
        return Xr, lr

    def _check_x(self, t, X, Xr):
        if self.x_exact:
            bad = ~((X == Xr) | (np.isnan(X) & np.isnan(Xr)))
            if bad.any():
                k = int(np.flatnonzero(bad.reshape(bad.shape[0], -1).any(axis=1))[0])
                raise AssertionError(f"step {t}: X not bit-identical first at {self._where(k)}: {X[k]!r} vs {Xr[k]!r}")
        else:
            self._close(t, "X", X, Xr, self.x_rtol, self.x_atol)

    # ---------------------------------------------------------------- step t
    def grid_points(self, u, scratch=None):
        """su_k of the reference (resampling.py:602 / 609; multinomial: the filter's own spacings z, z[k] / z[N])."""
        N = self.N
        if self.scheme == "systematic":
            return (np.float64(np.asarray(u).reshape(-1)[0]) + np.arange(N)) / N
        if self.scheme == "stratified":
            return (np.asarray(u, dtype=np.float64)[:N] + np.arange(N)) / N
        return scratch[:N] / scratch[N]

    def check_step(self, t, X_prev, lw_prev, summ, z, u, X, lw, A=None, cdf=None, scratch=None):
        """Step t >= 1 from the filter's state after step t - 1.  ``summ``: the summary table with rows 0..t; ``z``:
        the normals of step t in the oracle's layout; ``u``: the uniforms of step t as the reference consumes them;
        ``A``, ``cdf``, ``scratch`` (multinomial spacings, N + 1): the filter's buffers, read on resampling steps.
        Returns a dict of what the step did (``rs``, and on resampling steps the offspring counts)."""
        N = self.N
        self.check_summary(t - 1, X_prev, lw_prev, summ)
        aux, eta = self._aux(t - 1, X_prev, lw_prev)
        ma, Sa, Qa, ea = lse_stats(aux)
        ess_aux = float(Sa * Sa / Qa)
        thr = N * self.essrmin
        rs = bool(summ[t, 2] != 0)
        if not self.apf:           # the decision on the filter's own reported ESS, bit for bit
            assert rs == bool(summ[t - 1, 0] < thr), f"step {t}: rs {rs} but reported ESS {summ[t - 1, 0]!r}, N ESSrmin {thr}"
        if abs(ess_aux - thr) <= 1e-12 * thr:
            self.n_near += 1
        else:
            assert rs == (ess_aux < thr), f"step {t}: rs {rs} but ESS_aux {ess_aux!r}, N ESSrmin {thr}"
        out = {"rs": rs}
        if rs:
            self.n_rs += 1
            W = ea / Sa                                          # long double, normalised
            assert cdf is not None and A is not None
            assert np.all(np.diff(cdf) >= 0), f"step {t}: CDF decreases at {int(np.flatnonzero(np.diff(cdf) < 0)[0])}"
            assert abs(cdf[-1] - 1.0) <= 1e-13, f"step {t}: CDF ends at {cdf[-1]!r}"
            # |lw - max| is rounded once on each side before the exponential: allowed for on top of 1e-13
            with np.errstate(invalid="ignore"):
                slack = np.cumsum(W * (1 + np.abs(np.where(np.isfinite(aux), aux - ma, 0.0)))) * (8 * EPS)
            dev = np.abs(cdf - np.cumsum(W))
            bad = dev > 1e-13 + slack
            if bad.any():
                k = int(np.flatnonzero(bad)[0])
                raise AssertionError(f"step {t}: CDF off by {float(dev[k]):.3e} first at {self._where(k)}")
            if self.scheme == "multinomial":
                zref = np.cumsum(-np.log(np.asarray(u, dtype=np.float64)[:N + 1].astype(LD)))
                self._close(t, "multinomial spacings", scratch[:N + 1], zref.astype(np.float64), 1e-12, 0.0)
            su = self.grid_points(u, scratch)
            pos = np.searchsorted(cdf, su, side="left")
            Aref = np.minimum(pos, N - 1)
            if not np.array_equal(A, Aref):
                k = int(np.flatnonzero(A != Aref)[0])
                raise AssertionError(f"step {t}: ancestor {A[k]} vs searchsorted {Aref[k]} first at {self._where(k)} "
                                     f"(su {su[k]!r}; {int((A != Aref).sum())} of {N} differ)")
            W64 = np.exp(aux - ma) / float(Sa)
            drawn = (su > 0) & (pos < N)
            zero = drawn & ~(W64[A] > 0)
            assert not zero.any(), f"step {t}: {self._where(int(np.flatnonzero(zero)[0]))} draws a zero-weight entry"
            Xp = X_prev[A]
            if self.apf:                                       # core.py:302: log_mean_exp(logetat, W) - logetat[A]
                m, S, _, _ = lse_stats(lw_prev)
                reset_c = float((LD(ma) + np.log(Sa)) - (LD(m) + np.log(S)))
                base = reset_c - eta[A]
            else:
                base = np.zeros(N)
            out["counts"] = np.bincount(A, minlength=N)
        else:
            Xp, base = X_prev, lw_prev
        with np.errstate(all="ignore"):
            Xr = self.fk.M(t, Xp, z)
        self._check_x(t, X, Xr)
        with np.errstate(all="ignore"):
            lr = fix_nan(base + self.fk.logG(t, Xp, X))
        self._close(t, "lw", lw, lr, 1e-12, 1e-12)
        out["X"], out["lw"] = Xr, lr
        return out

    def check_last(self, T, X, lw, summ):
        """The summary row of the last step, which no later step checks."""
        return self.check_summary(T - 1, X, lw, summ)
