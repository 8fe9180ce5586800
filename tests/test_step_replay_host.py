"""The per-step replay (tests/step_replay.py) checked without a GPU: fed the NumPy oracle's own state after every step
of ``orc.SMC`` with injected noise, it must predict the oracle's next step -- the decision, the ancestors and the
particles bit for bit, the log-weights to the replay's tolerance -- and accept every summary row."""
import numpy as np
import pytest

from oracle import smc_numpy as orc
from step_replay import StepReplay


def lst(y):
    return [np.atleast_1d(v) for v in y]


def models(golden):
    return {
        "sv": (orc.StochVol(), lst(golden["data/sv_seed1_T1000"][:25])),
        "lg": (orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), lst(golden["data/lg_seed2_T100"][:25])),
        "cox": (orc.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), lst(golden["data/cox_seed6_T60"][:25])),
        "mvlg": (orc.MVLinearGauss_Guarniero_etal(0.4, 4), list(golden["data/mvlg_seed5_T30"][:25])),
        "bearings": (orc.BearingsOnly(), list(golden["data/bearings_seed0_T40"].reshape(-1, 1)[:25])),
    }


CASES = [("sv", "Bootstrap", "systematic", 0.5), ("sv", "GuidedPF", "stratified", 0.8),
         ("sv", "AuxiliaryPF", "multinomial", 0.5), ("sv", "AuxiliaryBootstrap", "systematic", 1.0),
         ("lg", "Bootstrap", "multinomial", 1.0), ("lg", "AuxiliaryPF", "stratified", 0.5),
         ("cox", "Bootstrap", "stratified", 0.5), ("mvlg", "GuidedPF", "systematic", 0.5),
         ("mvlg", "AuxiliaryPF", "multinomial", 0.7), ("bearings", "Bootstrap", "stratified", 0.5)]


@pytest.mark.parametrize("N", [1, 2, 257, 600])
@pytest.mark.parametrize("mname,fkname,scheme,essrmin", CASES)
def test_replay_predicts_oracle(golden, mname, fkname, scheme, essrmin, N):
    model, y = models(golden)[mname]
    T = len(y)
    fk = getattr(orc, fkname)(model, y)
    nz = {"mvlg": 4, "bearings": 2}.get(mname)
    r = np.random.RandomState(N)
    z = r.standard_normal((T, N) if nz is None else (T, N, nz))
    u = r.rand(T, N + 1)
    nu = {"systematic": 1, "stratified": N, "multinomial": N + 1}[scheme]
    ref = orc.SMC(fk, N=N, resampling=scheme, ESSrmin=essrmin, noise=orc.InjectedNoise(z, [row[:nu] for row in u]))
    rep = StepReplay(fk, N, scheme, essrmin, x_exact=True)
    summ = np.zeros((T, 4))
    prev = None
    with np.errstate(all="ignore"):
        for t in range(T):
            ref.step()
            summ[t] = [ref.wgts.ESS, ref.logLt, float(ref.rs_flag), ref.log_mean_w]
            X, lw = ref.X, ref.wgts.lw.copy()
            if t == 0:
                Xr, lr = rep.check_init(z[0], X, lw)
                assert np.array_equal(Xr, X) and np.array_equal(lr, lw)
            else:
                cdf = np.cumsum(ref.aux.W) if ref.rs_flag else None
                scratch = np.cumsum(-np.log(u[t])) if ref.rs_flag and scheme == "multinomial" else None
                out = rep.check_step(t, prev[0], prev[1], summ, z[t], u[t][:nu], X, lw,
                                     A=ref.A if ref.rs_flag else None, cdf=cdf, scratch=scratch)
                assert out["rs"] == ref.rs_flag
                assert np.array_equal(out["X"], X), t
                np.testing.assert_allclose(out["lw"], lw, rtol=1e-13, atol=1e-13)
                if ref.rs_flag:
                    assert out["counts"].sum() == N
            prev = (X, lw)
        rep.check_last(T, prev[0], prev[1], summ)
    assert rep.n_rs == sum(ref.rs_flags) and (N < 3 or rep.n_rs > 0)


def test_replay_rejects_a_wrong_step(golden):
    """The replay is sharp: one ancestor moved by one entry, one particle off by an ulp, a flipped decision and a CDF
    one ulp too short at its end are each reported."""
    model, y = models(golden)["sv"]
    N, T = 300, 6
    fk = orc.Bootstrap(model, y[:T])
    r = np.random.RandomState(0)
    z, u = r.standard_normal((T, N)), r.rand(T, N + 1)
    ref = orc.SMC(fk, N=N, ESSrmin=1.0, noise=orc.InjectedNoise(z, [row[:1] for row in u]))
    ref.step()
    X0, lw0 = ref.X, ref.wgts.lw.copy()
    summ = np.zeros((T, 4))
    summ[0] = [ref.wgts.ESS, ref.logLt, 0.0, ref.log_mean_w]
    ref.step()
    summ[1] = [ref.wgts.ESS, ref.logLt, 1.0, ref.log_mean_w]
    cdf = np.cumsum(ref.aux.W)
    rep = StepReplay(fk, N, "systematic", 1.0, x_exact=True)
    args = (1, X0, lw0, summ, z[1], u[1][:1])
    rep.check_step(*args, ref.X, ref.wgts.lw, A=ref.A, cdf=cdf)
    k = int(np.flatnonzero(np.diff(ref.A) > 0)[0])
    A = ref.A.copy()
    A[k] = A[k + 1]
    with pytest.raises(AssertionError, match="ancestor"):
        rep.check_step(*args, ref.X, ref.wgts.lw, A=A, cdf=cdf)
    X = ref.X.copy()
    X[7] = np.nextafter(X[7], np.inf)
    with pytest.raises(AssertionError, match="bit-identical"):
        rep.check_step(*args, X, ref.wgts.lw, A=ref.A, cdf=cdf)
    s2 = summ.copy()
    s2[1, 2] = 0.0
    with pytest.raises(AssertionError, match="rs"):
        rep.check_step(1, X0, lw0, s2, z[1], u[1][:1], ref.X, ref.wgts.lw, A=ref.A, cdf=cdf)
    c2 = cdf.copy()
    c2[-1] = 1.0 - 1e-12
    with pytest.raises(AssertionError, match="CDF"):
        rep.check_step(*args, ref.X, ref.wgts.lw, A=ref.A, cdf=c2)
