"""NumPy restatement of the reference's IBIS sampler (particles/smc_samplers.py:772-794) over the logistic-regression
model, with the FKSMCsampler resampling rule and the random-walk moves of oracle/samplers_numpy.py.  Random numbers
come from the legacy global ``numpy.random`` stream in the reference's order, so a run after the same
``np.random.seed`` reproduces the reference's run (tests/golden/golden_ibis.npz)."""
import numpy as np

from oracle import smc_numpy as orc
from oracle.samplers_numpy import AdaptiveTemperingWF, LogisticModel, ThetaParticles


class IBISSampler:
    """IBIS (smc_samplers.py:772-794) over ``model`` (``logpyt(theta, t)`` on the (N, d) array, ``prior``), with the
    FKSMCsampler resampling rule (740-745), the random-walk calibration (617-622) and the waste-free
    (MCMCSequenceWF, 672-683) or standard (AdaptiveMCMCSequence, 686-709, fixed length) move.  Particles carry
    theta and lpost only, as the reference's do."""

    def __init__(self, model, wastefree=True, len_chain=10):
        self.model, self.wastefree, self.len_chain = model, wastefree, len_chain
        self.tempering = AdaptiveTemperingWF(model, len_chain)     # calibrate / mh_step

    def loglik(self, theta, t):                              # StaticModel.loglik, 263-284
        ll = np.zeros(theta.shape[0])
        for s in range(t + 1):
            ll += self.model.logpyt(theta, s)
        np.nan_to_num(ll, copy=False, nan=-np.inf)
        return ll

    def target(self, t):                                     # IBIS.current_target, 778-782
        def func(x):
            x.lpost = self.model.prior.logpdf(x.theta) + self.loglik(x.theta, t)
        return func

    def M0(self, N):                                         # 767-769, 784-787
        x0 = ThetaParticles(theta=self.model.prior.rvs(N * self.len_chain if self.wastefree else N))
        self.target(-1)(x0)
        return x0

    def move(self, x, target):
        mh = self.tempering.mh_step
        if self.wastefree:
            return self.tempering.move(x, target)
        xout = x.copy()
        for _ in range(self.len_chain - 1):
            mh(xout, target)
        return xout

    def logG(self, t, x):                                    # 773-776
        lpyt = self.model.logpyt(x.theta, t)
        x.lpost = x.lpost + lpyt
        return lpyt


def run_ibis(model, N, wastefree=True, len_chain=10, ESSrmin=0.5, resampling="systematic"):
    """particles.SMC(fk=IBIS(model, wastefree, len_chain), N=N, ESSrmin=ESSrmin).run(): the loop of core.py:369-383
    and the summaries of 351-367 (ESSs, logLts, rs_flags)."""
    fk = IBISSampler(model, wastefree, len_chain)
    out = {"ESSs": [], "logLts": [], "rs_flags": []}
    X = fk.M0(N)
    wgts = orc.Weights().add(fk.logG(0, X))
    lmw = wgts.log_mean
    logLt = lmw
    out["ESSs"].append(wgts.ESS), out["logLts"].append(logLt), out["rs_flags"].append(False)
    for t in range(1, model.T):
        rs_flag = wgts.ESS < X.N * ESSrmin
        if rs_flag:
            fk.tempering.calibrate(wgts.W, X)
            A = orc.resampling(resampling, wgts.W, M=N)
            X = fk.move(X[A], fk.target(t - 1))
            wgts = orc.Weights()
        wgts = wgts.add(fk.logG(t, X))
        prec, lmw = lmw, wgts.log_mean
        logLt += lmw if rs_flag else lmw - prec
        out["ESSs"].append(wgts.ESS), out["logLts"].append(logLt), out["rs_flags"].append(bool(rs_flag))
    out.update(logLt=logLt, X=X, W=wgts.W)
    return out


class LogisticIBISModel(LogisticModel):
    """LogisticModel with the per-row factor IBIS reweights by (book/smc_samplers/logistic_reg.py:63-67)."""

    def logpyt(self, theta, t):
        return -np.logaddexp(0.0, -np.matmul(theta, self.data[t, :]))
