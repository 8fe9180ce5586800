"""NumPy restatement of the reference's nested sampling SMC (particles/nested.py:281-373) over the logistic-regression
model, with the calibration and Metropolis steps of oracle/samplers_numpy.py.  Random numbers come from the legacy
global ``numpy.random`` stream in the reference's order, so a run after the same ``np.random.seed`` reproduces the
reference's run (tests/golden/golden_nested.npz)."""
import numpy as np
from scipy import special

from oracle import smc_numpy as orc
from oracle.samplers_numpy import AdaptiveTemperingWF, ThetaParticles


def log_sum_exp_ab(a, b):                                    # resampling.py:273-288
    if a > b:
        return a + np.log1p(np.exp(b - a))
    return b + np.log1p(np.exp(a - b))


class NestedSampler:
    """NestedSamplingSMC (nested.py:281-373) over ``model`` (``loglik``, ``prior``), with the random-walk
    calibration (smc_samplers.py:617-622) and the waste-free (MCMCSequenceWF, 672-683) or standard
    (AdaptiveMCMCSequence, 686-709, fixed length) move."""

    def __init__(self, model, wastefree=True, len_chain=10, ESSrmin=0.1, eps=0.01):
        self.model, self.wastefree, self.len_chain = model, wastefree, len_chain
        self.ESSrmin, self.eps = ESSrmin, eps
        self.tempering = AdaptiveTemperingWF(model, len_chain)     # calibrate / mh_step / waste-free move

    def target(self, lt):                                    # current_target, 353-363
        def func(x):
            x.lprior = self.model.prior.logpdf(x.theta)
            x.llik = self.model.loglik(x.theta)
            if lt == -np.inf:
                x.lpost = x.lprior.copy()
            else:
                x.lpost = np.where(x.llik >= lt, x.lprior, -np.inf)
        return func

    def M0(self, N):                                         # 365-370
        x0 = ThetaParticles(theta=self.model.prior.rvs(N * self.len_chain if self.wastefree else N))
        x0.shared["lts"] = [-np.inf]
        x0.shared["log_evid"] = [-np.inf]
        self.target(-np.inf)(x0)
        return x0

    def move(self, x, target):
        if self.wastefree:
            return self.tempering.move(x, target)
        xout = x.copy()
        for _ in range(self.len_chain - 1):
            self.tempering.mh_step(xout, target)
        return xout

    def logG(self, t, x):                                    # 330-351
        curr_evid = x.shared["log_evid"][-1]
        lt = np.percentile(x.llik, 100.0 * (1.0 - self.ESSrmin))
        lZt = t * np.log(self.ESSrmin) - np.log(x.N) + special.logsumexp(x.llik[x.llik <= lt])
        new_evid = log_sum_exp_ab(curr_evid, lZt)
        lZt_final = t * np.log(self.ESSrmin) - np.log(x.N) + special.logsumexp(x.llik)
        new_evid_final = log_sum_exp_ab(curr_evid, lZt_final)
        if np.abs(new_evid - new_evid_final) < self.eps:
            lt = np.inf
            lw = np.zeros_like(x.llik)
            new_evid = new_evid_final
        else:
            lw = np.where(x.llik > lt, 0.0, -np.inf)
        x.shared["lts"].append(lt)
        x.shared["log_evid"].append(new_evid)
        return lw


def run_nested(model, N, wastefree=True, len_chain=10, ESSrmin=0.1, eps=0.01, resampling="systematic"):
    """particles.SMC(fk=NestedSamplingSMC(model, wastefree, len_chain, ESSrmin=ESSrmin, eps=eps), N=N).run(): the loop
    of core.py:369-383, resampling N of the particles at every step (nested.py:315-317) until lts[-1] == inf."""
    fk = NestedSampler(model, wastefree, len_chain, ESSrmin, eps)
    X = fk.M0(N)
    wgts = orc.Weights().add(fk.logG(0, X))
    t = 1
    while X.shared["lts"][-1] != np.inf:
        fk.tempering.calibrate(wgts.W, X)
        A = orc.resampling(resampling, wgts.W, M=N)
        Xp = X[A]
        X = fk.move(Xp, fk.target(Xp.shared["lts"][-1]))
        wgts = orc.Weights().add(fk.logG(t, X))
        t += 1
    return {"lts": list(X.shared["lts"]), "log_evid": list(X.shared["log_evid"]), "X": X, "W": wgts.W, "t": t}
