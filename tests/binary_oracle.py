"""NumPy restatement of the reference's SMC samplers on binary spaces (particles/binary_smc.py): chol_and_friends,
the loglik of BIC / BayesianVS / BayesianVS_gprior, NestedLogistic.predict_prob / rvs / logpdf / fit,
BinaryMetropolis.proposal and waste-free adaptive tempering with that move.  Random numbers come from the legacy
global ``numpy.random`` stream in the reference's order, or from injected uniforms in the device's ``noise=`` layout;
every draw returns the uniforms it consumed in that layout."""
import numpy as np
import scipy.linalg
from scipy.special import expit, logit

from oracle.samplers_numpy import AdaptiveTemperingWF, ThetaParticles, run_tempering


def log_no_warn(x):                                           # binary_smc.py:62-64
    return np.log(np.clip(x, 1e-300, None))


def chol_and_friends(gamma, xtx, xty, vm2):                   # binary_smc.py:165-180
    N, d = gamma.shape
    len_gam = np.sum(gamma, axis=1)
    ldet, wtw = np.zeros(N), np.zeros(N)
    for n in range(N):
        if len_gam[n] > 0:
            gam = gamma[n, :]
            xtxg = xtx[:, gam][gam, :] + vm2 * np.eye(len_gam[n])
            C = scipy.linalg.cholesky(xtxg, lower=True, overwrite_a=True, check_finite=False)
            w = scipy.linalg.solve_triangular(C, xty[gam], lower=True, check_finite=False)
            ldet[n] = np.sum(np.log(np.diag(C)))
            wtw[n] = w.T @ w
    return len_gam, ldet, wtw


class IIDBernoulli:
    """distributions.IID(binary_smc.Bernoulli(q), p): rvs draws p x N uniforms coordinate by coordinate."""

    def __init__(self, q, p):
        self.q, self.p = q, p

    def rvs(self, size):
        return np.stack([np.random.rand(size) < self.q for _ in range(self.p)], axis=1)

    def logpdf(self, x):
        return sum([np.where(x[..., i], log_no_warn(self.q), log_no_warn(1.0 - self.q)) for i in range(self.p)])


class VS:
    """VariableSelection and its three models (binary_smc.py:183-293): kind in {"bic", "bvs", "gprior"}."""

    def __init__(self, kind, x, y, prior=None, nu=4.0, lamb=None, iv2=None, g=None, bic_lamb=10.0):
        self.kind, self.x, self.y, self.prior = kind, x, y, prior
        self.n, self.p = x.shape
        self.xtx, self.yty, self.xty = x.T @ x, np.sum(y ** 2), x.T @ y
        if kind == "bic":
            self.lamb = bic_lamb
            self.coef_len = np.log(self.n) * self.lamb
            self.coef_log = self.n * self.lamb
            self.coef_in_log = self.yty
            self.iv2 = 0.0
            return
        self.nu = nu
        self.lamb = self.sig2_full() if lamb is None else lamb
        if kind == "bvs":
            self.iv2 = float(np.reshape(self.lamb / 10.0, -1)[0]) if iv2 is None else iv2
            self.coef_len = -0.5 * np.log(self.iv2)
            self.coef_log = 0.5 * (self.nu + self.n)
            self.coef_in_log = self.nu * self.lamb + self.yty
        else:
            self.iv2 = 0.0
            self.g = self.n if g is None else g
            self.coef_len = 0.5 * np.log(1 + self.g)
            self.coef_log = 0.5 * (self.n + self.nu)
            self.coef_in_log = self.nu * self.lamb + self.yty
            self.gogp1 = self.g / (self.g + 1.0)

    def sig2_full(self):
        _, _, btb = chol_and_friends(np.ones((1, self.p), dtype=bool), self.xtx, self.xty, 0.0)
        return (self.yty - btb) / self.n

    def chol(self, gamma):
        return chol_and_friends(gamma, self.xtx, self.xty, self.iv2)

    def loglik(self, gamma):
        len_gam, ldet, wtw = self.chol(gamma)
        if self.kind == "bic":
            return -(self.coef_len * len_gam + self.coef_log * np.log(self.coef_in_log - wtw))
        if self.kind == "bvs":
            return -(self.coef_len * len_gam + ldet + self.coef_log * np.log(self.coef_in_log - wtw))
        return -(self.coef_len * len_gam + self.coef_log * np.log(self.coef_in_log - self.gogp1 * wtw))


class NestedLogistic:                                          # binary_smc.py:83-143
    def __init__(self, coeffs, edgy):
        self.coeffs, self.edgy, self.dim = coeffs, edgy, len(edgy)

    def predict_prob(self, x, i):
        if self.edgy[i]:
            return self.coeffs[i, i]
        lin = 0.0 if i == 0 else np.sum(self.coeffs[i, :i] * x[:, :i], axis=1)
        return expit(self.coeffs[i, i] + lin)

    def rvs(self, size, u=None):
        """(draws, uniforms (p, size) consumed)."""
        out = np.empty((size, self.dim), dtype=bool)
        us = np.empty((self.dim, size))
        for i in range(self.dim):
            us[i] = np.random.rand(size) if u is None else u[i]
            out[:, i] = us[i] < self.predict_prob(out, i)
        return out, us

    def logpdf(self, x):
        lp = np.zeros(x.shape[0])
        for i in range(self.dim):
            p = self.predict_prob(x, i)
            lp += np.where(x[:, i], log_no_warn(p), log_no_warn(1.0 - p))
        return lp

    @classmethod
    def fit(cls, W, x, probs_thresh=0.02, corr_thresh=0.075):
        from sklearn.linear_model import LogisticRegression
        N, dim = x.shape
        coeffs = np.zeros((dim, dim))
        ph = np.average(x, weights=W, axis=0)
        edgy = (ph < probs_thresh) | (ph > 1.0 - probs_thresh)
        for i in range(dim):
            if edgy[i]:
                coeffs[i, i] = ph[i]
                continue
            preds = []
            for j in range(i):
                pij = np.average(x[:, i] & x[:, j], weights=W, axis=0)
                varij = ph[i] * (1.0 - ph[i]) * ph[j] * (1.0 - ph[j])
                corr = 0.0 if varij <= 0 else (pij - ph[i] * ph[j]) / np.sqrt(varij)
                if np.abs(corr) > corr_thresh:
                    preds.append(j)
            if preds:
                reg = LogisticRegression(penalty=None)
                reg.fit(x[:, preds], x[:, i], sample_weight=W)
                coeffs[i, i] = reg.intercept_[0]
                coeffs[i, preds] = reg.coef_
            else:
                coeffs[i, i] = logit(ph[i])
        return cls(coeffs, edgy)


def target(model, epn):                                       # Tempering.current_target, smc_samplers.py:836-845
    def func(x):
        x.lprior = model.prior.logpdf(x.theta)
        x.llik = model.loglik(x.theta)
        x.lpost = x.lprior + epn * x.llik if epn > 0.0 else x.lprior.copy()
    return func


def metropolis_step(x, tgt, prop, u_prop=None, u_acc=None):
    """BinaryMetropolis.proposal + ArrayMetropolis.step (binary_smc.py:158-162, smc_samplers.py:602-611):
    (mean acceptance, pb, proposal uniforms (p, N), acceptance uniforms (N,))."""
    xprop = ThetaParticles(theta=np.empty_like(x.theta))
    xprop.theta, us = prop.rvs(x.N, u_prop)
    delta_lp = prop.logpdf(x.theta) - prop.logpdf(xprop.theta)
    tgt(xprop)
    lp_acc = xprop.lpost - x.lpost + delta_lp
    pb = np.exp(np.clip(lp_acc, None, 0.0))
    ua = np.random.rand(x.N) if u_acc is None else u_acc
    x.copyto(xprop, where=ua < pb)
    return np.mean(pb), pb, us, ua


def wf_move(x, tgt, prop, P, u_prop=None, u_acc=None):
    """MCMCSequenceWF.__call__ (smc_samplers.py:672-683): (P*M particles, pb (P-1, M), noise in the device layout:
    proposal uniforms (P-1, p, M), acceptance uniforms (P-1, M))."""
    xs, pbs, ups, uas = [x], [], [], []
    for s in range(P - 1):
        x = x.copy()
        _, pb, us, ua = metropolis_step(x, tgt, prop, None if u_prop is None else u_prop[s],
                                        None if u_acc is None else u_acc[s])
        xs.append(x)
        pbs.append(pb), ups.append(us), uas.append(ua)
    return ThetaParticles.concatenate(*xs), np.array(pbs), (np.array(ups), np.array(uas))


class BinaryTemperingWF(AdaptiveTemperingWF):
    """AdaptiveTempering(model, len_chain=P, move=MCMCSequenceWF(BinaryMetropolis(), len_chain=P))."""

    def target(self, epn):
        return target(self.model, epn)

    def calibrate(self, W, x):
        x.shared["proposal"] = NestedLogistic.fit(W, x.theta)

    def mh_step(self, x, tgt):
        return metropolis_step(x, tgt, x.shared["proposal"])[0]


def run_binary_tempering(model, N, len_chain, ESSrmin=0.5):
    """particles.SMC(fk=AdaptiveTempering(...), N=N).run() for a binary model, after the caller's np.random.seed."""
    import oracle.samplers_numpy as sn
    saved = sn.AdaptiveTemperingWF
    sn.AdaptiveTemperingWF = BinaryTemperingWF
    try:
        return run_tempering(model, N, len_chain=len_chain, ESSrmin=ESSrmin)
    finally:
        sn.AdaptiveTemperingWF = saved


def boston_like(n=506, seed=0):
    """A Boston-shaped design: intercept + 13 correlated base columns (one binary, like CHAS), their squares (but the
    binary one's) and pairwise products, centred as papers/binarySMC/boston.py does: p = 104.  y = a log-price-like
    response from a sparse linear model on 12 of the columns."""
    r = np.random.RandomState(seed)
    L = np.linalg.cholesky(0.5 * np.eye(13) + 0.5 * np.ones((13, 13)) * r.uniform(0.2, 0.8))
    base = r.standard_normal((n, 13)) @ L.T
    base = base * r.uniform(0.5, 3.0, 13) + r.uniform(0.0, 5.0, 13)
    base[:, 3] = (base[:, 3] > np.median(base[:, 3])).astype(float)
    cols = [np.ones(n)]
    for i in range(13):
        cols.append(base[:, i])
        if i != 3:
            cols.append(base[:, i] ** 2)
        for j in range(i):
            cols.append(base[:, i] * base[:, j])
    X = np.stack(cols, axis=1)
    X[:, 1:] -= X[:, 1:].mean(axis=0)
    beta = np.zeros(X.shape[1])
    active = r.choice(np.arange(1, X.shape[1]), 12, replace=False)
    beta[active] = r.choice([-1.0, 1.0], 12) * r.uniform(0.5, 1.0, 12) / X[:, active].std(axis=0)
    y = 3.0 + X @ beta * 0.15 + 0.2 * r.standard_normal(n)
    return X, y


def small_design(n=60, p=10, seed=1):
    """A p = 10 design with a few active, correlated predictors."""
    r = np.random.RandomState(seed)
    X = r.standard_normal((n, p))
    X[:, 1] += 0.7 * X[:, 0]
    X[:, 5] -= 0.5 * X[:, 4]
    y = 1.5 * X[:, 0] - 1.0 * X[:, 4] + 0.5 * X[:, 7] + r.standard_normal(n)
    return X, y
