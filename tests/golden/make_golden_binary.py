"""Golden vectors for the SMC samplers on binary spaces (particles/binary_smc.py), from the LIVE reference, on seeded
synthetic designs (p = 10, and a Boston-shaped p = 104).

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<checkout of the reference> python tests/golden/make_golden_binary.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import particles  # noqa: E402
from particles import binary_smc as bin  # noqa: E402
from particles import distributions as dists  # noqa: E402
from particles import smc_samplers as ssp  # noqa: E402
from binary_oracle import boston_like, small_design  # noqa: E402  (data generators only)


def gammas(p, r, n=40):
    g = r.rand(n, p) < r.uniform(0.05, 0.6, (n, 1))
    g[0] = False
    g[1] = True
    g[2] = False
    g[2, p // 2] = True
    return g


if __name__ == "__main__":
    out = {}
    r = np.random.RandomState(5)
    for tag, (X, y) in (("p10", small_design()), ("p104", boston_like())):
        p = X.shape[1]
        out[tag + "/Xy_sums"] = np.array([X.sum(), y.sum()])
        prior = dists.IID(bin.Bernoulli(0.5), p)
        g = gammas(p, r)
        out[tag + "/gamma"] = g
        models = {"bic": bin.BIC(data=(X, y)), "bvs": bin.BayesianVS(data=(X, y), prior=prior),
                  "gprior": bin.BayesianVS_gprior(data=(X, y), prior=prior)}
        for name, m in models.items():
            m.prior = prior
            len_gam, ldet, wtw = m.chol_intermediate(g)
            out[tag + "/%s/len_gam" % name] = len_gam
            out[tag + "/%s/ldet" % name] = ldet
            out[tag + "/%s/wtw" % name] = wtw
            out[tag + "/%s/loglik" % name] = m.loglik(g)
            out[tag + "/%s/consts" % name] = np.hstack([m.iv2, m.coef_len, m.coef_log, m.coef_in_log]).astype(float)
        # NestedLogistic.fit on a weighted sample, then rvs under a fixed seed and logpdf
        xs = r.rand(1500, p) < np.linspace(0.01, 0.9, p)
        xs[:, 1] ^= xs[:, 0] & (r.rand(1500) < 0.6)
        W = r.rand(1500)
        W /= W.sum()
        nl = bin.NestedLogistic.fit(W, xs)
        out[tag + "/fit/x"], out[tag + "/fit/W"] = xs, W
        out[tag + "/fit/coeffs"], out[tag + "/fit/edgy"] = nl.coeffs, nl.edgy
        np.random.seed(11)
        draws = nl.rvs(size=500)
        out[tag + "/rvs/seed"] = np.array([11, 500])
        out[tag + "/rvs/x"] = draws
        out[tag + "/rvs/logpdf"] = nl.logpdf(draws)
    # one seeded waste-free adaptive tempering run at p = 10 (BayesianVS, N = 50 chains of length 20)
    X, y = small_design()
    prior = dists.IID(bin.Bernoulli(0.5), X.shape[1])
    model = bin.BayesianVS(data=(X, y), prior=prior)
    move = ssp.MCMCSequenceWF(mcmc=bin.BinaryMetropolis(), len_chain=20)
    np.random.seed(21)
    pf = particles.SMC(fk=ssp.AdaptiveTempering(model, len_chain=20, move=move), N=50)
    pf.run()
    out["run/exponents"] = np.array(pf.X.shared["exponents"])
    out["run/logLt"] = np.array(pf.logLt)
    out["run/meta"] = np.array([50, 20, 21])
    print("run: exponents", out["run/exponents"], "logLt", pf.logLt)
    np.savez_compressed(os.path.join(HERE, "golden_binary.npz"), **out)
