"""Golden vectors for IBIS (data tempering) on the logistic-regression model, from the LIVE reference.

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<checkout of the reference> python tests/golden/make_golden_ibis.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import particles  # noqa: E402
from particles import smc_samplers as ssp  # noqa: E402
from make_golden_tempering import make_model  # noqa: E402
from oracle.samplers_numpy import synthetic_logistic  # noqa: E402  (data generator only)

HERE = os.path.dirname(os.path.abspath(__file__))


def run(data, N, wastefree, len_chain, seed, ESSrmin=0.5):
    np.random.seed(seed)
    fk = ssp.IBIS(model=make_model(data), wastefree=wastefree, len_chain=len_chain)
    pf = particles.SMC(fk=fk, N=N, ESSrmin=ESSrmin)
    pf.run()
    return pf


if __name__ == "__main__":
    g = {}
    data = synthetic_logistic(150, 4, seed=3)
    g["exact/data"] = data
    # waste-free: N = 100 chains of length 8; standard: N = 100 particles, 3 Metropolis steps per move
    for tag, wf, lc, seed in (("wf", True, 8, 17), ("std", False, 4, 18)):
        pf = run(data, 100, wf, lc, seed)
        g["exact/%s/logLts" % tag] = np.array(pf.summaries.logLts)
        g["exact/%s/ESSs" % tag] = np.array(pf.summaries.ESSs)
        g["exact/%s/rs_flags" % tag] = np.array(pf.summaries.rs_flags)
        g["exact/%s/theta" % tag] = pf.X.theta["beta"]
        g["exact/%s/lpost" % tag] = pf.X.lpost
        g["exact/%s/meta" % tag] = np.array([100, lc, seed, int(wf)])
        print(tag, "logLt", pf.logLt, "resamplings", int(np.sum(pf.summaries.rs_flags)))
    # Monte-Carlo anchors: d = 6, n_data = 300, N = 200 chains x P = 20 (4000 particles), waste-free
    data2 = synthetic_logistic(300, 6, seed=4)
    g["stat/data"] = data2
    lls, means = [], []
    for r in range(12):
        pf = run(data2, 200, True, 20, 100 + r)
        lls.append(pf.logLt)
        means.append(np.average(pf.X.theta["beta"], weights=pf.W, axis=0))
    g["stat/logLt"] = np.array(lls)
    g["stat/post_mean"] = np.array(means)
    g["stat/meta"] = np.array([200, 20])
    np.savez_compressed(os.path.join(HERE, "golden_ibis.npz"), **g)
    print("stat logLt mean/sd", np.mean(lls), np.std(lls, ddof=1))
