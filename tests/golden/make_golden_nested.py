"""Golden vectors for nested sampling SMC on the logistic-regression model, from the LIVE reference.

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<checkout of the reference> python tests/golden/make_golden_nested.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import particles  # noqa: E402
from particles import nested  # noqa: E402
from particles import smc_samplers as ssp  # noqa: E402
from make_golden_tempering import make_model  # noqa: E402
from oracle.samplers_numpy import synthetic_logistic  # noqa: E402  (data generator only)

HERE = os.path.dirname(os.path.abspath(__file__))


def run(fk, N, seed):
    np.random.seed(seed)
    pf = particles.SMC(fk=fk, N=N)
    pf.run()
    return pf


if __name__ == "__main__":
    g = {}
    data = synthetic_logistic(150, 4, seed=3)
    g["exact/data"] = data
    # waste-free: N = 100 chains of length 8; standard: N = 100 particles, 3 Metropolis steps per move
    for tag, wf, lc, seed, alpha in (("wf", True, 8, 17, 0.3), ("std", False, 4, 18, 0.5)):
        fk = nested.NestedSamplingSMC(model=make_model(data), wastefree=wf, len_chain=lc, ESSrmin=alpha)
        pf = run(fk, 100, seed)
        g["exact/%s/lts" % tag] = np.array(pf.X.shared["lts"])
        g["exact/%s/log_evid" % tag] = np.array(pf.X.shared["log_evid"])
        g["exact/%s/theta" % tag] = pf.X.theta["beta"]
        g["exact/%s/lpost" % tag] = pf.X.lpost
        g["exact/%s/llik" % tag] = pf.X.llik
        g["exact/%s/meta" % tag] = np.array([100, lc, seed, int(wf), alpha, 0.01, pf.t])
        print(tag, "log_evid", pf.X.shared["log_evid"][-1], "generations", pf.t)
    # Monte-Carlo anchors: d = 6, n_data = 300, N = 200 chains x P = 20, ESSrmin = 0.5, waste-free; NS-SMC and
    # adaptive tempering on the same data
    data2 = synthetic_logistic(300, 6, seed=4)
    g["stat/data"] = data2
    ns, temp, gens = [], [], []
    for r in range(12):
        pf = run(nested.NestedSamplingSMC(model=make_model(data2), len_chain=20, ESSrmin=0.5), 200, 100 + r)
        ns.append(pf.X.shared["log_evid"][-1])
        gens.append(pf.t)
        pf = run(ssp.AdaptiveTempering(model=make_model(data2), len_chain=20, ESSrmin=0.5), 200, 200 + r)
        temp.append(pf.logLt)
    g["stat/ns_log_evid"] = np.array(ns)
    g["stat/ns_generations"] = np.array(gens)
    g["stat/tempering_logLt"] = np.array(temp)
    g["stat/meta"] = np.array([200, 20, 0.5, 0.01])
    np.savez_compressed(os.path.join(HERE, "golden_nested.npz"), **g)
    print("NS-SMC log_evid mean/sd", np.mean(ns), np.std(ns, ddof=1), "generations", gens)
    print("tempering logLt mean/sd", np.mean(temp), np.std(temp, ddof=1))
