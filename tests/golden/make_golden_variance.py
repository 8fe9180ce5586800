"""Single-run variance estimators of the LIVE reference (particles/variance_estimators.py, which needs numba) on small
seeded problems: the data fixture that tests/test_variance_host.py checks the NumPy oracle (tests/variance_oracle.py)
against, and that tests/test_gpu_variance.py replays through the device collectors.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_variance.py

For each case: simulate data, run a seeded ``particles.SMC(store_history=LAG)`` collecting ``Var``, ``Var_logLt``,
``Lag_based_var`` and ``Fixed_lag_smooth`` next to a recorder of the per-step X, lw and A (A = arange on steps that
do not resample, as core.py:335).  Also records hand-made ``var_estimate`` inputs and, for the statistical test,
the per-t mean and standard deviation of ``var_logLt``, ``var`` and ``logLts`` over RUNS runs of the model of the
reference's notebook docs/source/notebooks/variance_estimation.ipynb.  Writes tests/golden/golden_variance.npz."""
import os
import sys

import numpy as np

sys.path.insert(0, "/root/reference")
import particles  # noqa: E402
from particles import collectors as cols  # noqa: E402
from particles import kalman  # noqa: E402
from particles import state_space_models as ssms  # noqa: E402
from particles import variance_estimators as ve  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
T, N, LAG = 50, 200, 5
T_PLUGIN = 25
RUNS, T_STAT, N_STAT = 300, 50, 1000


def phi_sq(x):
    return x ** 2


def phi_fl(xs):                     # Fixed_lag_smooth: sum over the window of the first component
    return sum(x if x.ndim == 1 else x[:, 0] for x in xs)


# name -> (model, resampling, N, T, seed, vector phi?)
CASES = {
    "sv_sys": (lambda: ssms.StochVol(), "systematic", N, T, 41, False),
    "lg_multi": (lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "multinomial", N, T, 42, False),
    "sv_strat": (lambda: ssms.StochVol(), "stratified", N, T, 43, False),
    "mvlg2": (lambda: kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=2), "systematic", N, T, 44, True),
    # the plugin-path schemes run shorter, to keep the file under 1 MB
    "sv_ssp": (lambda: ssms.StochVol(), "ssp", N, T_PLUGIN, 45, False),
    "sv_resid": (lambda: ssms.StochVol(), "residual", N, T_PLUGIN, 46, False),
    "sv_kill": (lambda: ssms.StochVol(), "killing", N, T_PLUGIN, 47, False),
    "collapse": (lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "multinomial", 8, 120, 48, False),
}


class Rec(cols.Collector):
    def fetch(self, smc):
        A = np.arange(smc.N) if smc.A is None else np.asarray(smc.A)
        return (np.array(smc.X, dtype=float), np.array(smc.wgts.lw, dtype=float), A)


def run_case(name):
    make, scheme, n, t_len, seed, vector = CASES[name]
    model = make()
    np.random.seed(seed)
    _, y = model.simulate(t_len)
    np.random.seed(seed + 100)
    phi = None if vector else phi_sq
    pf = particles.SMC(fk=ssms.Bootstrap(ssm=model, data=y), N=n, resampling=scheme, store_history=LAG,
                       collect=[Rec(), ve.Var(phi=phi), ve.Var_logLt(), ve.Lag_based_var(phi=phi),
                                cols.Fixed_lag_smooth(phi=phi_fl)])
    pf.run()
    s = pf.summaries
    out = {f"{name}/data": np.array([np.asarray(v, dtype=float).reshape(-1) for v in y]),
           f"{name}/X": np.array([r[0] for r in s.rec]), f"{name}/lw": np.array([r[1] for r in s.rec]),
           f"{name}/A": np.array([r[2] for r in s.rec], dtype=np.int16), f"{name}/rs": np.array(s.rs_flags, dtype=bool),
           f"{name}/var": np.array(s.var, dtype=float), f"{name}/var_logLt": np.array(s.var_logLt, dtype=float),
           f"{name}/fixed_lag_smooth": np.array(s.fixed_lag_smooth, dtype=float)}
    lag = s.lag_based_var                         # list over t of lists of length min(t + 1, LAG)
    flat = np.full((t_len, LAG) + np.shape(lag[0][0]), np.nan)
    for t, row in enumerate(lag):
        flat[t, :len(row)] = np.array(row, dtype=float)
    out[f"{name}/lag_based_var"] = flat
    zeros = int(np.sum(np.array(s.var, dtype=float) == 0.0))
    print(name, scheme, "resampled", int(np.sum(s.rs_flags)), "zero var", zeros, flush=True)
    return out


def hand_made():
    r = np.random.RandomState(7)
    cases = {}
    W = r.uniform(size=30)
    W /= W.sum()
    phi = r.normal(size=30)
    cases["all_equal"] = (W, phi, np.full(30, 4))
    cases["unsorted_ends"] = (W, phi, np.array([3] + list(r.randint(0, 10, size=28)) + [3]))
    cases["unsorted"] = (W, phi, np.array([0] + list(r.randint(0, 10, size=28)) + [9]))
    cases["n1"] = (np.array([1.0]), np.array([2.5]), np.array([0]))
    cases["singletons"] = (W, phi, np.arange(30))
    cases["vector"] = (W, r.normal(size=(30, 3)), np.sort(r.randint(0, 6, size=30)))
    out = {}
    for k, (w, p, b) in cases.items():
        out[f"hand/{k}/W"], out[f"hand/{k}/phi"], out[f"hand/{k}/B"] = w, p, b
        out[f"hand/{k}/out"] = np.asarray(ve.var_estimate(w, p, b), dtype=float)
    return out


def statistics():
    """The notebook's model: LinearGauss(rho=0.9, sigmaX=1, sigmaY=0.2), T = 50, N = 1000, multinomial."""
    model = kalman.LinearGauss(rho=0.9, sigmaX=1.0, sigmaY=0.2)
    np.random.seed(1)
    _, y = model.simulate(T_STAT)
    fk = ssms.Bootstrap(ssm=model, data=y)
    np.random.seed(2)
    v, vl, ll = [], [], []
    for _ in range(RUNS):
        pf = particles.SMC(fk=fk, N=N_STAT, resampling="multinomial", collect=[ve.Var(), ve.Var_logLt()])
        pf.run()
        v.append(pf.summaries.var)
        vl.append(pf.summaries.var_logLt)
        ll.append(pf.summaries.logLts)
    out = {"stat/data": np.array([np.asarray(e, dtype=float).reshape(-1) for e in y])}
    for key, a in (("var", v), ("var_logLt", vl), ("logLts", ll)):
        a = np.array(a, dtype=float)
        out[f"stat/{key}_mean"], out[f"stat/{key}_sd"] = a.mean(0), a.std(0, ddof=1)
    out["stat/runs"] = np.array([RUNS, T_STAT, N_STAT])
    return out


def main():
    out = {}
    for name in CASES:
        out.update(run_case(name))
    out.update(hand_made())
    out.update(statistics())
    out["meta/T_N_LAG"] = np.array([T, N, LAG])
    np.savez_compressed(os.path.join(HERE, "golden_variance.npz"), **out)


if __name__ == "__main__":
    main()
