"""Write golden_sqmc.npz from the live reference (run where a checkout of it is importable):

    PYTHONPATH=<reference checkout> python tests/golden/make_golden_sqmc.py

* ``xint_d``, ``keys_d`` (d = 2..6): integer points and ``hilbert.hilbert_array`` of them.  The points mix standardised
  normal points scaled as ``hilbert_sort`` scales them (keys that wrap mod 2^64 from d = 4 on) with small coordinates,
  so that the number of chunks differs from point to point.
* ``x_d``, ``order_d`` (d = 1..4): float points and ``hilbert.hilbert_sort`` of them.
* ``run_k_*``: reference SQMC runs on recorded point sets (part (b) below).
"""
import os

import numpy as np
from particles import hilbert

rng = np.random.default_rng(20261018)
out = {}
for d in range(2, 7):
    n = 800
    x = rng.standard_normal((n, d))
    xs = hilbert.invlogit((x - x.mean(0)) / x.std(0))
    xint = np.floor(xs * np.floor(2 ** (62 / d))).astype(np.int64)
    xint[:200] = rng.integers(0, 2 ** rng.integers(1, 12, size=(200, 1)), size=(200, d))
    out[f"xint_{d}"] = xint
    out[f"keys_{d}"] = hilbert.hilbert_array(xint)
for d in range(1, 5):
    x = rng.standard_normal((500, d)) * rng.uniform(0.1, 10.0, size=d)
    out[f"x_{d}"] = x
    out[f"order_{d}"] = hilbert.hilbert_sort(x[:, 0] if d == 1 else x)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_sqmc.npz"), **out)


# ------------------------------------------------------------------------------------------------------------------
# (b) reference SQMC runs on recorded point sets.  particles.rqmc.sobol is replaced by a function that returns the
# recorded scrambled Sobol' points of each call in turn, so that a device run fed the same points must reproduce the
# reference's ancestors, particles, Hilbert orders, weights and logLt.  Case k stores
#   run_k_u{t}: the points of step t ((N, du) at t = 0, (N, du + 1) afterwards, already squeezed as rqmc.sobol does),
#   run_k_y: the data, run_k_{X,A,h,W}{t}, run_k_logLt: per step, and run_k_meta = [model code, kind code, N, T].
# ------------------------------------------------------------------------------------------------------------------
from scipy.stats import qmc  # noqa: E402
import particles  # noqa: E402
from particles import core, kalman, rqmc  # noqa: E402
from particles import state_space_models as ssm  # noqa: E402
import warnings  # noqa: E402

MODELS = {0: lambda: ssm.StochVol(), 1: lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
          2: lambda: ssm.Gordon_etal(), 3: lambda: ssm.BearingsOnly(),
          4: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=2), 5: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=3)}
KINDS = {0: ssm.Bootstrap, 1: ssm.GuidedPF, 2: ssm.AuxiliaryPF, 3: ssm.AuxiliaryBootstrap}
CASES = [(m, k, 100) for m in (0, 1) for k in range(4)] + [(2, 0, 100), (3, 0, 64)] + \
        [(4, k, 64) for k in range(4)] + [(5, 0, 64), (5, 1, 64)]
T = 5
warnings.simplefilter("ignore")
for c, (mc, kc, N) in enumerate(CASES):
    model = MODELS[mc]()
    np.random.seed(100 + c)
    _, y = model.simulate(T)
    fk = KINDS[kc](ssm=model, data=y)
    pts = [rqmc.sobol(N, fk.du) if t == 0 else rqmc.sobol(N, fk.du + 1) for t in range(T)]
    feed = iter(pts)
    saved, core.rqmc.sobol = core.rqmc.sobol, lambda n, d: next(feed)
    try:
        pf = particles.SMC(fk=fk, N=N, qmc=True)
        rec = {}
        for t in range(T):
            next(pf)
            X = np.asarray(pf.X, dtype=np.float64)
            rec[f"X{t}"], rec[f"W{t}"] = X.copy(), np.asarray(pf.W).copy()
            if t > 0:
                rec[f"A{t}"], rec[f"h{t}"] = np.asarray(pf.A).copy(), np.asarray(pf.h_order).copy()
            rec.setdefault("logLt", []).append(pf.logLt)
    finally:
        core.rqmc.sobol = saved
    out[f"run_{c}_meta"] = np.array([mc, kc, N, T])
    out[f"run_{c}_y"] = np.array([np.asarray(v, dtype=np.float64).reshape(-1) for v in y])
    for t in range(T):
        out[f"run_{c}_u{t}"] = pts[t]
    for k, v in rec.items():
        out[f"run_{c}_{k}"] = np.asarray(v)
out["n_runs"] = np.array(len(CASES))
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_sqmc.npz"), **out)
