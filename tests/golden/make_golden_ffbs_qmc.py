"""Write golden_ffbs_qmc.npz from the live reference (run where a checkout of it is importable):

    PYTHONPATH=<reference checkout> python tests/golden/make_golden_ffbs_qmc.py

The reference's QMC forward-filtering backward-sampling (``SMC(qmc=True, store_history=True)``, then
``hist.backward_sampling_qmc(M)``, smoothing.py:425-455) on recorded point sets: ``particles.rqmc.sobol`` is replaced by
a function that returns recorded scrambled Sobol' points in turn -- the forward pass's T sets, then the backward pass's
(M, T) set -- so that a device run fed the same points must reproduce the reference's history, Hilbert orders and
paths.  Case k stores
  k/meta = [model code, N, T, M], k/y: the data (T, dy);
  k/u{t}: the forward points of step t ((N, du) at t = 0, (N, du + 1) afterwards), k/ub: the backward points (M, T);
  k/X (T, N[, d]), k/lw (T, N), k/A (T, N) (row 0 unused), k/h (T-1, N): the history and its ``h_orders``;
  k/paths (T, M[, d]) and k/idx (T, M): the paths and the particle index of each component (found by equality).
"""
import os
import warnings

import numpy as np
import particles
from particles import core, kalman, rqmc
from particles import state_space_models as ssm

MODELS = {0: lambda: ssm.StochVol(), 1: lambda: kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
          2: lambda: ssm.Gordon_etal(), 3: lambda: ssm.DiscreteCox(), 4: lambda: ssm.BearingsOnly(),
          5: lambda: kalman.MVLinearGauss_Guarniero_etal(dx=2)}
# (model code, N, T, M)
CASES = [(0, 100, 10, 64), (1, 100, 10, 64), (2, 64, 8, 64), (3, 64, 8, 64), (4, 64, 6, 64), (5, 64, 6, 64),
         (0, 64, 1, 32)]

warnings.simplefilter("ignore")
out = {}
for c, (mc, N, T, M) in enumerate(CASES):
    model = MODELS[mc]()
    np.random.seed(700 + c)
    _, y = model.simulate(T)
    fk = ssm.Bootstrap(ssm=model, data=y)
    pts = [rqmc.sobol(N, fk.du) if t == 0 else rqmc.sobol(N, fk.du + 1) for t in range(T)]
    ub = rqmc.sobol(M, T)
    feed = iter(pts + [ub])
    saved = rqmc.sobol
    core.rqmc.sobol = lambda n, d: next(feed)
    try:
        pf = particles.SMC(fk=fk, N=N, qmc=True, store_history=True)
        pf.run()
        h = pf.hist
        paths = h.backward_sampling_qmc(M)
    finally:
        core.rqmc.sobol = saved
    X = np.array([np.asarray(x, dtype=np.float64) for x in h.X])
    P = np.array([np.asarray(p, dtype=np.float64).reshape((M,) + X.shape[2:]) for p in paths])
    idx = np.empty((T, M), dtype=np.int64)
    for t in range(T):
        for m in range(M):
            eq = X[t] == P[t, m]
            idx[t, m] = np.flatnonzero(eq if eq.ndim == 1 else eq.all(axis=1))[0]
    k = str(c)
    out[k + "/meta"] = np.array([mc, N, T, M])
    out[k + "/y"] = np.array([np.asarray(v, dtype=np.float64).reshape(-1) for v in y])
    for t in range(T):
        out[k + f"/u{t}"] = pts[t]
    out[k + "/ub"] = ub
    out[k + "/X"] = X
    out[k + "/lw"] = np.array([np.asarray(w.lw, dtype=np.float64) for w in h.wgts])
    out[k + "/A"] = np.array([np.zeros(N, dtype=np.int64)] + [np.asarray(a, dtype=np.int64) for a in h.A[1:]])
    out[k + "/h"] = np.array([np.asarray(o, dtype=np.int64) for o in h.h_orders]).reshape(T - 1, N)
    out[k + "/paths"] = P
    out[k + "/idx"] = idx
out["n_cases"] = np.array(len(CASES))
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_ffbs_qmc.npz"), **out)
