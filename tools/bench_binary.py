"""SMC on binary spaces on one GPU: the Boston-shaped variable-selection workload of the reference's
papers/binarySMC/boston.py -- p = 104 predictors (intercept, 13 base columns, squares, pairwise products, centred),
BayesianVS with an IID(Bernoulli(0.5), p) prior, N = 10^5 particles as M = 100 chains of len_chain P = 1000,
waste-free adaptive tempering with BinaryMetropolis.  The design is synthetic (tests/binary_oracle.boston_like).

One untimed tempering run from the prior brings the particles to a realistic state (the proposal fitted at the last
calibration, the exponent reached); then, at that state:
  * move_ms: device time of one fused waste-free move (smcb_binary_wf_move, all P-1 steps of all M chains), CUDA
    events around --reps moves after one untimed move;
  * vs_loglik_ms: device time of smcb_vs_loglik over the N = 10^5 particles of the last move, the same way;
  * fit_s: host wall time of NestedLogistic.fit (scikit-learn) on the N weighted particles, per calibration;
  * particle_steps_per_s: M (P - 1) / move time;
  * fp64 FLOP/s: sum over the realised gammas of |gamma|^3 / 3 + |gamma|^2 (Cholesky and the appended solve row),
    over kernel time, for the move (the proposals it evaluated are not kept: the count uses the states it wrote, which
    hold the accepted proposals and the repeated states) and for smcb_vs_loglik (exact).
--reference K adds the reference's own chol_and_friends + loglik on K of the particles, on one host core
(oracle/_ref), scaled to N.  The GPU's name and power limit are read in the same call.

    python tools/bench_binary.py [--reps 5] [--reference 2000] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_ibis import gpu_info  # noqa: E402


def chol_flops(len_gam):
    """fp64 operations of one factorisation of the augmented (k + 1) x (k + 1) system, summed: k^3 / 3 + k^2."""
    k = np.asarray(len_gam, dtype=np.float64)
    return float(np.sum(k ** 3 / 3.0 + k ** 2))


def device_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--M", type=int, default=100)
    ap.add_argument("--P", type=int, default=1000)
    ap.add_argument("--reference", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = gpu_info()
    import torch
    import particles_b200 as pb
    from particles_b200 import binary_smc as bs, distributions as dists, smc_samplers as ssp
    import binary_oracle as bo

    X, y = bo.boston_like()
    p = X.shape[1]
    model = bs.BayesianVS(data=(X, y), prior=dists.IID(bs.Bernoulli(0.5), p))
    M, P = args.M, args.P
    pb.seed(1)
    move = ssp.MCMCSequenceWF(mcmc=bs.BinaryMetropolis(), len_chain=P)
    fk = ssp.AdaptiveTempering(model, len_chain=P, move=move)
    t0 = time.perf_counter()
    pf = pb.SMC(fk=fk, N=M)
    pf.run()
    torch.cuda.synchronize()
    run_s = time.perf_counter() - t0
    X_last = pf.X
    epn = X_last.shared["exponents"][-1]
    # the state a move starts from: M chains resampled from the last generation, with its proposal
    W = pf.W
    t0 = time.perf_counter()
    bs.BinaryMetropolis().calibrate(W, X_last)
    fit_s = time.perf_counter() - t0
    A = torch.multinomial(W, M, replacement=True)
    x0 = X_last[A]
    out = {}
    move_ms = device_ms(lambda: out.__setitem__("x", model.wf_move(x0, epn, P)), args.reps)
    moved = out["x"]
    len_move = moved.theta.sum(dim=1).cpu().numpy()
    ll_ms = device_ms(lambda: model.loglik(moved.theta), args.reps)
    flops_move = chol_flops(len_move[M:])          # rows 1..P-1: one factorisation per step and chain
    flops_ll = chol_flops(len_move)
    res = dict(info, workload="boston-shaped BayesianVS p=%d, N=%d (M=%d chains x P=%d)" % (p, M * P, M, P),
               full_run_s=round(run_s, 2), tempering_steps=len(X_last.shared["exponents"]) - 1,
               move_ms=round(move_ms, 3), vs_loglik_ms=round(ll_ms, 3), fit_s=round(fit_s, 3),
               particle_steps_per_s=M * (P - 1) / (move_ms * 1e-3),
               move_fp64_gflops=flops_move / (move_ms * 1e-3) / 1e9,
               vs_loglik_fp64_gflops=flops_ll / (ll_ms * 1e-3) / 1e9,
               mean_len_gam=float(len_move.mean()), max_len_gam=int(len_move.max()),
               logLt=float(pf.logLt))
    if args.reference:
        ref_dir = os.path.join(ROOT, "oracle", "_ref")
        if os.path.isdir(os.path.join(ref_dir, "particles")):
            os.environ["OMP_NUM_THREADS"] = "1"
            sys.path.insert(0, ref_dir)
            from particles import binary_smc as rbin
            from particles import distributions as rdists
            rmodel = rbin.BayesianVS(data=(X, y), prior=rdists.IID(rbin.Bernoulli(0.5), p))
            g = moved.theta[:args.reference].cpu().numpy()
            t0 = time.perf_counter()
            rmodel.loglik(g)
            dt = time.perf_counter() - t0
            res["reference_loglik_s_per_1e5"] = dt * 1e5 / args.reference
            res["reference_sample"] = args.reference
        else:
            res["reference_loglik_s_per_1e5"] = "not measured (oracle/_ref missing)"
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
