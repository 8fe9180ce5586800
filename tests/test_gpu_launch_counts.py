"""Kernel launches per C entry point: smcb_launch_count (bench.py's gpu_launches) must advance by exactly the number
of kernels each entry point enqueues.  Every launching entry point is called once at a small size, directly through
the C-ABI or, for the descriptor-driven ones, through the Python layer with each C call's delta recorded."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 64


@pytest.fixture(scope="module")
def ctx():
    from particles_b200.device import context
    return context()


def buf(n=4096, dtype=torch.float64, fill=0.0):
    return torch.full((n,), fill, dtype=dtype, device="cuda")


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def hp(a):
    return a.ctypes.data_as(C.c_void_p)


def launches(ctx, fn, *args):
    from particles_b200 import _lib
    c0 = ctx.lib.smcb_launch_count(ctx.handle)
    _lib.check(fn(ctx.handle, *args))
    torch.cuda.synchronize()
    return ctx.lib.smcb_launch_count(ctx.handle) - c0


def test_weights_scan_search_resample(ctx):
    L = ctx.lib
    lw, W, out, stats = buf(fill=-1.0), buf(fill=1.0 / N), buf(), buf()
    x, A = buf(fill=0.5), buf(dtype=torch.int64)
    cdf = torch.linspace(1.0 / N, 1.0, N, dtype=torch.float64, device="cuda")
    got = {
        "normalise": launches(ctx, L.smcb_normalise, p(lw), N, p(W), p(stats)),
        "normalise, no W": launches(ctx, L.smcb_normalise, p(lw), N, None, p(stats)),
        "weights_from_stats": launches(ctx, L.smcb_weights_from_stats, p(lw), N, p(stats), p(out)),
        "lse sum": launches(ctx, L.smcb_lse, 0, p(lw), None, N, p(out)),
        "lse mean": launches(ctx, L.smcb_lse, 1, p(lw), None, N, p(out)),
        "lse weighted mean": launches(ctx, L.smcb_lse, 1, p(lw), p(W), N, p(out)),
        "lse essl": launches(ctx, L.smcb_lse, 2, p(lw), None, N, p(out)),
        "exp_and_normalise": launches(ctx, L.smcb_exp_and_normalise, p(lw), N, p(W)),
        "wmean_and_var": launches(ctx, L.smcb_wmean_and_var, p(W), p(x), N, 2, p(out)),
        "cumsum": launches(ctx, L.smcb_cumsum, p(W), N, p(out)),
        "searchsorted": launches(ctx, L.smcb_searchsorted, p(cdf), N, p(x), N, p(A)),
        "gather": launches(ctx, L.smcb_gather, p(x), N, p(A), N, 2, p(out)),
        "gather_rows": launches(ctx, L.smcb_gather_rows, p(x), N, p(A), N, 2, p(out)),
    }
    W = buf(fill=1.0 / N)
    scratch = buf(int(L.smcb_resample_scratch_doubles(N, N)) + 64)
    for name, code in (("systematic", 2), ("stratified", 1), ("multinomial", 0), ("residual", 3), ("ssp", 4)):
        got[name] = launches(ctx, L.smcb_resample, code, p(W), N, N, p(A), None, p(scratch))
    # the scans and the search take two launches each; without injected uniforms a resampling draws them first
    assert got == {"normalise": 2, "normalise, no W": 1, "weights_from_stats": 1, "lse sum": 1, "lse mean": 1,
                   "lse weighted mean": 1, "lse essl": 1, "exp_and_normalise": 2, "wmean_and_var": 1, "cumsum": 2,
                   "searchsorted": 2, "gather": 1, "gather_rows": 1, "systematic": 5, "stratified": 5,
                   "multinomial": 7, "residual": 9, "ssp": 5}


def test_distributions_and_law_table(ctx):
    L = ctx.lib
    x, out = buf(fill=0.25), buf()
    loc0, scale0 = np.zeros(16), np.ones(16)
    pars = np.array([1.0, 1.0, 1.0, 0.0])        # scalar parameters of law codes 7-11
    got = {
        "uniform": launches(ctx, L.smcb_uniform, p(out), N),
        "standard_normal": launches(ctx, L.smcb_standard_normal, p(out), N),
        "normal_rvs": launches(ctx, L.smcb_normal_rvs, None, 0.0, None, 1.0, None, p(out), N),
        **{f"dist_logpdf {law}": launches(ctx, L.smcb_dist_logpdf, law, p(x), 0.0, None, None, None, None, hp(pars),
                                          p(out), N) for law in range(7, 12)},
        "device_math": launches(ctx, L.smcb_device_math, 0, p(x), p(out), N),
        "device_math table": launches(ctx, L.smcb_device_math, 4, p(x), p(out), N),
    }
    for d in (2, 12):                       # factor in the kernel parameters / in shared memory
        Lh = np.ascontiguousarray(np.eye(d))
        got[f"mvnormal_rvs d={d}"] = launches(ctx, L.smcb_mvnormal_rvs, None, hp(loc0), None, hp(scale0), hp(Lh), d,
                                              None, p(out), N // d)
        got[f"mvnormal_logpdf d={d}"] = launches(ctx, L.smcb_mvnormal_logpdf, p(x), None, hp(loc0), None,
                                                 hp(scale0), hp(Lh), d, p(out), N // d)
    assert set(got.values()) == {1}, got


def test_samplers(ctx):
    L = ctx.lib
    n, d, P, nd = 16, 2, 3, 8
    theta, data, Lf, lw = buf(fill=0.1), buf(fill=0.5), buf(), buf(fill=-1.0)
    lp, ll, lq, out, W = buf(), buf(), buf(), buf(), buf(fill=1.0 / n)
    th2, lp2, ll2, lq2, pb_ = buf(fill=0.2), buf(), buf(), buf(), buf()
    Lf[0] = Lf[d + 1] = 1.0
    acc = buf(dtype=torch.uint8)
    move = (n, d, P, p(theta), p(lp), p(ll), p(lq), p(data), nd, 5.0)
    move_out = (p(Lf), None, None, p(th2), p(lp2), p(ll2), p(lq2), p(pb_))
    got = {
        "logistic_target": launches(ctx, L.smcb_logistic_target, p(theta), n, d, p(data), nd, 5.0, 0.5, p(lp), p(ll),
                                    p(lq)),
        "logistic_ns_target": launches(ctx, L.smcb_logistic_ns_target, p(theta), n, d, p(data), nd, 5.0, -1e9, p(lp),
                                       p(ll), p(lq)),
        "logistic_wf_move": launches(ctx, L.smcb_logistic_wf_move, *move, 0.5, *move_out),
        "logistic_ns_move": launches(ctx, L.smcb_logistic_ns_move, *move, -1e9, *move_out),
        "logistic_logpyt": launches(ctx, L.smcb_logistic_logpyt, p(theta), n, d, p(data), nd, 0, 2, 1, p(lw), p(lq),
                                    p(ll), None),
        "rw_propose": launches(ctx, L.smcb_rw_propose, p(theta), n, d, p(Lf), None, p(th2)),
        "mh_accept": launches(ctx, L.smcb_mh_accept, n, d, p(theta), p(lp), p(ll), p(lq), p(th2), p(lp2), p(ll2),
                              p(lq2), None, p(out)),
        "mh_accept_flags": launches(ctx, L.smcb_mh_accept_flags, n, d, p(theta), p(lp), p(ll), p(lq), p(th2),
                                    p(lp2), p(ll2), p(lq2), None, p(out), p(acc)),
        "next_annealing_epn": launches(ctx, L.smcb_next_annealing_epn, p(lw), n, 0.2, 0.5, p(out)),
        "rw_calibrate": launches(ctx, L.smcb_rw_calibrate, p(W), p(theta), n, d, 1.0, p(Lf)),
        "wcov_sums": launches(ctx, L.smcb_wcov_sums, p(W), p(theta), n, d, None, p(out)),
        "wcov_sums, mean": launches(ctx, L.smcb_wcov_sums, p(W), p(theta), n, d, p(th2), p(out)),
        "chol_from_sums": launches(ctx, L.smcb_chol_from_sums, p(W), p(W), d, 1.0, p(out)),
        "essl_grid": launches(ctx, L.smcb_essl_grid, p(lw), n, 0.0, 1.0, p(W), p(out)),
        "ns_threshold": launches(ctx, L.smcb_ns_threshold, p(ll), n, 4, 5, 0.5, 1, -0.1, 0.0, 0.01, p(lw), p(out)),
    }
    # next_annealing_epn: the maximum, 11 root-finding passes and the result; ns_threshold: 6 radix passes + 4
    assert got == {"logistic_target": 1, "logistic_ns_target": 1, "logistic_wf_move": 1, "logistic_ns_move": 1,
                   "logistic_logpyt": 1, "rw_propose": 1, "mh_accept": 1, "mh_accept_flags": 1,
                   "next_annealing_epn": 13, "rw_calibrate": 2, "wcov_sums": 1, "wcov_sums, mean": 1,
                   "chol_from_sums": 1, "essl_grid": 1, "ns_threshold": 10}


def test_binary_and_bank_keys(ctx):
    from particles_b200 import _lib
    L = ctx.lib
    pdim, n = 4, 8
    xtx, xty = buf(fill=0.0), buf(fill=0.1)
    xtx[: pdim * pdim: pdim + 1] = 1.0
    m = _lib.VsDesc(p=pdim, use_ldet=1, xtx=xtx.data_ptr(), xty=xty.data_ptr(), vm2=1.0, coef_len=-0.5,
                    coef_log=-0.5, coef_in_log=1.0, gw=1.0, lq=-1.0, l1q=-0.5)
    gam, err = buf(dtype=torch.uint8), buf(dtype=torch.int32)
    coeffs, edgy = buf(fill=0.1), buf(dtype=torch.uint8)
    a = [buf() for _ in range(8)]
    x1 = buf(dtype=torch.uint8)
    keys = buf(dtype=torch.int64)
    got = {
        "vs_loglik": launches(ctx, L.smcb_vs_loglik, C.byref(m), p(gam), n, pdim, 1.0, 1.0, *map(p, a[:6]), p(err)),
        "nested_logistic draw": launches(ctx, L.smcb_nested_logistic, pdim, p(coeffs), p(edgy), n, 1, p(x1), None,
                                         p(a[0])),
        "nested_logistic logpdf": launches(ctx, L.smcb_nested_logistic, pdim, p(coeffs), p(edgy), n, 0, p(gam),
                                           None, p(a[0])),
        "binary_wf_move": launches(ctx, L.smcb_binary_wf_move, C.byref(m), p(coeffs), p(edgy), n, 2, 1.0, p(gam),
                                   p(a[0]), p(a[1]), p(a[2]), None, None, p(x1), p(a[3]), p(a[4]), p(a[5]), p(a[6]),
                                   p(err)),
        "bank_keys": launches(ctx, L.smcb_bank_keys, p(keys), n, 1, 2),
    }
    assert set(got.values()) == {1}, got


def _int(v):
    return int(getattr(v, "value", v) or 0)


def expected_launches(name, args):
    """The kernels one call enqueues, from its arguments (calls on empty inputs launch nothing)."""
    from particles_b200 import _lib
    d = getattr(args[1], "_obj", None) if len(args) > 1 else None
    if name == "smcb_variance":
        return 1 if d.method == _lib.VAR_EVE else 4           # EVE: one kernel; SUMS: two passes + two finals
    if name == "smcb_bank_advance":
        return int((d.n_idx if d.idx else d.R) > 0)
    if name == "smcb_bank_gather":                           # fill, min, rows
        return 3 if _int(args[3]) > 0 and d.R > 0 else 0
    if name == "smcb_bank_merge":
        return int(d.R > 0)
    if name == "smcb_bank_keys":
        return int(_int(args[2]) > 0)
    if name == "smcb_csmc_run":
        return int(d.R > 0)
    if name in ("smcb_filter_step", "smcb_filter_step_timed"):     # init or step per step, then the tail
        n = _int(args[1])
        return n + 1 if n > 0 else 0
    if name == "smcb_filter_create":
        return 0
    return 1


class Recorder:
    """Replaces the bound C functions `names` by wrappers that record each call's arguments and the context's
    launch-count delta."""

    def __init__(self, ctx, names):
        self.ctx, self.names, self.calls = ctx, names, []

    def __enter__(self):
        lib, h = self.ctx.lib, self.ctx.handle
        self.saved = {nm: getattr(lib, nm) for nm in self.names}
        for nm, fn in self.saved.items():
            def wrap(*args, _fn=fn, _nm=nm):
                c0 = lib.smcb_launch_count(h)
                rc = _fn(*args)
                self.calls.append((_nm, args, lib.smcb_launch_count(h) - c0))
                return rc
            setattr(lib, nm, wrap)
        return self

    def __exit__(self, *exc):
        for nm, fn in self.saved.items():
            setattr(self.ctx.lib, nm, fn)

    def check(self):
        """Every recorded call launched what it should; returns {name: {descriptor method}} of the calls seen."""
        seen = {}
        for nm, args, d in self.calls:
            assert d == expected_launches(nm, args), (nm, d, args)
            desc = getattr(args[1], "_obj", None) if len(args) > 1 else None
            seen.setdefault(nm, set()).add(getattr(desc, "method", None))
        return seen


def _sv(T):
    from particles_b200 import state_space_models as ssm
    from oracle import smc_numpy as orc
    return ssm.Bootstrap(ssm=ssm.StochVol(), data=[np.atleast_1d(v) for v in orc.config2_data(T, 1)])


def test_descriptor_entry_points(ctx):
    import particles_b200 as pb
    from particles_b200 import hmm, kalman
    names = ["smcb_hmm", "smcb_kalman", "smcb_batch_run", "smcb_backward_sample"]
    rng = np.random.RandomState(0)
    with Recorder(ctx, names) as rec:
        bw = hmm.BaumWelch(hmm=hmm.GaussianHMM(trans_mat=np.array([[0.9, 0.1], [0.2, 0.8]]), mus=np.array([0.0, 1.0]),
                                               sigmas=np.ones(2)), data=rng.randn(10))
        bw.run()
        bw.sample(N=4)
        kf = kalman.Kalman(ssm=kalman.LinearGauss(), data=rng.randn(10))
        kf.filter()
        kf.smoother()
        pb.multiSMC(fk=_sv(10), N=128, nruns=2, collect="off")
        pf = pb.SMC(fk=_sv(10), N=128, store_history=True)
        pf.run()
        pf.hist.backward_sampling_ON2(8)
        torch.cuda.synchronize()
    assert set(rec.check()) == set(names)


def test_smoothing_and_variance_entry_points(ctx):
    import particles_b200 as pb
    from particles_b200 import _lib, kalman, collectors as cols, variance_estimators as ve
    from particles_b200 import state_space_models as ssm
    names = ["smcb_variance", "smcb_online_smooth", "smcb_two_filter"]
    T, N = 10, 256
    LG = type("LG", (kalman.LinearGauss,), {"add_func": lambda self, t, xp, x: 1.0 * x,
                                            "upper_bound_log_pt": lambda self, t: -0.5 * np.log(2.0 * np.pi)})
    model = LG(sigmaX=1.0, sigmaY=0.5, rho=0.9)
    _, y = model.simulate(T)
    with Recorder(ctx, names) as rec:
        pb.SMC(fk=_sv(T), N=N, collect=[ve.Var(), ve.Var_logLt()], seed=1).run()
        pb.SMC(fk=ssm.Bootstrap(ssm=model, data=y), N=N, collect=[cols.Paris(), cols.Online_smooth_ON2()],
               seed=2).run()
        lg = kalman.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9)
        pf = pb.SMC(fk=ssm.Bootstrap(ssm=lg, data=y), N=N, store_history=True, seed=3)
        pf.run()
        info = pb.SMC(fk=ssm.Bootstrap(ssm=lg, data=y[::-1]), N=N, store_history=True, seed=4)
        info.run()
        lgam = lambda x: -x * x / 2.0                                                      # noqa: E731
        pf.hist.two_filter_smoothing(2, info, lambda x, xf: x, lgam)
        pf.hist.two_filter_smoothing(2, info, lambda x, xf: x, lgam, linear_cost=True)
        torch.cuda.synchronize()
    seen = rec.check()
    assert seen == {"smcb_variance": {_lib.VAR_EVE, _lib.VAR_SUMS},
                    "smcb_online_smooth": {_lib.ONLINE_PARIS, _lib.ONLINE_ON2_W, _lib.ONLINE_PHI_PARIS,
                                           _lib.ONLINE_PHI_ON2},
                    "smcb_two_filter": {_lib.TF_ON2_ROWS, _lib.TF_ON_LOGW}}, seen


def test_bank_and_csmc_entry_points(ctx):
    import particles_b200 as pb
    from particles_b200 import distributions as dists, kalman, mcmc, smc_samplers as ss
    names = ["smcb_bank_keys", "smcb_bank_advance", "smcb_bank_gather", "smcb_bank_merge", "smcb_csmc_run"]

    class FixedTheta(mcmc.ParticleGibbs):
        def update_theta(self, theta, x):
            return theta

    th = dict(rho=0.9, sigmaX=1.0, sigmaY=0.5)
    _, y = kalman.LinearGauss(**th).simulate(10)
    y = np.array([float(v.reshape(-1)[0]) for v in y])
    with Recorder(ctx, names) as rec:
        torch.manual_seed(0)
        fk = ss.SMC2(ssm_cls=kalman.LinearGauss, prior=dists.StructDist({"sigmaY": dists.Gamma(a=2.0, b=4.0)}),
                     data=y, init_Nx=20)
        pb.SMC(fk=fk, N=64, seed=0).run()
        prior = dists.StructDist({k: dists.Normal(loc=v) for k, v in th.items()})
        theta0 = np.array([tuple(th.values())], dtype=[(k, float) for k in th])
        FixedTheta(niter=3, ssm_cls=kalman.LinearGauss, prior=prior, data=y, theta0=theta0, Nx=64, nchains=2,
                   seed=1).run()
        torch.cuda.synchronize()
    assert set(rec.check()) == set(names)


def test_filter_entry_points(ctx):
    """The fused filter: smcb_filter_step (init or step per step, then the tail), smcb_filter_step_timed, and the
    host-driven sharded path -- two ranks of one filter on this device, the all-gather done by a copy:
    step_local = init or step + publish, step_finish = the tail."""
    import particles_b200 as pb
    from particles_b200.core import _FusedEngine
    from particles_b200.parallel import ShardedFilter
    from particles_b200.state_space_models import fused_spec
    T = 6
    with Recorder(ctx, ["smcb_filter_create", "smcb_filter_step", "smcb_filter_step_timed"]) as rec:
        pf = pb.SMC(fk=_sv(T), N=4096, seed=0)
        assert pf.fused
        pf.run()
        eng = _FusedEngine(fused_spec(_sv(T)), 4096, "systematic", 0.5, 0)
        eng.step_timed(2)
        eng.step(3)
        torch.cuda.synchronize()
    assert set(rec.check()) == {"smcb_filter_create", "smcb_filter_step", "smcb_filter_step_timed"}

    spec = fused_spec(_sv(T))
    ranks = [ShardedFilter(spec, 2048, "systematic", 0.5, 0, r, 2, exchange="nccl") for r in range(2)]
    got = []
    for t in range(T):
        got += [launches(ctx, lambda h, f=f: ctx.lib.smcb_filter_step_local(f.handle)) for f in ranks]
        stats = torch.cat([f.local_stats for f in ranks])
        for f in ranks:
            f.gathered.copy_(stats)
        got += [launches(ctx, lambda h, f=f: ctx.lib.smcb_filter_step_finish(f.handle)) for f in ranks]
    assert got == [2, 2, 1, 1] * T, got
