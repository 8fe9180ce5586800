"""Nested sampling SMC on the device: the threshold step (smcb_ns_threshold) against np.percentile and a long-double
restatement, the constrained target and waste-free move against the high-precision replay of tests/sampler_replay.py,
whole runs against the live reference's runs (tests/golden/golden_nested.npz) and against adaptive tempering, the
generic ``StaticModel`` path against a closed-form evidence, and the paper's ``multiSMC`` call."""
import os

import numpy as np
import pytest
from scipy import stats

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import samplers_numpy as sp  # noqa: E402
import sampler_replay as sr  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SCALE = 5.0
LD = np.longdouble


def host(t):
    return t.detach().cpu().numpy()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.int64)


@pytest.fixture(scope="module")
def ctx():
    from particles_b200.device import context
    return context()


def lib_call(ctx, name, *args):
    from particles_b200 import _lib
    _lib.check(getattr(ctx.lib, name)(ctx.handle, *args))


def P(t):
    from particles_b200.device import ptr
    return ptr(t)


@pytest.fixture(scope="module")
def gn():
    return np.load(os.path.join(HERE, "golden", "golden_nested.npz"))


# ------------------------------------------------------------------------------------ smcb_ns_threshold
def lse_ld(v):
    """logsumexp in long double (scipy's shift: the maximum, or 0 when it is not finite); -inf for no entries."""
    v = np.asarray(v, dtype=np.float64)
    if v.size == 0:
        return LD(-np.inf)
    m = v.max()
    m = m if np.isfinite(m) else 0.0
    with np.errstate(divide="ignore"):
        return np.log(np.sum(np.exp(v.astype(LD) - LD(m)))) + LD(m)


def lsab_ld(a, b):
    with np.errstate(invalid="ignore"):
        a, b = LD(a), LD(b)
        return a + np.log1p(np.exp(b - a)) if a > b else b + np.log1p(np.exp(a - b))


def threshold_ld(llik, lt, t, alpha, log_evid):
    """(new_evid, new_evid_final) of nested.py:331-342 in long double, at the device's lt."""
    with np.errstate(invalid="ignore"):
        base = LD(t) * np.log(LD(alpha)) - np.log(LD(llik.size))
        return lsab_ld(log_evid, base + lse_ld(llik[llik <= lt])), lsab_ld(log_evid, base + lse_ld(llik))


def _threshold_inputs():
    r = np.random.RandomState(11)
    for n in (1, 2, 3, 1000, 100_003, 10_000_001):
        yield "normal", n, r.standard_normal(n) * 30.0 - 180.0
        if n > 10_000:
            continue
        yield "ties", n, np.round(r.standard_normal(n) * 2.0) - 50.0
        v = r.standard_normal(n) - 20.0
        v[: (n + 1) // 2] = -np.inf                        # a block of -inf, the lower half and then some
        yield "neginf-block", n, r.permutation(v)
        yield "equal", n, np.full(n, -7.5)
        yield "all-neginf", n, np.full(n, -np.inf)
        if n >= 3:
            v = np.where(r.rand(n) < 0.6, -0.0, r.standard_normal(n))          # a level at a block of -0.0
            yield "negzero", n, v
    for n in (1000, 100_003):
        # distinct values spread over several orders of magnitude below a tied maximum that holds the top 20 %: at
        # ESSrmin = 0.1 the level is that maximum, so no entry is above it and the stop must fire at any eps > 0 --
        # which needs both evidence sums to add these terms in the same order
        v = -100.0 - np.exp(r.uniform(-3.0, 4.0, n))
        v[r.rand(n) < 0.2] = -100.0
        yield "tied-max", n, v


THRESHOLD_CASES = [(name, n) for name, n, _ in _threshold_inputs()]


@pytest.mark.parametrize("name,n", THRESHOLD_CASES)
def test_threshold_vs_numpy(ctx, name, n):
    """lt has the bits of np.percentile (NaN when both order statistics are -inf); lw is 0 / -inf by llik > lt; the
    evidence terms are within 1e-13 relative of the long-double restatement; stop agrees with it away from the eps
    boundary, and an input with no entry above lt always stops; two calls give the same bits."""
    from particles_b200 import nested
    v = next(a for nm, k, a in _threshold_inputs() if (nm, k) == (name, n))
    llik = dev(v)
    alphas = (0.1, 0.5, 0.9) if n > 10_000 else (0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99)
    for alpha in alphas:
        for t, log_evid, eps in ((0, -np.inf, 0.01), (4, -150.25, 0.01), (9, -170.0, 1e-300)):
            lw, lt, new_evid, stop = nested.threshold(llik, alpha, t, log_evid, eps)
            with np.errstate(invalid="ignore"):
                want_lt = np.percentile(v, 100.0 * (1.0 - alpha))
            ev, ev_final = threshold_ld(v, want_lt, t, alpha, log_evid)
            with np.errstate(invalid="ignore"):
                diff = float(abs(ev - ev_final))
                want_stop = diff < eps
            if abs(diff - eps) > 1e-12 * max(1.0, abs(float(ev_final))):
                assert stop == want_stop, (alpha, t, diff, eps)
            if not np.any(v > want_lt) and not np.isnan(want_lt):
                assert stop, (alpha, t)
            if stop:
                assert lt == np.inf and np.all(host(lw) == 0.0)
                want = ev_final
            else:
                assert bits(lt) == bits(want_lt), (alpha, t, lt, want_lt)
                with np.errstate(invalid="ignore"):
                    assert np.array_equal(bits(host(lw)), bits(np.where(v > want_lt, 0.0, -np.inf)))
                want = ev
            if np.isnan(float(want)):
                assert np.isnan(new_evid)
            elif np.isinf(float(want)):
                assert new_evid == float(want)
            else:
                assert abs(LD(new_evid) - want) <= 1e-13 * abs(want), (alpha, t, new_evid, float(want))
            if name == "tied-max" and alpha == 0.1:
                assert want_lt == v.max() and stop, (t, eps)
            lw2, lt2, ne2, st2 = nested.threshold(llik, alpha, t, log_evid, eps)
            assert bits(lt2) == bits(lt) and bits(ne2) == bits(new_evid) and st2 == stop
            assert np.array_equal(bits(host(lw2)), bits(host(lw)))


def test_threshold_counts_launches_and_rejects_bad_statistics(ctx):
    from particles_b200 import _lib
    llik = dev(np.arange(10.0))
    lw, out = torch.empty(10, dtype=torch.float64, device="cuda"), torch.empty(3, dtype=torch.float64, device="cuda")
    before = ctx.launches
    lib_call(ctx, "smcb_ns_threshold", P(llik), 10, 4, 5, 0.5, 1, np.log(0.5), -3.0, 0.01, P(lw), P(out))
    assert ctx.launches - before == 10
    assert host(out)[0] == 4.5
    for k0, k1 in ((-1, 0), (9, 10), (3, 5), (5, 4)):
        with pytest.raises(ValueError, match="order statistics"):
            _lib.check(ctx.lib.smcb_ns_threshold(ctx.handle, P(llik), 10, k0, k1, 0.5, 1, 0.0, -3.0, 0.01, P(lw),
                                                 P(out)))


# ------------------------------------------------------------------------------------ constrained target and move
def ns_raw(ctx, entry, theta0, lpr0, ll0, lp0, data_dev, n_rows, scale, lmin, L, P_, z=None, u=None):
    M, d = theta0.shape
    out = [torch.empty((P_ * M, d), dtype=torch.float64, device="cuda")] + [
        torch.empty(P_ * M, dtype=torch.float64, device="cuda") for _ in range(3)]
    pb = torch.empty((P_ - 1, M), dtype=torch.float64, device="cuda")
    lib_call(ctx, entry, M, d, P_, P(theta0), P(lpr0), P(ll0), P(lp0), P(data_dev), n_rows, scale, lmin, P(L), P(z),
             P(u), *[P(t) for t in out], P(pb))
    th, lpr, ll, lp = (host(t) for t in out)
    rows = [{"theta": th[s * M:(s + 1) * M], "lprior": lpr[s * M:(s + 1) * M], "llik": ll[s * M:(s + 1) * M],
             "lpost": lp[s * M:(s + 1) * M]} for s in range(P_)]
    return rows, host(pb)


def check_ns_generation(s, prev, out, pb, z, u, L, data, scale, lmin, d, z_rel):
    """Generation s of the constrained move from the kernel's own row s - 1, as sampler_replay.check_generation does
    for the tempered one: the long-double proposal and target, a floor decision wherever |llik' - lmin| exceeds the
    likelihood's bound, then the Metropolis decision on lprior' - lprior (-inf below the floor).  Returns the masks
    (accepted, rejected at the floor, rejected above it, decided)."""
    D = sr.tier(d)
    prop, bprop = sr.propose_ld(prev["theta"], z, L)
    bprop = bprop + sr.propose_bound_z(z, L, z_rel)
    propf = prop.astype(np.float64)
    (lp, ll, _), (bp, bl, _) = sr.target_bounds(propf, data, scale, 0.0, D, D // 2 + 1, data.shape[0] + 4)
    absx = np.abs(np.asarray(data, np.float64)).sum(axis=0)
    with np.errstate(invalid="ignore", over="ignore"):
        bp = bp + ((np.abs(propf) + bprop) / scale ** 2 * bprop).sum(axis=1)
        bl = bl + (absx[None, :] * bprop).sum(axis=1)
        above = ll >= LD(lmin)
        floor_decided = ~(np.abs((ll - LD(lmin)).astype(np.float64)) <= bl)
        post = np.where(above, lp, LD(-np.inf))
        lp_acc = post - np.asarray(prev["lpost"], np.float64).astype(LD)
        tol = bp + sr.U * np.abs(lp_acc.astype(np.float64)) + 2 * sr.EPS
    tol = np.where(np.isfinite(tol), tol, np.inf)
    acc, decided = sr.decisions(u, lp_acc, tol)
    decided = decided & floor_decided
    same = np.all(out["theta"] == prev["theta"], axis=1)
    for k in ("lprior", "llik", "lpost"):                # a rejected chain's row s: row s - 1, bit for bit
        assert np.array_equal(bits(out[k][same]), bits(prev[k][same])), (s, k)
    dev_acc = ~same
    flip = decided & (acc != dev_acc)
    assert not flip.any(), (s, int(np.flatnonzero(flip)[0]), int(flip.sum()))
    A = dev_acc
    if A.any():
        sr.assert_close(f"generation {s}: accepted theta", out["theta"][A], prop[A], bprop[A], "chain")
        sr.assert_close(f"generation {s}: accepted lprior", out["lprior"][A], lp[A], bp[A], "chain")
        sr.assert_close(f"generation {s}: accepted llik", out["llik"][A], ll[A], bl[A], "chain")
        assert np.array_equal(bits(out["lpost"][A]), bits(out["lprior"][A]))     # above the floor: lpost = lprior
        assert np.all(out["llik"][A] >= lmin)
    floor_rej = decided & ~above & ~dev_acc
    assert np.all(pb[floor_rej] == 0.0)                  # below the floor: pb = 0 whatever u is
    want = sr.pb_ld(lp_acc)
    with np.errstate(invalid="ignore", over="ignore"):
        bpb = np.abs(want.astype(np.float64)) * np.expm1(np.minimum(tol, 700.0)) + sr.EPS
    ok = floor_decided
    sr.assert_close(f"generation {s}: pb", pb[ok], want[ok], bpb[ok], "chain")
    return dev_acc, floor_rej, decided & above & ~dev_acc, decided


def lower_factor(d, seed, scale):
    r = np.random.RandomState(seed)
    return scale * (np.tril(r.randn(d, d) * 0.2) + np.diag(1.0 + r.rand(d)))


def run_ns_move(ctx, d, M, P_, n_rows, mode, seed, expect):
    """Starting points resampled above a floor at the median of their log-likelihoods (as NS-SMC's are), a factor
    wide enough that proposals fall on both sides of it, and a prior as narrow as the likelihood so that the prior
    ratio rejects some proposals above the floor; every generation replayed."""
    from particles_b200 import smc_samplers as ssp
    assert sr.wf_resident(d, n_rows) == (expect == "resident"), (d, n_rows)
    data = sp.synthetic_logistic(n_rows, d, seed=seed)
    r = np.random.RandomState(seed + 1)
    sigma = 1.0 / np.sqrt(n_rows * 0.15 + 1.0 / SCALE ** 2)
    cand = r.randn(d) * sigma * 0.5 + r.randn(4 * M + 8, d) * sigma
    scale = sigma
    model = ssp.LogisticRegression(data=data, prior_scale=scale)
    x = ssp.ThetaParticles(theta=dev(cand))
    model.target(x, 0.0, lmin=-np.inf)
    ll0 = host(x.llik)
    lmin = float(np.median(ll0))
    keep = np.flatnonzero(ll0 > lmin)
    theta0 = cand[keep[r.randint(0, keep.size, M)]]
    x = ssp.ThetaParticles(theta=dev(theta0))
    model.target(x, 0.0, lmin=lmin)
    assert np.array_equal(bits(host(x.lpost)), bits(host(x.lprior)))
    L = lower_factor(d, seed, 1.5 * sigma / np.sqrt(d))
    Ld = dev(L)
    args = (x.theta, x.lprior, x.llik, x.lpost, model.data, n_rows, scale)
    if mode == "injected":
        z, u = r.standard_normal((P_ - 1, M, d)), r.rand(P_ - 1, M)
        rows, pb = ns_raw(ctx, "smcb_logistic_ns_move", *args, lmin, Ld, P_, dev(z), dev(u))
        zs, us, zrel = list(z), list(u), 0.0
        # lmin = -inf: the bits of the tempered move at epn = 0
        r1, pb1 = ns_raw(ctx, "smcb_logistic_ns_move", *args, -np.inf, Ld, P_, dev(z), dev(u))
        r2, pb2 = ns_raw(ctx, "smcb_logistic_wf_move", *args, 0.0, Ld, P_, dev(z), dev(u))
    else:
        key = 0x4E530000 + seed
        ctx.seed(key)
        ns_raw(ctx, "smcb_logistic_ns_move", *args, lmin, Ld, P_)               # call 0
        rows, pb = ns_raw(ctx, "smcb_logistic_ns_move", *args, lmin, Ld, P_)    # call 1
        zs = [sr.wf_normals(M, d, s, 1, key) for s in range(1, P_)]
        us = [sr.wf_uniforms(M, s, 1, key) for s in range(1, P_)]
        zrel = sr.Z_REL
        ctx.seed(key)
        r1, pb1 = ns_raw(ctx, "smcb_logistic_ns_move", *args, -np.inf, Ld, P_)
        ctx.seed(key)
        r2, pb2 = ns_raw(ctx, "smcb_logistic_wf_move", *args, 0.0, Ld, P_)
    assert np.array_equal(bits(pb1), bits(pb2))
    for a, b in zip(r1, r2):
        for k in a:
            assert np.array_equal(bits(a[k]), bits(b[k])), k
    assert np.array_equal(rows[0]["theta"], theta0)
    n_acc = n_floor = n_rej = n_dec = 0
    for s in range(1, P_):
        acc, floor_rej, rej, decided = check_ns_generation(s, rows[s - 1], rows[s], pb[s - 1], zs[s - 1], us[s - 1], L,
                                                           data, scale, lmin, d, zrel)
        n_acc += int(acc.sum())
        n_floor += int(floor_rej.sum())
        n_rej += int(rej.sum())
        n_dec += int(decided.sum())
    total = M * (P_ - 1)
    assert n_dec >= total - max(1, total // 1000)
    assert n_acc > 0 and n_floor > 0 and n_rej > 0, (n_acc, n_floor, n_rej, total)


NS_MOVE_CASES = [(D, branch) for D in sr.TIERS for branch in ("resident", "streamed")]


@pytest.mark.parametrize("mode", ["injected", "device"])
@pytest.mark.parametrize("D,branch", NS_MOVE_CASES)
def test_ns_move_vs_replay(ctx, D, branch, mode):
    """Each tier at its largest d, data resident (n_rows = tile_rows(D)) and streamed with a partial last tile; 65
    chains (three CTAs), P = 9: floor rejections, ordinary accepts and ordinary rejections all occur."""
    t = sr.tile_rows(D)
    n_rows = t if branch == "resident" else int(2.5 * t) + 7
    run_ns_move(ctx, D, 65, 9, n_rows, mode, seed=D * 10 + len(branch), expect=branch)
    assert sr.wf_grid(65) == 3


@pytest.mark.parametrize("d,n", [(1, 257), (4, 1), (9, 100_003), (20, 513), (32, 257)])
def test_ns_target_vs_replay(ctx, d, n):
    """lprior / llik as the tempered target's, lpost = lprior where llik >= lmin and -inf elsewhere (decided where
    the margin exceeds the bound); lmin = -inf gives the bits of smcb_logistic_target at epn = 0."""
    from particles_b200 import smc_samplers as ssp
    data = sp.synthetic_logistic(41, d, seed=d)
    r = np.random.RandomState(d + n)
    theta = r.randn(n, d) * 0.7
    model = ssp.LogisticRegression(data=data, prior_scale=SCALE)
    a = ssp.ThetaParticles(theta=dev(theta))
    b = ssp.ThetaParticles(theta=dev(theta))
    model.target(a, 0.0, lmin=-np.inf)
    model.target(b, 0.0)
    for k in ("lprior", "llik", "lpost"):
        assert np.array_equal(bits(host(getattr(a, k))), bits(host(getattr(b, k)))), k
    lmin = float(np.median(host(a.llik)))
    model.target(a, 0.0, lmin=lmin)
    (lp, ll, _), (bp, bl, _) = sr.target_bounds(theta, data, SCALE, 0.0, sr.tier(d), sr.tier(d), data.shape[0])
    sr.assert_close("lprior", host(a.lprior), lp, bp)
    sr.assert_close("llik", host(a.llik), ll, bl)
    assert np.array_equal(bits(host(a.lprior)), bits(host(b.lprior)))
    assert np.array_equal(bits(host(a.llik)), bits(host(b.llik)))
    got = host(a.lpost)
    above = host(a.llik) >= lmin
    assert np.array_equal(bits(got[above]), bits(host(a.lprior)[above]))
    assert np.all(got[~above] == -np.inf)
    assert n == 1 or 0 < above.sum() < n


# ------------------------------------------------------------------------------------ whole runs
def ns_runs(data, wastefree, lc, N, alpha, seeds):
    import particles_b200 as pb
    from particles_b200 import nested
    from particles_b200 import smc_samplers as ssp
    out = []
    for s in seeds:
        fk = nested.NestedSamplingSMC(model=ssp.LogisticRegression(data=data), wastefree=wastefree, len_chain=lc,
                                      ESSrmin=alpha)
        pf = pb.SMC(fk=fk, N=N, seed=s)
        pf.run()
        lts, ev = pf.X.shared["lts"], pf.X.shared["log_evid"]
        assert lts[-1] == np.inf and len(lts) == len(ev) == pf.t + 1
        assert np.all(np.diff(lts) >= 0.0), lts
        assert pf.X.N == N * (lc if wastefree else 1)
        out.append(ev[-1])
    return np.array(out)


@pytest.mark.parametrize("wastefree", [True, False])
def test_whole_runs_vs_reference_and_tempering(gn, wastefree):
    """12 seeds of device NS-SMC (one-launch waste-free move, or the standard move: proposal, constrained target,
    accept) on the data of the reference's anchors: the mean log-evidence is within the combined 3 sigma of the
    reference's NS-SMC runs and of the device's AdaptiveTempering on the same model."""
    import particles_b200 as pb
    from particles_b200 import smc_samplers as ssp
    data = gn["stat/data"]
    N, lc = (int(v) for v in gn["stat/meta"][:2])
    alpha = float(gn["stat/meta"][2])
    ref = gn["stat/ns_log_evid"]
    R = 12
    if wastefree:
        ev = ns_runs(data, True, lc, N, alpha, range(500, 500 + R))
    else:
        ev = ns_runs(data, False, 10, N * lc, alpha, range(600, 600 + R))
    tls = []
    for s in range(R):
        tp = pb.SMC(fk=ssp.AdaptiveTempering(model=ssp.LogisticRegression(data=data), len_chain=lc, ESSrmin=alpha),
                    N=N, seed=700 + s)
        tp.run()
        tls.append(tp.logLt)
    tls = np.array(tls)
    comb = np.sqrt(ev.var(ddof=1) / R + ref.var(ddof=1) / ref.size)
    assert abs(ev.mean() - ref.mean()) < 3 * comb + 1e-6, (ev.mean(), ref.mean(), comb)
    comb = np.sqrt(ev.var(ddof=1) / R + tls.var(ddof=1) / R)
    assert abs(ev.mean() - tls.mean()) < 3 * comb + 1e-6, (ev.mean(), tls.mean(), comb)


# ------------------------------------------------------------------------------------ plugin path
def test_linear_regression_static_model_vs_closed_form():
    """A conjugate linear regression through the generic StaticModel path (user logpyt on CUDA tensors): T = 30,
    d = 3, sigma = 0.1, prior scale 10.  Over 12 seeds the mean NS-SMC log-evidence is within 3 sigma (+ the Jensen
    bias sd^2 / 2) of the closed form."""
    import particles_b200 as pb
    from particles_b200 import distributions as dists
    from particles_b200 import nested
    from particles_b200 import smc_samplers as ssp
    T, d, sig, scale = 30, 3, 0.1, 10.0
    r = np.random.RandomState(0)
    preds = r.randn(T, d)
    preds[:, 0] = 1.0
    response = preds @ np.array([0.3, 1.0, -0.2]) + sig * r.randn(T)
    data = np.empty((T, d + 1))
    data[:, 0], data[:, 1:] = response, preds
    evid = stats.multivariate_normal.logpdf(response, cov=sig ** 2 * np.eye(T) + scale ** 2 * preds @ preds.T)

    class LinearRegression(ssp.StaticModel):
        def logpyt(self, theta, t):
            lin = theta["beta"] @ self.data[t, 1:]
            return -0.5 * ((self.data[t, 0] - lin) / sig) ** 2 - np.log(sig) - 0.5 * np.log(2 * np.pi)

    prior = dists.StructDist({"beta": dists.MvNormal(scale=scale, cov=np.eye(d))})
    R, evs = 12, []
    for s in range(R):
        fk = nested.NestedSamplingSMC(model=LinearRegression(data=data, prior=prior), len_chain=20, ESSrmin=0.5)
        pf = pb.SMC(fk=fk, N=200, seed=800 + s)
        pf.run()
        assert pf.X.shared["lts"][-1] == np.inf and pf.X.theta.shape == (4000, d)
        evs.append(pf.X.shared["log_evid"][-1])
    evs = np.array(evs)
    sd = evs.std(ddof=1)
    assert abs(evs.mean() - evid) < 3 * sd / np.sqrt(R) + 0.5 * sd ** 2, (evs.mean(), evid, sd)


def logistic_static_model(data, scales):
    """The paper's model (papers/nested/tempering_vs_nested_logistic.py) as a StaticModel on CUDA tensors."""
    from particles_b200 import distributions as dists
    from particles_b200 import smc_samplers as ssp
    p = data.shape[1]

    class LogisticRegression(ssp.StaticModel):
        def logpyt(self, theta, t):
            lin = theta["beta"] @ self.data[t, :]
            return -torch.logaddexp(torch.zeros_like(lin), -lin)

    prior = dists.StructDist({"beta": dists.MvNormal(scale=scales, cov=np.eye(p))})
    return LogisticRegression(data=data, prior=prior)


def test_logistic_static_model_agrees_with_device_likelihood():
    """The logistic model written as a StaticModel (prior scale 5) and LogisticRegression on the same data: their
    NS-SMC log-evidence means over 12 seeds each agree within the combined 3 sigma."""
    import particles_b200 as pb
    from particles_b200 import nested
    data = sp.synthetic_logistic(100, 4, seed=9)
    R = 12
    evs = []
    for s in range(R):
        fk = nested.NestedSamplingSMC(model=logistic_static_model(data, 5.0), len_chain=10, ESSrmin=0.5)
        pf = pb.SMC(fk=fk, N=100, seed=900 + s)
        pf.run()
        evs.append(pf.X.shared["log_evid"][-1])
    evs = np.array(evs)
    dv = ns_runs(data, True, 10, 100, 0.5, range(950, 950 + R))
    comb = np.sqrt(evs.var(ddof=1) / R + dv.var(ddof=1) / R)
    assert abs(evs.mean() - dv.mean()) < 3 * comb + 1e-6, (evs.mean(), dv.mean(), comb)


def test_paper_multismc_call():
    """papers/nested/tempering_vs_nested_logistic.py at small sizes: multiSMC over {'nested', 'tempering'} with the
    paper's out_func; one dict per run with the reference's keys, the fk keys, and the out_func values (NS-SMC reads
    log_evid, tempering falls back to logLt).  Tempering needs the device likelihood (``LogisticRegression``, prior
    scale 5), so both samplers run on it here; the paper's own model (intercept scale 20) runs NS-SMC on the
    StaticModel path through the same call."""
    import particles_b200 as pb
    from particles_b200 import nested
    from particles_b200 import smc_samplers as ssp
    data = sp.synthetic_logistic(60, 3, seed=2)
    T, p = data.shape
    lc, N, nruns = 5, 50, 2

    def out_func(pf):
        try:
            est = pf.X.shared["log_evid"][-1]
        except (KeyError, IndexError):
            est = pf.logLt
        return {"nevals": N * ((lc - 1) * pf.t + 1), "est": est, "t": pf.t}

    model = ssp.LogisticRegression(data=data, prior_scale=5.0)
    for a in (0.3, 0.7):
        fks = {"nested": nested.NestedSamplingSMC(model=model, len_chain=lc, ESSrmin=a),
               "tempering": ssp.AdaptiveTempering(model=model, len_chain=lc, ESSrmin=a)}
        np.random.seed(3)
        res = pb.multiSMC(fk=fks, N=N, verbose=False, nruns=nruns, out_func=out_func, nprocs=0)
        assert len(res) == 2 * nruns
        assert sorted(r["fk"] for r in res) == ["nested"] * nruns + ["tempering"] * nruns
        for r in res:
            assert set(r) == {"run", "fk", "seed", "nevals", "est", "t"}, set(r)
            assert np.isfinite(r["est"]) and r["nevals"] == N * ((lc - 1) * r["t"] + 1)
        ests = {k: [r["est"] for r in res if r["fk"] == k] for k in ("nested", "tempering")}
        assert abs(np.mean(ests["nested"]) - np.mean(ests["tempering"])) < 2.0, ests
    scales = 5.0 * np.ones(p)
    scales[0] = 20.0
    fks = {"nested": nested.NestedSamplingSMC(model=logistic_static_model(data, scales), len_chain=lc, ESSrmin=0.5)}
    res = pb.multiSMC(fk=fks, N=N, verbose=False, nruns=nruns, out_func=out_func, nprocs=0)
    assert [r["fk"] for r in res] == ["nested"] * nruns
    assert all(np.isfinite(r["est"]) and r["t"] > 1 for r in res)
