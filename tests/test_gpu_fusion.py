"""Fused pairs of streaming steps (SMCB_FUSE): a launch that runs step t and step t + 1 in one pass over the
particles, and the launch t + 1 that finds its step done or overwrites it, must leave exactly what two unfused
launches leave -- summaries, moments, both particle and log-weight buffers, ancestors -- bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def host(t):
    return t.detach().cpu().numpy()


def models():
    from particles_b200 import kalman, state_space_models as ssm
    return {"sv": (ssm.StochVol(), "data/sv_seed1_T1000"),
            "lg": (kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), "data/lg_seed2_T100"),
            "gordon": (ssm.Gordon_etal(), "data/gordon_seed3_T50")}


FK = {"boot": "Bootstrap", "guided": "GuidedPF", "apf": "AuxiliaryPF", "auxboot": "AuxiliaryBootstrap"}


def make_spec(golden, mname, fkname, T):
    from particles_b200 import state_space_models as ssm
    model, dkey = models()[mname]
    y = [np.atleast_1d(v) for v in golden[dkey][:T]]
    spec = ssm.fused_spec(getattr(ssm, FK[fkname])(ssm=model, data=y))
    assert spec is not None
    return spec


def run(monkeypatch, spec, N, scheme, essrmin, mode, batches, moments=False, noise=None, seed=31):
    """One fused filter made with SMCB_FUSE=mode, stepped in `batches`; its outputs and fusion counters."""
    from particles_b200.core import _FusedEngine
    monkeypatch.setenv("SMCB_FUSE", str(mode))
    e = _FusedEngine(spec, N, scheme, essrmin, seed, noise=noise, moments=moments)
    e.A.zero_()                     # written by resampling steps only
    for b in batches:
        e.step(b)
    torch.cuda.synchronize()
    out = {"summ": e.summ.clone(), "X0": e.X[0].clone(), "X1": e.X[1].clone(), "lw0": e.lw[0].clone(),
           "lw1": e.lw[1].clone(), "A": e.A.clone()}
    if moments:
        out["mom"] = e.mom.clone()
    stats = e.fusion_stats()
    e.close()
    return out, stats


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs"


def check_counters(stats, out, N, essrmin, mode, batches):
    """The device counters agree with the host replay of the predictor on the run's own summaries."""
    from particles_b200.core import fusion_schedule
    kinds = fusion_schedule(host(out["summ"]), N, essrmin, mode, batches)
    assert stats == {k: kinds.count(k) for k in ("fused", "noop", "mispredicted")}
    assert kinds.count("fused") == kinds.count("noop") + kinds.count("mispredicted")
    return kinds


CASES = [   # model, Feynman-Kac kind, scheme, ESSrmin, N, moments
    ("sv", "boot", "systematic", 0.5, 2000, False),
    ("sv", "boot", "stratified", 0.5, 2049, True),
    ("sv", "boot", "multinomial", 0.5, 1_000_000, False),
    ("sv", "boot", "systematic", 0.0, 2049, False),
    ("sv", "boot", "stratified", 1.0, 2000, True),
    ("sv", "guided", "multinomial", 0.5, 2049, False),
    ("sv", "apf", "systematic", 0.5, 2000, True),
    ("sv", "apf", "stratified", 0.5, 1_000_000, False),
    ("sv", "auxboot", "multinomial", 0.0, 2049, False),
    ("lg", "boot", "multinomial", 0.5, 2049, True),
    ("lg", "guided", "systematic", 0.5, 1_000_000, True),
    ("lg", "apf", "stratified", 1.0, 2049, False),
    ("gordon", "boot", "stratified", 0.5, 2000, False),
    ("gordon", "boot", "systematic", 0.5, 1_000_000, True),
]


@pytest.mark.parametrize("mname,fkname,scheme,essrmin,N,moments", CASES)
def test_fused_pairs_bit_identical(golden, monkeypatch, mname, fkname, scheme, essrmin, N, moments):
    T = 40
    spec = make_spec(golden, mname, fkname, T)
    ref, st0 = run(monkeypatch, spec, N, scheme, essrmin, 0, [T], moments)
    assert st0 == {"fused": 0, "noop": 0, "mispredicted": 0}
    rs_ = host(ref["summ"])[:, 2] != 0
    streaming = not rs_[1:T - 1].all()           # some launch before the last one may fuse
    for mode in (1, 2):
        out, st = run(monkeypatch, spec, N, scheme, essrmin, mode, [T], moments)
        assert_same(out, ref)
        check_counters(st, out, N, essrmin, mode, [T])
        if streaming and (mode == 2 or essrmin == 0.0):      # (mode 1: the predictor may decline every pair)
            assert st["fused"] > 0
    # the recovery path for certain: a batch that starts at launch q - 1, the streaming step before a resampling
    # step q, so that SMCB_FUSE=2 pre-computes step q there
    q = next((t for t in range(2, T) if rs_[t] and not rs_[t - 1]), None)
    if q is not None:
        out, st = run(monkeypatch, spec, N, scheme, essrmin, 2, [q - 1, T - q + 1], moments)
        assert_same(out, ref)
        check_counters(st, out, N, essrmin, 2, [q - 1, T - q + 1])
        assert st["mispredicted"] > 0


@pytest.mark.parametrize("mode", [1, 2])
def test_fused_pairs_respect_batches(golden, monkeypatch, mode):
    """A pair never reaches past the steps a step() call asked for: 7 + 5 + 1 steps == 13 steps in one call, and
    the caller sees the same buffers (Xp included) after every call."""
    T, N = 13, 2049
    spec = make_spec(golden, "sv", "boot", T)
    ref, _ = run(monkeypatch, spec, N, "systematic", 0.5, 0, [7, 5, 1])
    one, _ = run(monkeypatch, spec, N, "systematic", 0.5, mode, [T])
    split, st = run(monkeypatch, spec, N, "systematic", 0.5, mode, [7, 5, 1])
    assert_same(one, ref)
    assert_same(split, ref)
    kinds = check_counters(st, split, N, 0.5, mode, [7, 5, 1])
    assert kinds[5] != "fused" and kinds[10] != "fused"          # launches 6 and 11 end their batch
    for b in ([6], [6, 1], [7, 2]):                               # stop after an odd or an even step
        part, _ = run(monkeypatch, spec, N, "systematic", 0.5, mode, b)
        stop, _ = run(monkeypatch, spec, N, "systematic", 0.5, 0, b)
        assert_same(part, stop)


@pytest.mark.parametrize("scheme", ["systematic", "multinomial"])
def test_fused_pairs_injected_noise(golden, monkeypatch, scheme):
    """Injected normals are read at step t + 1's offset by the second half of a pair."""
    T, N = 30, 2049
    spec = make_spec(golden, "sv", "guided", T)
    r = np.random.RandomState(5)
    noise = (r.standard_normal((T, N)), r.rand(T, N + 1))
    ref, _ = run(monkeypatch, spec, N, scheme, 0.5, 0, [T], noise=noise)
    for mode in (1, 2):
        out, st = run(monkeypatch, spec, N, scheme, 0.5, mode, [T], noise=noise)
        assert_same(out, ref)
        assert st["fused"] > 0
