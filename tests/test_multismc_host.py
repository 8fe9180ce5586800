"""multiSMC on the host: the multiplexer against the live reference's output structure (golden_multismc.json,
tests/golden/make_golden_multismc.py), and the routing of runs into batched groups or the per-run path."""
import json
import os

import numpy as np
import pytest

from particles_b200 import utils

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_multismc.json")


def fake(**kw):
    return ";".join(f"{k}={kw[k]!r}" for k in sorted(kw))


def fake_dict(**kw):
    return {"n_args": len(kw), "N2": 2 * kw.get("N", 0)}


def as_pairs(res):
    out = []
    for d in res:
        out.append([[k, int(v) if isinstance(v, np.integer) else v] for k, v in d.items()])
    return out


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", ["lists_dicts", "one_run", "one_run_seeded", "dict_result", "no_seeding",
                                  "collect_protected"])
def test_multiplexer_matches_reference(golden, case):
    g = golden[case]
    np.random.seed(g["seed"])
    res = utils.multiplexer(f={"fake": fake, "fake_dict": fake_dict}[g["f"]], protected_args=g["protected"],
                            **g["kwargs"])
    assert as_pairs(res) == g["result"]


@pytest.mark.parametrize("case,of", [("multismc_float", lambda kw: float(5)),
                                     ("multismc_dict", lambda kw: {"t": 5, "N": kw["N"]})])
def test_multismc_structure_matches_reference(golden, case, of):
    """multiSMC seeds every run (also nruns = 1) and protects ``collect``: the same structure from the expansion
    multiSMC uses, with a stand-in for the runs."""
    g = golden[case]
    np.random.seed(g["seed"])
    inputs, outputs = utils.expand(nruns=2, seeding=True, protected_args={"collect": None}, fk={"boot": object()},
                                   N=[20, 30])
    res = [utils.add_to_dict(op, of(ip)) for ip, op in zip(inputs, outputs)]
    assert as_pairs(res) == g["result"]
    np.random.seed(golden["multismc_one_run"]["seed"])
    inputs, outputs = utils.expand(nruns=1, seeding=True, protected_args={"collect": None}, fk=object(), N=20)
    res = [utils.add_to_dict(op, 5) for op in outputs]
    assert as_pairs(res) == golden["multismc_one_run"]["result"]


def test_multiplexer_rejects_missing_function():
    with pytest.raises(TypeError):
        utils.multiplexer(f=None, N=[1])


def sv_data(T):
    return [np.array([0.1 * np.sin(t)]) for t in range(T)]


def test_grouping():
    """Which runs share a batched launch, and which take the per-run path."""
    from particles_b200 import collectors as col, core, kalman, state_space_models as ssm
    y = sv_data(20)
    boot = lambda m: ssm.Bootstrap(ssm=m, data=y)          # noqa: E731
    k1, _ = core.batch_key(dict(fk=boot(ssm.StochVol()), N=1000))
    k2, _ = core.batch_key(dict(fk=boot(ssm.StochVol(mu=-0.5, rho=0.9)), N=1000, ESSrmin=0.3))
    assert k1 is not None and k1 == k2                       # other constants / ESSrmin: same launch
    assert core.batch_key(dict(fk=boot(ssm.StochVol()), N=2000))[0] != k1
    assert core.batch_key(dict(fk=boot(ssm.StochVol()), N=1000, resampling="stratified"))[0] != k1
    assert core.batch_key(dict(fk=ssm.GuidedPF(ssm=ssm.StochVol(), data=y), N=1000))[0] != k1
    assert core.batch_key(dict(fk=boot(kalman.LinearGauss()), N=1000))[0] != k1
    km = core.batch_key(dict(fk=boot(ssm.StochVol()), N=1000, collect=[col.Moments()]))[0]
    assert km is not None and km != k1
    assert core.batch_key(dict(fk=boot(ssm.StochVol()), N=1000, collect="off"))[0] not in (None, k1)

    class Toy(ssm.StateSpaceModel):
        def PX0(self):
            return None

    per_run = [dict(fk=boot(ssm.StochVol()), N=1000, resampling="residual"),
               dict(fk=boot(ssm.StochVol()), N=1000, store_history=True),
               dict(fk=boot(ssm.StochVol()), N=1000, verbose=True),
               dict(fk=boot(Toy()), N=1000),
               dict(fk=boot(ssm.StochVol()), N=1000, collect=[col.Paris()]),
               dict(fk=boot(ssm.StochVol()), N=1000, collect=[col.Moments(mom_func=lambda W, X: 0.0)]),
               dict(fk=boot(ssm.BearingsOnly()), N=1000)]
    for kw in per_run:
        assert core.batch_key(kw) == (None, None), kw


def test_batch_routing_rule():
    """The routing rule reproduces the verdicts measured on an H100 (tools/bench_multismc.py --crossover): batched at
    small N whatever R, per run for a handful of runs that each fill a large share of the GPU."""
    from particles_b200 import _lib, core
    res, st = _lib.BATCH_RESIDENT, _lib.BATCH_STREAMING
    assert core.batch_pays(256, 1, res, 396) and core.batch_pays(4096, 1, res, 132)
    # (N, R, grid, batched faster as measured)
    for N, R, grid, faster in [(16384, 16, 16, True), (65536, 8, 8, False), (65536, 32, 32, True),
                               (65536, 128, 128, True), (131072, 32, 32, True), (131072, 132, 132, True),
                               (262144, 64, 64, True), (262144, 396, 396, True), (1048576, 132, 132, True),
                               (16384, 611, 396, True), (65536, 153, 153, True)]:
        assert core.batch_pays(N, R, st, grid) == faster, (N, R)
    assert not core.batch_pays(65536, 10, st, 10) and not core.batch_pays(10 ** 7, 2, st, 2)
    assert core.loop_step_s(10 ** 9) == pytest.approx(core.LOOP_STEP[-1][1])
    assert core.loop_step_s(1) == pytest.approx(core.LOOP_STEP[0][1])
