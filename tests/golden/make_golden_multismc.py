"""The output STRUCTURE of the live reference's ``multiplexer`` / ``multiSMC`` (particles/utils.py, core.py): key
order, ``'run'``, labels of dict-valued arguments, ``'seed'`` values after ``np.random.seed``, and the merging of dict
results.  tests/test_multismc_host.py replays every case through ``particles_b200.utils`` with the same fake run
function and compares.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_multismc.py

Writes tests/golden/golden_multismc.json."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, "/root/reference")
import particles  # noqa: E402
from particles import state_space_models as ssms  # noqa: E402
from particles import utils  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def fake(**kw):
    """A deterministic stand-in for one run: a string of its arguments."""
    return ";".join(f"{k}={kw[k]!r}" for k in sorted(kw))


def fake_dict(**kw):
    return {"n_args": len(kw), "N2": 2 * kw.get("N", 0)}


def plain(v):
    if isinstance(v, (np.integer,)):
        return int(v)
    if isinstance(v, (np.floating,)):
        return float(v)
    return v


def record(res):
    return [[[k, plain(v)] for k, v in d.items()] for d in res]


# name -> (np seed, fake function name, multiplexer keyword arguments); "collect" goes to protected_args
CASES = {
    "lists_dicts": (1, "fake", dict(nruns=3, N=[10, 20], resampling=["systematic", "multinomial"],
                                    fk={"a": 1, "b": 2}, ESSrmin=0.5, collect=[1, 2])),
    "one_run": (2, "fake", dict(nruns=1, N=[10, 20], fk={"x": 7})),
    "one_run_seeded": (3, "fake", dict(nruns=1, seeding=True, N=100)),
    "dict_result": (4, "fake_dict", dict(nruns=2, N=[5, 6], verbose=False)),
    "no_seeding": (5, "fake", dict(nruns=4, seeding=False, N=[1, 2])),
    "collect_protected": (6, "fake", dict(nruns=2, collect=["c0", "c1", "c2"], resampling=["stratified"])),
}


def main():
    out = {}
    for name, (seed, fname, kw) in CASES.items():
        kw = dict(kw)
        protected = {"collect": kw.pop("collect")} if "collect" in kw else None
        np.random.seed(seed)
        res = utils.multiplexer(f=globals()[fname], protected_args=None if protected is None else dict(protected),
                                **kw)
        out[name] = {"seed": seed, "f": fname, "kwargs": kw, "protected": protected, "result": record(res)}
    # multiSMC itself (always seeds, collect protected, out_func float / dict), on a tiny real model
    y = [np.array([0.1 * t]) for t in range(5)]
    fk = ssms.Bootstrap(ssm=ssms.StochVol(), data=y)
    for name, of in (("multismc_float", lambda pf: float(pf.t)), ("multismc_dict", lambda pf: {"t": pf.t, "N": pf.N})):
        np.random.seed(7)
        res = particles.multiSMC(fk={"boot": fk}, N=[20, 30], nruns=2, nprocs=1, out_func=of, collect=None)
        out[name] = {"seed": 7, "result": record(res)}
    np.random.seed(8)
    res = particles.multiSMC(fk=fk, N=20, nruns=1, nprocs=1, out_func=lambda pf: pf.t)
    out["multismc_one_run"] = {"seed": 8, "result": record(res)}
    path = os.path.join(HERE, "golden_multismc.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(path)


if __name__ == "__main__":
    main()
