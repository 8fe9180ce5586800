"""Argument multiplexing for ``multiSMC`` (the interface of particles/utils.py:90-269), host only.

``multiplexer(f, nruns, nprocs, seeding, protected_args, **args)`` evaluates ``f`` for every element of the
cartesian product of the list- and dict-valued arguments, ``nruns`` times each, and returns one dict per
evaluation: ``'run'``, the varied arguments (dict-valued ones by their keys), ``'seed'`` when seeding, then
``'output'`` (or the keys of a dict that ``f`` returns).  Seeds are drawn from the global ``numpy.random`` stream
as the reference draws them, so ``np.random.seed(s)`` gives the reference's seeds.

This module imports no CUDA code.  ``nprocs`` is accepted and ignored: evaluations run one after another in this
process (``multiSMC`` gets its parallelism from the device instead).
"""
import itertools

import numpy as np

MAX_INT_32 = np.iinfo(np.uint32).max      # (the reference's name for 2^32 - 1)


def cartesian_lists(d):
    """Dict of lists -> list of dicts, one per element of the cartesian product (last key varies fastest)."""
    keys = list(d.keys())
    return [dict(zip(keys, combo)) for combo in itertools.product(*d.values())]


def cartesian_args(args, listargs, dictargs):
    """(inputs, outputs): the inputs take fixed ``args``, the product of ``listargs`` and of the values of
    ``dictargs``; the outputs record the varied list values and the keys of the dict-valued arguments."""
    ils = {k: [v] for k, v in args.items()}
    ils.update(listargs)
    ils.update({k: list(v.values()) for k, v in dictargs.items()})
    ols = dict(listargs)
    ols.update({k: list(v.keys()) for k, v in dictargs.items()})
    return cartesian_lists(ils), cartesian_lists(ols)


def add_to_dict(d, obj, key="output"):
    """Merge a dict result into ``d``, or store any other result under ``key``."""
    if isinstance(obj, dict):
        d.update(obj)
    else:
        d[key] = obj
    return d


def distinct_seeds(k):
    """k distinct seeds in [0, 2^32 - 1): one uniform draw in each of k equal bins (stratified)."""
    bw = MAX_INT_32 // k
    return np.arange(0, k * bw, bw) + np.random.randint(bw, size=k)


def expand(nruns=1, seeding=None, protected_args=None, **args):
    """The evaluations ``multiplexer`` makes, without making them: (inputs, outputs), where inputs[i] are the
    keyword arguments of evaluation i (``seed`` included when seeding) and outputs[i] its result dict so far."""
    fixed = dict(protected_args or {})
    listargs, dictargs = {"run": list(range(nruns))}, {}
    for k, v in args.items():
        if isinstance(v, list):
            listargs[k] = v
        elif isinstance(v, dict):
            dictargs[k] = v
        else:
            fixed[k] = v
    inputs, outputs = cartesian_args(fixed, listargs, dictargs)
    for ip in inputs:
        del ip["run"]                     # an identifier of the output, not an argument
    if seeding is None:
        seeding = nruns > 1
    if seeding:
        for ip, op, s in zip(inputs, outputs, distinct_seeds(len(inputs))):
            ip["seed"] = s
            op["seed"] = s
    return inputs, outputs


def _seeded(f):
    def g(**kw):
        s = kw.pop("seed", None)
        if s:
            np.random.seed(s)
        return f(**kw)
    return g


def multiplexer(f=None, nruns=1, nprocs=1, seeding=None, protected_args=None, **args):
    """Evaluate ``f(**kwargs)`` for every combination of the arguments (see the module docstring).  With seeding,
    ``numpy.random`` is seeded with the evaluation's seed before each call."""
    if not callable(f):
        raise TypeError("multiplexer: function f missing, or not callable")
    seeding = nruns > 1 if seeding is None else seeding
    inputs, outputs = expand(nruns=nruns, seeding=seeding, protected_args=protected_args, **args)
    g = _seeded(f) if seeding else f
    return [add_to_dict(op, g(**ip)) for ip, op in zip(inputs, outputs)]
