"""The reference's per-step attributes of a device-run filter (``core._Results``), driven on the host with hand-made
summary tables and CPU tensors: first steps, resampled and non-resampled last steps, the formulas ``BatchRun`` used
before it shared them, and the host reads of a fused ``SMC``'s attributes."""
import types

import numpy as np
import pytest
import torch

from particles_b200 import core


def table_of(rs_flags, seed=0):
    """(T, 4) summary table (ESS, logLt, rs_flag, log_mean_w) with the given resampling flags."""
    rng = np.random.RandomState(seed)
    T = len(rs_flags)
    return np.column_stack([rng.uniform(1.0, 100.0, T), np.cumsum(rng.standard_normal(T)),
                            np.asarray(rs_flags, dtype=np.float64), rng.standard_normal(T)])


def results(table, t, N=5):
    X = torch.arange(2 * N, dtype=torch.float64).reshape(2, N)
    A = torch.tensor([4, 4, 0, 1, 2])[:N]
    return core._Results(t, N, table.__getitem__, lambda s: X[s & 1], lambda: A), X, A


def old_batchrun(table, X, A, N):
    """rs_flag, logLt, log_mean_w, loglt, X, A and (non-resampled) Xp as BatchRun derived them from its own table."""
    T = table.shape[0]
    rs_flag, log_mean_w = bool(table[-1, 2]), float(table[-1, 3])
    loglt = log_mean_w if T == 1 or rs_flag else log_mean_w - float(table[-2, 3])
    gen = lambda s: X[s & 1]                                                     # noqa: E731
    anc = None if T <= 1 else (A if rs_flag else torch.arange(N))
    Xp = None if T <= 1 or rs_flag else gen(T - 2)
    return rs_flag, float(table[-1, 1]), log_mean_w, loglt, gen(T - 1), anc, Xp


def test_one_step():
    table = table_of([0])
    r, X, _ = results(table, 1)
    assert r.rs_flag is False and r.logLt == table[0, 1] and r.loglt == table[0, 3] == r.log_mean_w
    assert torch.equal(r.X, X[0]) and r.A is None and r.Xp is None


def test_before_and_after_the_first_step():
    table = table_of([1, 0, 0])                  # a first step's loglt is its log_mean_w, flag or not
    r, X, _ = results(table, 0)
    assert r.rs_flag is False and r.logLt == 0.0 and r.X is None and r.A is None and r.Xp is None
    r, X, _ = results(table, 1)
    assert r.rs_flag is True and r.loglt == table[0, 3] and r.logLt == table[0, 1]
    assert torch.equal(r.X, X[0]) and r.A is None and r.Xp is None


@pytest.mark.parametrize("last", [0, 1])
def test_last_step(last):
    table = table_of([0, 1, 0, last], seed=last)
    r, X, A = results(table, 4)
    assert r.rs_flag is bool(last) and r.logLt == table[3, 1] and r.log_mean_w == table[3, 3]
    assert torch.equal(r.X, X[1])
    if last:
        assert r.loglt == table[3, 3] and r.A is A
    else:
        assert r.loglt == table[3, 3] - table[2, 3]
        assert torch.equal(r.A, torch.arange(5)) and torch.equal(r.Xp, X[0])


def test_agrees_with_old_batchrun_formulas():
    rng = np.random.RandomState(7)
    for T in range(1, 7):
        for k in range(8):
            table = table_of(rng.rand(T) < 0.5, seed=10 * T + k)
            r, X, A = results(table, T)
            new = (r.rs_flag, r.logLt, r.log_mean_w, r.loglt, r.X, r.A, None if r.rs_flag else r.Xp)
            for a, b in zip(new, old_batchrun(table, X, A, 5)):
                if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
                    assert torch.equal(a, b), (T, k)
                else:
                    assert a == b and type(a) is type(b), (T, k)


class _CountingTable:
    """Device table stand-in that records each row read."""

    def __init__(self, table):
        self.table, self.reads = torch.from_numpy(table), []

    def __getitem__(self, t):
        self.reads.append(t)
        return self.table[t]


def test_fused_smc_reads_each_row_once():
    """Reading every attribute of a fused SMC after each step reads each summary row once: ``loglt``'s row t - 1
    stays cached next to ``rs_flag``'s row t."""
    N, flags = 5, [0, 0, 1, 0, 0, 1]
    table = table_of(flags)
    pf = core.SMC.__new__(core.SMC)
    X, A = torch.arange(2.0 * N).reshape(2, N), torch.tensor([4, 4, 0, 1, 2])
    pf._engine = types.SimpleNamespace(summ=_CountingTable(table), X=[X[0], X[1]], A=A)
    pf.N, pf._row_cache = N, {}
    for t in range(1, len(flags) + 1):
        pf._done = t
        before = len(pf._engine.summ.reads)
        for _ in range(2):
            got = (pf.rs_flag, pf.logLt, pf.log_mean_w, pf.loglt, pf.X, pf.A, pf.rs_flag)
            if not pf.rs_flag:
                assert (pf.Xp is None) == (t == 1)
        assert pf._engine.summ.reads[before:] == [t - 1], t
        assert got[:4] == (bool(flags[t - 1]), table[t - 1, 1], table[t - 1, 3],
                           table[t - 1, 3] - (0.0 if t == 1 or flags[t - 1] else table[t - 2, 3]))
