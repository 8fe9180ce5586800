"""Single-run variance estimators on the CPU: the NumPy oracle (tests/variance_oracle.py) against the live reference's
output (tests/golden/golden_variance.npz, written by make_golden_variance.py), and the branch-sum algebra of
csrc/smcb_variance.cuh, compiled for the host by tests/variance_host.cpp, against the oracle on adversarial rows."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import variance_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_build")
CASES = ["sv_sys", "lg_multi", "sv_strat", "mvlg2", "sv_ssp", "sv_resid", "sv_kill", "collapse"]
HAND = ["all_equal", "unsorted_ends", "unsorted", "n1", "singletons", "vector"]


@pytest.fixture(scope="module")
def gv():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_variance.npz"))


def phi_of(name):
    return (lambda x: 1.0 * x) if name == "mvlg2" else (lambda x: x ** 2)


def phi_fl(xs):
    return sum(x if x.ndim == 1 else x[:, 0] for x in xs)


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference(gv, name):
    lag = int(gv["meta/T_N_LAG"][2])
    X, lw, A = gv[f"{name}/X"], gv[f"{name}/lw"], gv[f"{name}/A"].astype(np.int64)
    out = vo.replay(X, lw, A, phi_of(name), lag, phi_fl)
    for key in ("var", "var_logLt", "fixed_lag_smooth"):
        np.testing.assert_allclose(np.array(out[key], dtype=float), gv[f"{name}/{key}"], rtol=1e-13, atol=0,
                                   err_msg=key)
    ref_zero = gv[f"{name}/var"] == 0.0
    assert np.array_equal(np.array(out["var"], dtype=float) == 0.0, ref_zero)
    lagv = gv[f"{name}/lag_based_var"]
    for t, row in enumerate(out["lag_based_var"]):
        np.testing.assert_allclose(np.array(row, dtype=float), lagv[t, :len(row)], rtol=1e-13, atol=0)
        assert np.isnan(lagv[t, len(row):]).all()
    if name == "collapse":
        assert ref_zero[1:].all()
    # the Eve rows of the schemes with non-decreasing ancestors stay sorted; residual and killing break that
    rows_sorted = all(np.all(np.diff(B) >= 0) for B in vo.eve_rows(A))
    assert rows_sorted == (name not in ("sv_resid", "sv_kill"))


@pytest.mark.parametrize("case", HAND)
def test_oracle_hand_made_inputs(gv, case):
    W, phi, B = (gv[f"hand/{case}/{k}"] for k in ("W", "phi", "B"))
    got = np.asarray(vo.var_estimate(W, phi, B), dtype=float)
    np.testing.assert_allclose(got, gv[f"hand/{case}/out"], rtol=1e-13, atol=0)
    if case in ("all_equal", "unsorted_ends", "n1"):
        assert np.all(gv[f"hand/{case}/out"] == 0.0)


_lib = None


def host_lib():
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "libvariance_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"),
                               os.path.join(ROOT, "tests", "variance_host.cpp"), "-o", so])
        _lib = C.CDLL(so)
        _lib.vh_branch_sums.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p]
    return _lib


def host_sums(B, v, chunk, tree):
    B, v = np.ascontiguousarray(B, dtype=np.int64), np.ascontiguousarray(v, dtype=np.float64)
    out = np.zeros(3)
    host_lib().vh_branch_sums(B.ctypes.data, v.ctypes.data, B.shape[0], chunk, int(tree), out.ctypes.data)
    return out


def adversarial_rows():
    r = np.random.RandomState(3)
    yield "one_run", np.full(37, 5)
    yield "all_distinct", np.arange(41)
    yield "long_runs", np.repeat(np.arange(4), [1, 29, 3, 17])          # runs across many chunks
    yield "random", np.sort(r.randint(0, 12, size=103))                  # N not a multiple of the chunk
    yield "n1", np.array([0])
    yield "singletons_then_run", np.concatenate([np.arange(7), np.full(20, 7), np.arange(8, 11)])


@pytest.mark.parametrize("chunk", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("tree", [False, True])
def test_host_chunk_and_carry_match_oracle(chunk, tree):
    r = np.random.RandomState(chunk)
    for name, B in adversarial_rows():
        v = r.normal(size=B.shape[0])
        got = host_sums(B, v, chunk, tree)
        exp = np.sum(vo.branch_sums(v, B, N=int(B.max()) + 1) ** 2)
        np.testing.assert_allclose(got[0], exp, rtol=1e-13, atol=1e-300, err_msg=name)
        assert got[1] == float(B[0] == B[-1]) and got[2] == 0.0, name


def test_host_flags_unsorted_rows():
    B = np.array([0, 0, 3, 1, 1, 4])
    for chunk in (1, 2, 4, 6):
        assert host_sums(B, np.ones(6), chunk, False)[2] == 1.0
