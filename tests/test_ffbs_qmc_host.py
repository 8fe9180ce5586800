"""QMC backward sampling without a GPU: the Sobol' direction numbers past 32 dimensions (host build of
csrc/smcb_sqmc.cuh) against scipy, the NumPy restatement of the reference's ``backward_sampling_qmc`` against the
reference's own paths (tests/golden/golden_ffbs_qmc.npz), and the refusals of ``ParticleHistory``."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
from scipy.stats import qmc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ffbs_qmc_oracle as fo  # noqa: E402
import test_sqmc_host as hh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_build")
_lib = None


def dims_lib():
    """g++ build of tests/sobol_dims_host.cpp."""
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "libsobol_dims_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "sobol_dims_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.sd_dirs.argtypes = [C.c_int, C.c_int, C.c_void_p]
        _lib = lib
    return _lib


def dirs(j, tab):
    out = np.empty(30, dtype=np.uint32)
    dims_lib().sd_dirs(j, int(tab), out.ctypes.data)
    return out


def test_bounds():
    from particles_b200 import hilbert, rqmc
    assert dims_lib().sd_max_dim() == rqmc.MAX_DIM == 4096
    assert dims_lib().sd_tab_dim() == hilbert.MAX_DIM == 32


def test_expansion_equals_the_committed_table():
    for j in range(1, 32):
        assert np.array_equal(dirs(j, True), dirs(j, False)), j


@pytest.mark.parametrize("d,n", [(33, 1000), (100, 777), (1000, 300), (4096, 129)])
def test_unscrambled_points_equal_scipy(d, n):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = qmc.Sobol(d, scramble=False).random(n)
    u, raw = hh.host_sobol(d, n, scramble=False)
    assert np.array_equal(raw.T * 2.0 ** -30, ref)
    assert np.array_equal(u.T, hh.squeeze(ref))


def test_scrambled_dimensions_do_not_depend_on_d():
    a, ra = hh.host_sobol(40, 257, scramble=True, seed=5, call=3)
    b, rb = hh.host_sobol(33, 257, scramble=True, seed=5, call=3)
    assert np.array_equal(ra[:33], rb) and np.array_equal(a[:33], b)
    # the net property of the scrambled points, per dimension, past the table
    _, raw = hh.host_sobol(300, 256, scramble=True, seed=9, call=1)
    for j in (32, 99, 299):
        assert np.array_equal(np.sort(raw[j] >> 22), np.arange(256))


@pytest.mark.parametrize("k", range(7))
def test_oracle_reproduces_the_reference_paths(k):
    g = np.load(fo.GOLDEN)
    (mc, N, T, M), c = fo.case(g, k)
    om = fo.oracle_model(mc)
    X = [c["X"][t] for t in range(T)]
    idx = fo.backward_qmc(X, list(c["lw"]), list(c["h"]), lambda t, xp, x: om.PX(t, xp).logpdf(x), c["ub"])
    assert np.array_equal(idx, c["idx"])
    assert np.array_equal(np.array([X[t][idx[t]] for t in range(T)]), c["paths"])


def test_history_refusals():
    from particles_b200.smoothing import HilbertOrdersError, ParticleHistory
    h = ParticleHistory(None, False)
    h.X = [0, 0]
    with pytest.raises(NotImplementedError, match="qmc=True"):
        h.backward_sampling_qmc(4)
    with pytest.raises(ValueError):
        h.backward_sampling_qmc(4)
    assert issubclass(HilbertOrdersError, NotImplementedError) and issubclass(HilbertOrdersError, ValueError)
    h = ParticleHistory(None, True)
    assert h.h_orders == []
    h.X = [0] * 4097
    with pytest.raises(NotImplementedError, match="4096"):
        h.backward_sampling_qmc(4)
