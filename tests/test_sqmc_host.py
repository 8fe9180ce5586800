"""The SQMC building blocks of particles_b200/csrc/smcb_sqmc.cuh compiled for the CPU by tests/sqmc_host.cpp:
Sobol' points against scipy.stats.qmc.Sobol, the net property of the scrambled points, the inverse normal CDF against
scipy.special.ndtri, and the Hilbert keys against the reference's (tests/golden/golden_sqmc.npz)."""
import ctypes as C
import os
import subprocess
import warnings

import numpy as np
import pytest
from scipy.special import ndtri
from scipy.stats import qmc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_build")
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_sqmc.npz")
# the largest error of the device Phi^-1 against ndtri over the squeezed points, in ulp (DESIGN.md section 5.17)
NDTRI_ULP = 8

_lib = None


def build_sqmc_host():
    """g++ build of tests/sqmc_host.cpp (smcb_sqmc.cuh compiled for the host)."""
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "libsqmc_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "sqmc_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        vp = C.c_void_p
        lib.sh_ndtri.argtypes = [vp, vp, C.c_long]
        lib.sh_sobol.argtypes = [C.c_int, C.c_long, C.c_long, C.c_int, C.c_uint64, C.c_uint64, vp, vp]
        lib.sh_hilbert_keys.argtypes = [vp, C.c_long, C.c_int, vp]
        _lib = lib
    return _lib


def host_sobol(d, n, scramble=True, seed=0, call=0, i0=0):
    """(u, raw), each (d, n) component-major, as smcb_sobol writes them."""
    u = np.empty((d, n))
    raw = np.empty((d, n), dtype=np.int32)
    build_sqmc_host().sh_sobol(d, i0, n, int(scramble), seed, call, u.ctypes.data, raw.ctypes.data)
    return u, raw


def host_ndtri(p):
    p = np.ascontiguousarray(p, dtype=np.float64)
    out = np.empty_like(p)
    build_sqmc_host().sh_ndtri(p.ctypes.data, out.ctypes.data, p.size)
    return out


def host_hilbert_keys(xint):
    xint = np.ascontiguousarray(xint, dtype=np.int64)
    out = np.empty(xint.shape[0], dtype=np.int64)
    build_sqmc_host().sh_hilbert_keys(xint.ctypes.data, xint.shape[0], xint.shape[1], out.ctypes.data)
    return out


def hilbert_ints(x):
    """hilbert_sort's integer points of the (N, d) float points x (NumPy's mean and std)."""
    d = x.shape[1]
    xs = 1.0 / (1.0 + np.exp(-((x - np.mean(x, axis=0)) / np.std(x, axis=0))))
    return np.floor(xs * np.floor(2 ** (62 / d))).astype(np.int64)


def squeeze(u):
    return 0.5 + (1.0 - 1e-10) * (u - 0.5)


@pytest.mark.parametrize("d", [1, 2, 3, 5, 8, 13, 21, 32])
@pytest.mark.parametrize("n", [1, 2, 7, 64, 1000, 4097, 65536])
def test_unscrambled_points_equal_scipy(d, n):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = qmc.Sobol(d, scramble=False).random(n)
    u, raw = host_sobol(d, n, scramble=False)
    assert np.array_equal(raw.T * 2.0 ** -30, ref)
    assert np.array_equal(u.T, squeeze(ref))


@pytest.mark.parametrize("m", [1, 4, 9, 12, 16])
def test_scrambled_points_are_nets(m):
    n, d = 2 ** m, 6
    _, raw = host_sobol(d, n, seed=987654321, call=5)
    for j in range(d):          # every coordinate: one point per interval of length 2^-m
        assert np.array_equal(np.sort(raw[j] >> (30 - m)), np.arange(n))
    for a in range(m + 1):      # pair (0, 1): one point per elementary interval of area 2^-m
        cell = ((raw[0].astype(np.int64) >> (30 - a)) << (m - a)) | (raw[1].astype(np.int64) >> (30 - (m - a)))
        assert np.array_equal(np.sort(cell), np.arange(n))


def test_scrambling_depends_on_seed_and_call_only():
    a, b = host_sobol(4, 100, seed=1, call=2), host_sobol(4, 100, seed=1, call=2)
    assert np.array_equal(a[1], b[1])
    assert not np.array_equal(a[1], host_sobol(4, 100, seed=1, call=3)[1])
    assert not np.array_equal(a[1], host_sobol(4, 100, seed=2, call=2)[1])
    # a prefix of the sequence: points i0 .. i0 + n - 1 equal those of one longer call
    assert np.array_equal(host_sobol(4, 50, seed=1, call=2, i0=50)[1], a[1][:, 50:])


def test_ndtri_within_stated_ulp():
    rng = np.random.default_rng(3)
    grid = np.arange(0, 2 ** 30, 101, dtype=np.float64) * 2.0 ** -30
    ends = np.array([0.0, (2 ** 30 - 1) * 2.0 ** -30, 2.0 ** -30, 0.5, 0.075, 0.925])
    p = squeeze(np.concatenate([grid, rng.random(10 ** 6), ends]))
    ref = ndtri(p)
    got = host_ndtri(p)
    ulp = np.abs(got - ref) / np.spacing(np.abs(ref))
    assert ulp.max() <= NDTRI_ULP, (ulp.max(), p[np.argmax(ulp)])
    assert np.array_equal(np.sign(got), np.sign(ref))


@pytest.mark.parametrize("d", [2, 3, 4, 5, 6])
def test_hilbert_keys_equal_reference(d):
    g = np.load(GOLDEN)
    keys = host_hilbert_keys(g[f"xint_{d}"])
    assert np.array_equal(keys, g[f"keys_{d}"])
    if d >= 4:
        assert (keys < 0).any()             # the wrapped keys are part of the fixture


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_hilbert_order_equals_reference(d):
    g = np.load(GOLDEN)
    x, order = g[f"x_{d}"], g[f"order_{d}"]
    if d == 1:
        assert np.array_equal(np.sort(x[:, 0]), x[order, 0])
        return
    keys = host_hilbert_keys(hilbert_ints(x))
    assert np.array_equal(np.sort(order), np.arange(x.shape[0]))
    assert np.array_equal(keys[order], np.sort(keys))       # the reference's order sorts our keys
