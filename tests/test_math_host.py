"""The fp64 elementary functions of the step kernel (particles_b200/csrc/smcb_math.cuh), compiled for the
CPU by tests/math_host.cpp and checked against NumPy / mpmath: the polynomial family (stand-alone kernels) and
the table-assisted family the step kernels run on (tables of csrc/smcb_tables.h).  The GPU counterpart
(test_gpu_kernels.py::test_device_math) checks the device build of both."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_build")


_lib = None


def build_math_host():
    """g++ build of tests/math_host.cpp (device math + model headers compiled for the host)."""
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "libmath_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"),
                               "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "math_host.cpp"), "-o", so])
        _lib = C.CDLL(so)
        _lib.mh_init()
    return _lib


def ulps(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return np.abs(got - ref) / np.spacing(np.abs(ref))


class _Fam:
    """The host library with one family selected (tab = 0 polynomial, 1 table-assisted)."""

    def __init__(self, lib, tab):
        self.lib, self.tab = lib, tab


@pytest.fixture(scope="module", params=[0, 1], ids=["polynomial", "table"])
def mh(request):
    return _Fam(build_math_host(), request.param)


def call(fam, name, *arrays, extra=(), tab=True):
    n = arrays[0].shape[0]
    args = [a.ctypes.data_as(C.c_void_p) for a in arrays]
    tail = (C.c_int(fam.tab),) if tab else ()
    getattr(fam.lib, name)(*args, C.c_long(n), *extra, *tail)


def test_exp(mh):
    r = np.random.RandomState(0)
    x = np.concatenate([r.uniform(-708, 709, 200_000), r.uniform(-40, 5, 200_000), r.uniform(-1e-3, 1e-3, 50_000),
                        np.array([0.0, -0.0, 1.0, -1.0, 709.0, -708.0, 1e-300, -745.0])])
    want = np.exp(x.astype(np.longdouble)).astype(np.float64)
    for kind in (0, 1, 2):
        xs = x if kind != 1 else -np.abs(x)
        w = want if kind != 1 else np.exp((-np.abs(x)).astype(np.longdouble)).astype(np.float64)
        y = np.empty_like(xs)
        call(mh, "mh_exp", xs, y, extra=(C.c_int(kind),))
        ok = (xs >= -708.0) if kind != 2 else (np.abs(xs) < 700)
        assert ulps(y[ok], w[ok]).max() <= 1.5, (kind, ulps(y[ok], w[ok]).max())      # measured in long double: 0.94 / 1.0
        if kind != 2:
            assert np.all(y[xs < -708.0] == 0.0)
    if mh.tab:      # texp_sat: clamped power of two instead of selects -- saturates, never wraps
        xs = np.array([-800.0, -5000.0, -1e6, -1e8, 800.0, 5000.0, 1e8, -708.3, 709.7])
        y = np.empty_like(xs)
        call(mh, "mh_exp", xs, y, extra=(C.c_int(2),))
        assert np.all(y[:4] > 0) and np.all(y[:4] < 1e-307) and np.all(y[4:7] > 8e307) and np.all(np.isfinite(y))
        np.testing.assert_allclose(y[7:], np.exp(xs[7:]), rtol=3e-16)
    sp = np.array([-np.inf, np.inf, np.nan, 710.0, -1000.0])
    y = np.empty_like(sp)
    call(mh, "mh_exp", sp, y, extra=(C.c_int(0),))
    assert y[0] == 0.0 and y[1] == np.inf and np.isnan(y[2]) and y[3] == np.inf and y[4] == 0.0


def test_log(mh):
    r = np.random.RandomState(1)
    x = np.concatenate([r.uniform(0, 1, 300_000), 2.0 ** r.uniform(-54, 0, 100_000), 1 - 2.0 ** r.uniform(-53, -1, 50_000),
                        r.uniform(0.7, 1.5, 100_000), np.array([1.0, 0.5, 2.0 ** -54, 1 - 2.0 ** -53, np.sqrt(0.5), np.sqrt(2.0)])])
    x = x[x > 0]
    y = np.empty_like(x)
    call(mh, "mh_log", x, y)
    want = np.log(x.astype(np.longdouble)).astype(np.float64)
    nz = want != 0
    if mh.tab:
        # table family: log(m) = -log(1/c_j) + log1p(m/c_j - 1) cancels near 1, so the error is 3 ulp of the result
        # PLUS an absolute 3e-19 (half an ulp of the largest table term next to 1, 2.4e-4).  It only feeds
        # Box-Muller, where |log u| >= 1.1e-16 and an absolute 3e-19 moves the radius by < 1e-11 relative
        assert np.all(np.abs(y - want) <= 3.0 * np.spacing(np.abs(want)) + 3e-19)
    else:
        assert ulps(y[nz], want[nz]).max() <= 3.0, ulps(y[nz], want[nz]).max()      # 2.8
        assert np.all(y[~nz] == 0.0)                      # log(1) == 0 exactly


def test_sincos(mh):
    u = np.concatenate([np.random.RandomState(2).uniform(0, 1, 300_000), np.arange(9) / 8.0, [1 - 2.0 ** -53, 2.0 ** -53]])
    s, c = np.empty_like(u), np.empty_like(u)
    call(mh, "mh_sincos2pi", u, s, c)
    ul = u.astype(np.longdouble)
    ws = np.sin(2 * np.pi * ul.astype(np.float64))     # tolerance is absolute: argument reduction in fp64
    import mpmath as mp
    idx = np.random.RandomState(3).choice(u.shape[0], 2000, replace=False)
    for i in idx:
        assert abs(s[i] - float(mp.sin(2 * mp.pi * mp.mpf(float(u[i]))))) < 7e-16
        assert abs(c[i] - float(mp.cos(2 * mp.pi * mp.mpf(float(u[i]))))) < 7e-16
    assert np.abs(s - ws).max() < 1e-15
    assert np.abs(s * s + c * c - 1).max() < 1.5e-15


def test_box_muller_and_lse3(mh):
    r = np.random.RandomState(4)
    words = r.randint(0, 2 ** 32, size=(200_000, 4), dtype=np.uint64).astype(np.uint32)
    z = np.empty(2 * words.shape[0])
    mh.lib.mh_box_muller(words.ctypes.data_as(C.c_void_p), z.ctypes.data_as(C.c_void_p), C.c_long(words.shape[0]),
                         C.c_int(mh.tab))
    a, b = words[:, 0].astype(np.uint64), words[:, 1].astype(np.uint64)
    u1 = (((a >> 5) << 26) | (b >> 6)).astype(np.float64) + 0.5
    u1 *= 2.0 ** -53
    a, b = words[:, 2].astype(np.uint64), words[:, 3].astype(np.uint64)
    u2 = (((a >> 5) << 26) | (b >> 6)).astype(np.float64) * 2.0 ** -53
    rad = np.sqrt(-2 * np.log(u1))
    np.testing.assert_allclose(z[0::2], rad * np.cos(2 * np.pi * u2), rtol=0, atol=5e-15)
    np.testing.assert_allclose(z[1::2], rad * np.sin(2 * np.pi * u2), rtol=0, atol=5e-15)
    assert abs(z.mean()) < 5e-3 and abs(z.std() - 1) < 5e-3
    v = r.randn(100_003) * 30 - 200
    v[::97] = -np.inf
    out = np.zeros(3)
    mh.lib.mh_lse3(v.ctypes.data_as(C.c_void_p), C.c_long(v.shape[0]), out.ctypes.data_as(C.c_void_p))
    m = v.max()
    e = np.exp(v - m)
    assert out[0] == m
    np.testing.assert_allclose(out[1:], [e.sum(), (e * e).sum()], rtol=1e-13)


def test_tile_search():
    """The in-tile CDF search of the step kernel's multinomial and global-resampling move passes
    (smcb_search.cuh tile_search) against np.searchsorted(slice, v, 'left'): slices with ties and flat runs of zero
    mass, keys below the first and above the last entry, slices of 1 and 2 entries, and start offsets up to the
    first key's answer (at cnt when every entry lies below it)."""
    lib = build_math_host()
    r = np.random.RandomState(6)
    for trial in range(400):
        cnt = [1, 2, 3, 5, 8, 64, 4096][trial % 7]
        steps = r.exponential(1.0, cnt) * (r.rand(cnt) < 0.6)          # zero steps: ties / flat runs
        if trial % 5 == 0:
            steps[r.randint(0, cnt):] = 0.0                               # a long flat tail
        s = np.cumsum(steps) + r.uniform(-1.0, 1.0)
        lo, hi = s[0] - 1.0, s[-1] + 1.0
        m = 300
        v0 = np.concatenate([r.uniform(lo, hi, m - 20), s[r.randint(0, cnt, 10)], [lo - 5.0] * 5, [hi + 5.0] * 5])
        gap = np.where(r.rand(m) < 0.5, r.exponential(2.0 * (hi - lo) / cnt, m), 0.0)
        v1 = v0 + gap * (r.rand(m) < 0.9) + (hi - lo + 10.0) * (r.rand(m) < 0.05)     # some far past the slice
        eq = r.rand(m) < 0.1
        v1[eq] = v0[eq]                                                   # both outputs on one key
        want0, want1 = np.searchsorted(s, v0, "left"), np.searchsorted(s, v1, "left")
        l0 = (r.rand(m) * (want0 + 1)).astype(np.int32)
        near = r.rand(m) < 0.3
        l0[near] = want0[near]                                            # start at the answer (up to cnt)
        v = np.ascontiguousarray(np.stack([v0, v1], axis=1))
        out = np.empty((m, 2), dtype=np.int32)
        lib.mh_tile_search(s.ctypes.data_as(C.c_void_p), C.c_int(cnt), l0.ctypes.data_as(C.c_void_p),
                           v.ctypes.data_as(C.c_void_p), C.c_long(m), out.ctypes.data_as(C.c_void_p))
        assert np.array_equal(out[:, 0], want0), (cnt, trial)
        assert np.array_equal(out[:, 1], want1), (cnt, trial)


def test_sqrt_and_tables():
    """tsqrt_pos (reciprocal-square-root seed truncated to what MUFU.RSQ64H delivers + one third-order step) and
    the lookup tables themselves against mpmath."""
    lib = build_math_host()
    r = np.random.RandomState(5)
    x = np.concatenate([r.uniform(0, 80, 200_000), 2.0 ** r.uniform(-60, 7, 100_000), np.array([1.0, 4.0, 2.0, 1e-300, 75.0])])
    y = np.empty_like(x)
    lib.mh_sqrt(x.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), C.c_long(x.shape[0]))
    assert ulps(y, np.sqrt(x.astype(np.longdouble)).astype(np.float64)).max() <= 2.5
    import mpmath as mp
    mp.mp.prec = 120
    lib.mh_tables.restype = C.POINTER(C.c_double)
    n = lib.mh_table_doubles()
    t = np.ctypeslib.as_array(lib.mh_tables(), shape=(n,)).copy()
    assert n == 8192
    for j in r.choice(4096, 300, replace=False):
        assert abs(t[j] - float(mp.power(2, mp.mpf(int(j)) / 4096))) <= 0.51 * np.spacing(t[j])
    for j in r.choice(1024, 300, replace=False):
        inv, nl = t[4096 + 2 * j], t[4096 + 2 * j + 1]
        c = (1 + (int(j) + 0.5) / 1024) * (0.5 if j >= 0x1A8 else 1.0)
        assert abs(inv * c - 1) < 3e-16
        assert abs(nl + float(mp.log(mp.mpf(float(inv))))) <= 0.51 * np.spacing(abs(nl)) + 1e-300
        s_, c_ = t[6144 + 2 * j], t[6144 + 2 * j + 1]
        a = 2 * mp.pi * int(j) / 1024
        assert abs(s_ - float(mp.sin(a))) < 1.2e-16 and abs(c_ - float(mp.cos(a))) < 1.2e-16
    assert t[6144] == 0.0 and t[6145] == 1.0 and t[6144 + 2 * 256] == 1.0 and t[6145 + 2 * 256] == 0.0
