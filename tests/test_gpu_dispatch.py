"""The (model, dim, Feynman-Kac kind, scheme) combinations the library does not build: each entry point answers with
its own return code and message (csrc/smcb_dispatch.cuh is the one table; the callers word the errors).  The Python
layer turns -1 into ValueError and -3 into NotImplementedError, so these codes and texts are what users see."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL, ENOSYS = -1, -3


@pytest.fixture(scope="module")
def env():
    from particles_b200 import _lib, device
    ctx = device.context()
    buf = torch.zeros(64, dtype=torch.float64, device=ctx.device)      # never read: every call fails before a launch
    return _lib, _lib.load(), ctx.handle, buf.data_ptr(), buf


def last_error(lib):
    return lib.smcb_last_error().decode()


@pytest.mark.parametrize("model, fk, scheme, dim, rc, msg", [
    (2, 2, 2, 1, ENOSYS, "fused filter: model 2 implements no proposal/logeta (Feynman-Kac kind 2)"),
    (4, 0, 2, 3, EINVAL, "fused BearingsOnly: state dimension must be 4"),
    (4, 0, 2, 1, ENOSYS, "fused filter: model id 4 is not available in the fused 1-D family"),
    (5, 0, 2, 1, ENOSYS, "fused filter: model id 5 is not available in the fused 1-D family"),
    (9, 0, 2, 1, ENOSYS, "fused filter: model id 9 is not available in the fused 1-D family"),
    (9, 0, 2, 2, ENOSYS, "fused filter: model id 9 has no d-dimensional kernel"),
    (0, 0, 2, 2, ENOSYS, "fused filter: model id 0 has no d-dimensional kernel"),
    (0, 7, 2, 1, EINVAL, "fused filter: unknown Feynman-Kac kind 7"),
    (2, 7, 2, 1, EINVAL, "fused filter: unknown Feynman-Kac kind 7"),
    (0, 0, 3, 1, ENOSYS, "fused filter: resampling scheme 3 is not fused (use systematic, stratified or multinomial, "
                         "or the unfused path)"),
])
def test_filter_create(env, model, fk, scheme, dim, rc, msg):
    _lib, lib, ctx, p, _ = env
    d = _lib.FilterDesc()
    d.model, d.fk, d.scheme, d.dim, d.dy = model, fk, scheme, dim, 1
    d.n, d.T, d.essrmin = 4, 2, 0.5
    d.X[0] = d.X[1] = d.lw[0] = d.lw[1] = d.A = d.cdf = d.data = d.summaries = p
    out = C.c_void_p()
    assert lib.smcb_filter_create(ctx, C.byref(d), C.byref(out)) == rc
    assert last_error(lib) == msg
    assert not out.value


@pytest.mark.parametrize("model, fk, scheme, rc, msg", [
    (4, 0, 2, ENOSYS, "batched filter: model id 4 is not built"),
    (5, 0, 2, ENOSYS, "batched filter: model id 5 is not built"),
    (9, 0, 2, ENOSYS, "batched filter: model id 9 is not built"),
    (2, 2, 2, ENOSYS, "batched filter: Feynman-Kac kind 2 is not built for model 2"),
    (0, 7, 2, ENOSYS, "batched filter: Feynman-Kac kind 7 is not built for model 0"),
    (0, 0, 3, ENOSYS, "batched filter: resampling scheme 3 is not built"),
])
def test_batch_plan(env, model, fk, scheme, rc, msg):
    _lib, lib, ctx, _, _ = env
    d = _lib.BatchDesc()
    d.model, d.fk, d.scheme, d.dim, d.dy = model, fk, scheme, 1, 1
    d.N, d.T, d.R = 4, 2, 1
    out = (C.c_int64 * 2)()
    assert lib.smcb_batch_plan(ctx, C.byref(d), out) == rc
    assert last_error(lib) == msg


@pytest.mark.parametrize("model, dim, rc, msg", [
    (9, 1, ENOSYS, "smcb_backward_sample: no transition density for model 9, dim 1"),
    (5, 5, ENOSYS, "smcb_backward_sample: no transition density for model 5, dim 5"),
    (4, 3, EINVAL, "smcb_backward_sample: dim 3 does not match the model's 4"),
])
def test_backward_sample(env, model, dim, rc, msg):
    _lib, lib, ctx, p, _ = env
    d = _lib.SmoothDesc()
    d.method, d.model, d.dim = _lib.SMOOTH_ON2, model, dim
    d.T, d.N, d.M = 2, 4, 4
    d.X = d.idx = d.paths = d.lw = d.idx_T = p
    assert lib.smcb_backward_sample(ctx, C.byref(d)) == rc
    assert last_error(lib) == msg


@pytest.mark.parametrize("model, dim, rc, msg", [
    (9, 1, ENOSYS, "smcb_online_smooth: no transition density for model 9, dim 1"),
    (5, 5, ENOSYS, "smcb_online_smooth: no transition density for model 5, dim 5"),
    (4, 3, EINVAL, "smcb_online_smooth: dim 3 does not match the model's 4"),
])
def test_online_smooth(env, model, dim, rc, msg):
    _lib, lib, ctx, p, _ = env
    d = _lib.OnlineDesc()
    d.method, d.model, d.dim = _lib.ONLINE_PARIS, model, dim
    d.N, d.Np = 4, 1
    d.X_prev = d.X = d.lw_prev = d.B = d.counts = p
    assert lib.smcb_online_smooth(ctx, C.byref(d)) == rc
    assert last_error(lib) == msg
