"""The model / Feynman-Kac maps of the fused step kernel (particles_b200/csrc/smcb_models.cuh), compiled for
the CPU by tests/math_host.cpp and driven with the constants particles_b200.state_space_models builds for
the device, against the oracle's closures: same normals in, same particles / log-weight increments / logeta
out, for every fused (model, Feynman-Kac kind) pair.  No resampling here (ESSrmin = 0): resampling parity is
the GPU tests' business.  Runs for the default math and for the table-assisted variants."""
import ctypes as C

import numpy as np
import pytest

from oracle import smc_numpy as orc
from test_math_host import build_math_host

P = C.c_void_p


def ptr(a):
    return None if a is None else a.ctypes.data_as(P)


@pytest.fixture(scope="module")
def mh(request):
    lib = build_math_host()
    lib.mh_model_step.restype = C.c_int
    return lib


def lst(y):
    return [np.atleast_1d(v) for v in y]


def cases(golden, golden_stats):
    from particles_b200 import kalman, state_space_models as ssm
    sv, lg = (ssm.StochVol(), orc.StochVol()), (kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
                                                 orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9))
    y_sv, y_lg = lst(golden["data/sv_seed1_T1000"][:40]), lst(golden["data/lg_seed2_T100"][:40])
    out = []
    for kind in ("Bootstrap", "GuidedPF", "AuxiliaryPF", "AuxiliaryBootstrap"):
        out.append((f"sv-{kind}", sv, y_sv, kind, 1))
        out.append((f"lg-{kind}", lg, y_lg, kind, 1))
    out += [
        ("gordon", (ssm.Gordon_etal(), orc.Gordon_etal()), lst(golden["data/gordon_seed3_T50"]), "Bootstrap", 1),
        ("thetalogistic", (ssm.ThetaLogistic(), orc.ThetaLogistic()), lst(golden["data/thetalogistic_seed4_T50"]), "Bootstrap", 1),
        ("cox", (ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), orc.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9)),
         lst(golden["data/cox_seed6_T60"]), "Bootstrap", 1),
        ("svlev", (ssm.StochVolLeverage(phi=-0.6), orc.StochVolLeverage(phi=-0.6)), lst(golden["data/svlev_seed7_T60"]), "Bootstrap", 1),
        ("bearings", (ssm.BearingsOnly(), orc.BearingsOnly()), list(golden_stats["data/bearings_seed0_T40"].reshape(-1, 1)), "Bootstrap", 2),
    ]
    ym = list(golden_stats["data/mvlg_seed5_T30"])
    for kind in ("Bootstrap", "GuidedPF", "AuxiliaryPF", "AuxiliaryBootstrap"):
        out.append((f"mvlg4-{kind}", (kalman.MVLinearGauss_Guarniero_etal(0.4, 4), orc.MVLinearGauss_Guarniero_etal(0.4, 4)),
                    ym, kind, 4))
    return out


def test_fused_model_maps_vs_oracle(mh, golden, golden_stats):
    from particles_b200 import state_space_models as ssm
    N = 500
    for name, (dev_m, orc_m), y, kind, nz in cases(golden, golden_stats):
        spec = ssm.fused_spec(getattr(ssm, kind)(ssm=dev_m, data=y))
        assert spec is not None, name
        fk_o = getattr(orc, kind)(orc_m, y)
        T, dim, dy = len(y), int(spec.get("dim", 1)), int(spec.get("dy", 1))
        r = np.random.RandomState(11)
        z = r.standard_normal((T, N)) if nz == 1 and dim == 1 else r.standard_normal((T, N, nz))
        with np.errstate(all="ignore"):
            ref = orc.SMC(fk_o, N=N, ESSrmin=0.0, noise=orc.InjectedNoise(z, [np.zeros(1)] * T))
            params = np.ascontiguousarray(spec["params"], dtype=np.float64)
            data = np.ascontiguousarray(spec["data"], dtype=np.float64).reshape(-1)
            sc = spec.get("step_consts")
            sc = None if sc is None else np.ascontiguousarray(sc, dtype=np.float64)
            x = lw = None
            for t in range(T):
                ref.step()
                assert not ref.rs_flag
                zt = np.ascontiguousarray(z[t].reshape(N, -1).T)               # (NZ, n) as on the device
                xn, delta, leta = np.empty((dim, N)), np.empty(N), np.empty(N)
                rc = mh.mh_model_step(spec["model"], spec["fk"], dim, ptr(params), ptr(data), C.c_long(T), dy, ptr(sc),
                                      C.c_long(t), ptr(x), ptr(zt), C.c_long(N), ptr(xn), ptr(delta), ptr(leta))
                assert rc == 0, (name, rc)
                delta = np.where(np.isnan(delta), -np.inf, delta)                # resampling.py:220
                lw = delta if lw is None else lw + delta
                x = xn
                X = xn[0] if dim == 1 else xn.T
                np.testing.assert_allclose(X, ref.X, rtol=1e-11, atol=1e-13, err_msg=f"{name} t={t} X")
                np.testing.assert_allclose(lw, ref.wgts.lw, rtol=1e-10, atol=1e-10, err_msg=f"{name} t={t} lw")
                if fk_o.isAPF and t + 1 < T:
                    np.testing.assert_allclose(leta, fk_o.logeta(t, ref.X), rtol=1e-9, atol=1e-9,
                                               err_msg=f"{name} t={t} logeta")
            if name == "sv-Bootstrap":      # pure IEEE arithmetic in the state map: bit-identical particles
                assert np.array_equal(X, ref.X)


def test_unfused_combinations_answer_enosys(mh):
    z = np.zeros((1, 4))
    out = np.empty((1, 4))
    d = np.empty(4)
    data = np.zeros(2)
    rc = mh.mh_model_step(4, 1, 4, ptr(np.zeros(16)), ptr(data), C.c_long(2), 1, None, C.c_long(0), None, ptr(z),
                          C.c_long(4), ptr(out), ptr(d), None)          # BearingsOnly has no proposal
    assert rc == -3

    def step(model, fk, dim):
        return mh.mh_model_step(model, fk, dim, ptr(np.zeros(64)), ptr(data), C.c_long(2), 1, None, C.c_long(0), None,
                                ptr(z), C.c_long(4), ptr(out), ptr(d), ptr(np.empty(4)))

    assert step(8, 0, 1) == -3 and step(-1, 0, 1) == -3                 # unknown model ids
    assert step(0, 4, 1) == -3                                          # unknown Feynman-Kac kind
    assert step(5, 0, 5) == -3 and step(5, 0, 1) == -3                  # MVLinearGauss is fused for dx = 2, 3, 4
    # Gordon, ThetaLogistic, BearingsOnly, DiscreteCox, StochVolLeverage: no proposal / logeta, so bootstrap only
    for model, dim in ((2, 1), (3, 1), (4, 4), (6, 1), (7, 1)):
        for fk in (1, 2, 3):
            assert step(model, fk, dim) == -3, (model, fk)
