"""Off-line smoothing on the CPU: the NumPy oracle's FFBS samplers and RTS smoother against the live reference's
output (tests/golden/golden_smoothing.npz, written by make_golden_smoothing.py), the host build of the device
transition density (TransDensity, csrc/smcb_models.cuh) against the oracle's PX(t, xp).logpdf(x), and the
recogniser that decides which models get the device density."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = C.c_void_p
_trans = None


def build_trans_host():
    """g++ build of tests/trans_host.cpp (the transition density of smcb_models.cuh compiled for the host)."""
    global _trans
    if _trans is None:
        import subprocess
        out = os.path.join(ROOT, "oracle", "_build")
        os.makedirs(out, exist_ok=True)
        so = os.path.join(out, "libtrans_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "particles_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "trans_host.cpp"), "-o", so])
        _trans = C.CDLL(so)
        _trans.mh_init()
    return _trans


@pytest.fixture(scope="module")
def gs():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_smoothing.npz"))


SEEDS = {"lg": 11, "sv": 12, "cox": 13, "mvlg2": 14}


def oracle_model(name):
    return {"lg": lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9),
            "sv": lambda: orc.StochVol(),
            "cox": lambda: orc.DiscreteCox(mu=0.0, sigma=0.5, phi=0.9),
            "mvlg2": lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[name]()


def history(gs, name):
    return {"X": list(gs[f"{name}/X"]), "lw": list(gs[f"{name}/lw"]), "A": list(gs[f"{name}/A"])}


@pytest.mark.parametrize("name", list(SEEDS))
def test_oracle_backward_samplers_reproduce_reference(gs, name):
    """Same history, same global-stream seed -> the reference's indices bit-for-bit, and its acc_rate."""
    h, logpt = history(gs, name), osm.px_logpt(oracle_model(name))
    M = int(gs["meta/T_N_M"][2])
    bound = gs[f"{name}/bound"]
    seed = SEEDS[name]
    state = np.random.get_state()
    try:
        np.random.seed(seed + 200)
        idx, _ = osm.backward_ON2(h, logpt, M)
        assert np.array_equal(idx, gs[f"{name}/idx_on2"])
        np.random.seed(seed + 300)
        idx, _ = osm.backward_mcmc(h, logpt, M, nsteps=2)
        assert np.array_equal(idx, gs[f"{name}/idx_mcmc"])
        np.random.seed(seed + 400)
        idx, acc, _ = osm.backward_reject(h, logpt, M, lambda t: bound[t])
        assert np.array_equal(idx, gs[f"{name}/idx_reject"])
        assert np.array_equal(acc, gs[f"{name}/acc_rate"])
        np.random.seed(seed + 500)
        idx, acc, noise = osm.backward_reject(h, logpt, M, lambda t: bound[t], max_trials=2)
        assert np.array_equal(idx, gs[f"{name}/idx_reject2"])
        assert np.array_equal(acc, gs[f"{name}/acc_rate2"])
        assert np.any(noise["u_exact"] > 0)              # the exact fallback was exercised
    finally:
        np.random.set_state(state)


@pytest.mark.parametrize("name", ["lg", "mvlg2"])
def test_oracle_rts_smoother_matches_reference_kalman(gs, name):
    model = oracle_model(name)
    if name == "lg":                                 # kalman.LinearGauss as the reference's MVLinearGauss parameters
        model.F, model.G, model.covX = np.array([[model.rho]]), np.eye(1), np.array([[model.sigmaX ** 2]])
        model.covY, model.mu0, model.cov0 = np.array([[model.sigmaY ** 2]]), np.zeros(1), np.array([[model.sigma0 ** 2]])
    mean, cov = osm.kalman_smoother(model, list(gs[f"{name}/data"]))
    np.testing.assert_allclose(mean, gs[f"{name}/kalman_mean"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(cov, gs[f"{name}/kalman_cov"], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------
# host build of the device transition density
# ---------------------------------------------------------------------------
def _trans_cases():
    from particles_b200 import kalman, state_space_models as ssm
    return [
        ("StochVol", ssm.StochVol(), orc.StochVol(), 1, "exact"),
        ("StochVolLeverage", ssm.StochVolLeverage(phi=-0.6), orc.StochVolLeverage(phi=-0.6), 1, "exact"),
        ("LinearGauss", kalman.LinearGauss(rho=0.9), orc.LinearGauss(rho=0.9), 1, "exact"),
        ("DiscreteCox", ssm.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), orc.DiscreteCox(mu=0.5, sigma=0.5, phi=0.9), 1,
         "exact"),
        ("ThetaLogistic", ssm.ThetaLogistic(), orc.ThetaLogistic(), 1, 1e-13),
        ("Gordon_etal", ssm.Gordon_etal(), orc.Gordon_etal(), 1, 1e-13),
        ("MVLinearGauss2", kalman.MVLinearGauss_Guarniero_etal(0.4, 2), orc.MVLinearGauss_Guarniero_etal(0.4, 2), 2,
         1e-11),
        ("MVLinearGauss4", kalman.MVLinearGauss_Guarniero_etal(0.4, 4), orc.MVLinearGauss_Guarniero_etal(0.4, 4), 4,
         1e-11),
        ("BearingsOnly", ssm.BearingsOnly(), orc.BearingsOnly(), 4, "dirac"),
    ]


@pytest.mark.parametrize("case", _trans_cases(), ids=lambda c: c[0])
def test_trans_logpdf_host_matches_oracle(case):
    from particles_b200 import state_space_models as ssm
    name, dev_m, orc_m, dim, tol = case
    lib = build_trans_host()
    T, n = 12, 400
    y = [np.array([1.0])] * T
    spec = ssm.transition_spec(ssm.Bootstrap(ssm=dev_m, data=y))
    assert spec is not None and spec["dim"] == dim, name
    r = np.random.RandomState(5)
    xp = r.standard_normal((n, dim)) if dim > 1 else r.standard_normal(n)
    if name == "BearingsOnly":
        xp = xp * 0.01 + np.array([0.0, 0.0, 1.0, 1.0])
        x = orc_m.PX(0, xp).rvs(n, r.standard_normal((n, 2)))
        x[::3, 2] += 1e-9                              # break one Dirac in three particles
        x[1::5, 3] = np.nextafter(x[1::5, 3], 2.0)     # and the other one by one ulp
    else:
        x = xp * 0.9 + r.standard_normal(xp.shape)
    params = np.ascontiguousarray(spec["params"], dtype=np.float64)
    sc = spec["step_consts"]
    sc = None if sc is None else np.ascontiguousarray(sc, dtype=np.float64)
    soa = lambda a: np.ascontiguousarray(a.reshape(n, -1).T)      # noqa: E731
    xp_s, x_s = soa(xp), soa(x)
    for t in (1, 5, T - 1):
        out = np.empty(n)
        rc = lib.mh_trans_logpdf(spec["model"], dim, params.ctypes.data_as(P),
                                 None if sc is None else sc.ctypes.data_as(P), C.c_long(t),
                                 xp_s.ctypes.data_as(P), x_s.ctypes.data_as(P), C.c_long(n), out.ctypes.data_as(P))
        assert rc == 0
        ref = orc_m.PX(t, xp).logpdf(x)
        if tol == "exact":
            assert np.array_equal(out, ref), (name, t, np.max(np.abs(out - ref)))
        elif tol == "dirac":
            assert np.array_equal(np.isinf(out), np.isinf(ref)) and np.isinf(ref).any() and np.isfinite(ref).any()
            np.testing.assert_allclose(out[np.isfinite(ref)], ref[np.isfinite(ref)], rtol=1e-15)
        else:
            np.testing.assert_allclose(out, ref, rtol=tol, atol=0)


def test_transition_spec_recogniser():
    from particles_b200 import _lib, state_space_models as ssm
    y = [np.array([1.0])] * 5

    class DiscreteCox_with_add_f(ssm.DiscreteCox):        # the book's smoothing scripts subclass in __main__
        def upper_bound_log_pt(self, t):
            return -0.5 * np.log(2 * np.pi)
    DiscreteCox_with_add_f.__module__ = "__main__"
    s = ssm.transition_spec(ssm.Bootstrap(ssm=DiscreteCox_with_add_f(), data=y))
    assert s is not None and s["model"] == _lib.MODEL_DISCRETECOX
    assert ssm.fused_spec(ssm.Bootstrap(ssm=DiscreteCox_with_add_f(), data=y)) is None    # the filter's rule is stricter

    class MyPX(ssm.DiscreteCox):
        def PX(self, t, xp):
            return ssm.DiscreteCox.PX(self, t, xp)
    MyPX.__module__ = "__main__"
    assert ssm.transition_spec(ssm.Bootstrap(ssm=MyPX(), data=y)) is None

    class MyLogpt(ssm.Bootstrap):
        def logpt(self, t, xp, x):
            return ssm.Bootstrap.logpt(self, t, xp, x)
    assert ssm.transition_spec(MyLogpt(ssm=ssm.DiscreteCox(), data=y)) is None
    for kind in ("GuidedPF", "AuxiliaryPF", "AuxiliaryBootstrap"):     # every kind inherits Bootstrap.logpt
        assert ssm.transition_spec(getattr(ssm, kind)(ssm=ssm.StochVol(), data=y))["model"] == _lib.MODEL_STOCHVOL
    g = ssm.transition_spec(ssm.Bootstrap(ssm=ssm.Gordon_etal(), data=y))
    assert np.array_equal(g["step_consts"], [8.0 * np.cos(1.2 * (t - 1)) for t in range(5)])


def test_bound_methods_follow_the_reference():
    from particles_b200 import state_space_models as ssm
    fk = ssm.Bootstrap(ssm=ssm.StochVol(), data=[np.zeros(1)] * 3)
    with pytest.raises(NotImplementedError, match="missing method upper_bound_log_pt"):
        fk.upper_bound_trans(1)

    class SV(ssm.StochVol):
        def upper_bound_log_pt(self, t):
            return 1.5
    assert ssm.Bootstrap(ssm=SV(), data=[np.zeros(1)]).upper_bound_trans(2) == 1.5
