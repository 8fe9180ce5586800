"""Host checks of the Kalman test infrastructure and of ``particles_b200.kalman``'s host logic: the NumPy oracle
(tests/kalman_oracle.py) and the long-double replay of the device algorithm (tests/kalman_replay.py) against the
live reference's fixture (tests/golden/golden_kalman.npz); batched models, their refusals, the data-shape rules and
the dimension bound, all without a GPU."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kalman_oracle as ko  # noqa: E402
import kalman_replay as rp  # noqa: E402
from oracle import smoothing_numpy as sn  # noqa: E402
from particles_b200 import kalman, state_space_models as ssm  # noqa: E402

CASES = "abcdefgh"
PARAMS = ("F", "G", "covX", "covY", "mu0", "cov0")
FIELDS = ("pred_mean", "pred_cov", "filt_mean", "filt_cov", "logpyt", "smth_mean", "smth_cov")
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_kalman.npz"))


class _Model:
    def __init__(self, g, c):
        for k in PARAMS:
            setattr(self, k, g[c + "_" + k])


def rel(a, ref):
    """max |a - ref| over max |ref|: the error of a field in units of its own scale."""
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(a - ref)) / max(np.max(np.abs(ref)), np.finfo(float).tiny))


@pytest.mark.parametrize("c", CASES)
def test_oracle_reproduces_reference(g, c):
    """The oracle runs the reference's array operations; it departs from the fixture only where BLAS picks another
    kernel for the gain's memory layout (the reference solves with overwrite_b=True): a few ulp of each field's
    scale (observed <= 2), bounded by 32."""
    y = list(g[c + "_y"])
    pred, filt, logpyt = ko.kalman_filter(_Model(g, c), y)
    sm, sc = ko.kalman_smoother(_Model(g, c), y)
    got = {"pred_mean": [p[0] for p in pred], "pred_cov": [p[1] for p in pred], "filt_mean": [f[0] for f in filt],
           "filt_cov": [f[1] for f in filt], "logpyt": logpyt, "smth_mean": sm, "smth_cov": sc}
    for k in FIELDS:
        assert rel(got[k], g[c + "_" + k]) <= 32 * EPS, k


def test_oracle_incremental_smoothing(g):
    T = 10
    means, covs = [], []
    for i in range(T):
        sm, sc = ko.kalman_smoother(_Model(g, "a"), list(g["a_y"][:i + 1]))
        means.append(sm.reshape(i + 1, 1))
        covs.append(sc.reshape(i + 1, 1, 1))
    assert rel(np.concatenate(means), g["a_smth_steps_mean"]) <= 32 * EPS
    assert rel(np.concatenate(covs), g["a_smth_steps_cov"]) <= 32 * EPS


@pytest.mark.parametrize("c", CASES)
def test_oracle_smoother_is_the_existing_oracle(g, c):
    """tests/kalman_oracle.py's filter feeds the smoother the very bits of oracle/smoothing_numpy.kalman_smoother."""
    y = list(g[c + "_y"])
    for a, b in zip(ko.kalman_smoother(_Model(g, c), y), sn.kalman_smoother(_Model(g, c), y)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("c", CASES)
def test_replay_agrees_with_fixture(g, c):
    """Long double in the device's order against LAPACK's fp64 order.  Observed <= 1.5e-14 of each field's scale
    (case a's filtering variance, where P - K G P cancels 40-fold); the bound 1e-12 is the GPU tests' own."""
    out = rp.run(*(g[c + "_" + k] for k in PARAMS), g[c + "_y"])
    for k in FIELDS:
        assert rel(out[k][0].astype(np.float64), g[c + "_" + k]) <= 1e-12, k


@pytest.mark.parametrize("c", CASES)
def test_fp64_replay_rounding_is_small(g, c):
    """The fp64 replay performs the device's roundings: its distance to the long-double replay is the device's
    expected error on the fixture's cases: observed <= 1.5e-14 of each field's scale (case a's 40-fold cancellation
    again), an order of magnitude under the GPU tests' 1e-12 even at the bound of 1e-13."""
    args = [g[c + "_" + k] for k in PARAMS] + [g[c + "_y"]]
    ld, f64 = rp.run(*args), rp.run(*args, dtype=np.float64)
    for k in FIELDS:
        assert rel(f64[k], ld[k].astype(np.float64)) <= 1e-13, k


def test_replay_cholesky_and_nan():
    A = np.array([[[4.0, 2.0], [2.0, 3.0]]])
    L = rp.chol(A.astype(rp.LD), rp.LD)
    assert np.allclose((L[0] @ L[0].T).astype(float), A[0], rtol=0, atol=1e-15)
    x = rp.chol_solve_rows(L, np.array([[[1.0, 2.0]]], rp.LD), rp.LD)
    assert np.allclose(A[0] @ x[0, 0].astype(float), [1.0, 2.0], rtol=0, atol=1e-15)
    L = rp.chol(np.array([[[1.0, 2.0], [2.0, 1.0]]], rp.LD), rp.LD)
    assert np.isnan(float(L[0, 1, 1]))
    out = rp.run(1.0, 1.0, 1.0, -2.0, 0.0, 1.0, np.zeros((1, 3, 1)))          # S = 1 + 1 - 2 = 0 at t = 0
    assert np.all(np.isnan(out["filt_mean"].astype(float))) and np.all(np.isnan(out["logpyt"].astype(float)))


# ------------------------------------------------------------------------------------------------------------------
# batched models
# ------------------------------------------------------------------------------------------------------------------
def test_batched_mvlineargauss():
    B, dx, dy = 5, 3, 2
    covX = np.broadcast_to(np.eye(dx), (B, dx, dx)).copy()
    m = kalman.MVLinearGauss(F=0.5 * np.eye(dx), G=np.ones((dy, dx)), covX=covX, covY=np.eye(dy))
    assert m.batch == B and (m.dx, m.dy) == (dx, dy) and m.cov0.shape == (B, dx, dx) and m.mu0.shape == (dx,)
    assert kalman.MVLinearGauss(covX=np.eye(2), covY=1.0, mu0=np.zeros((4, 2))).batch == 4
    assert kalman.MVLinearGauss(covX=np.eye(2), covY=1.0).batch is None
    with pytest.raises(ValueError, match="disagree"):
        kalman.MVLinearGauss(covX=np.zeros((3, 2, 2)) + np.eye(2), covY=np.ones((4, 1, 1)))
    with pytest.raises(ValueError, match="shape"):
        kalman.MVLinearGauss(covX=np.zeros((3, 2, 2)) + np.eye(2), covY=1.0, F=np.eye(3))


def test_batched_lineargauss():
    rho = np.array([0.1, 0.5, 0.9])
    m = kalman.LinearGauss(rho=rho, sigmaX=np.array([1.0, 2.0, 3.0]))
    assert m.batch == 3 and m.F.shape == (3, 1, 1) and m.covY.shape == (3, 1, 1) and m.G.shape == (1, 1)
    np.testing.assert_array_equal(m.sigma0, np.array([1.0, 2.0, 3.0]) / np.sqrt(1.0 - rho ** 2))
    np.testing.assert_array_equal(m.cov0[:, 0, 0], m.sigma0 ** 2)
    np.testing.assert_array_equal(m.covY[:, 0, 0], np.full(3, 0.2 ** 2))
    one = kalman.LinearGauss(rho=np.array([0.5]))
    assert one.batch is None and one.F.shape == (1, 1)
    assert kalman.LinearGauss(rho=0.5, sigma0=np.array([1.0, 2.0])).batch == 2
    with pytest.raises(ValueError, match="one or B"):
        kalman.LinearGauss(rho=np.array([0.1, 0.2]), sigmaX=np.array([1.0, 2.0, 3.0]))


@pytest.mark.parametrize("make", [lambda: kalman.LinearGauss(rho=np.array([0.1, 0.5])),
                                  lambda: kalman.MVLinearGauss(covX=np.ones((2, 1, 1)), covY=1.0)])
def test_batched_model_refuses_the_particle_path(make):
    m = make()
    calls = {"PX0": lambda: m.PX0(), "PX": lambda: m.PX(1, np.zeros(3)), "PY": lambda: m.PY(1, None, np.zeros(3)),
             "proposal0": lambda: m.proposal0([0.0]), "proposal": lambda: m.proposal(1, np.zeros(3), [0.0, 0.0]),
             "logeta": lambda: m.logeta(0, np.zeros(3), [0.0, 0.0]), "simulate": lambda: m.simulate(3)}
    for name, call in calls.items():
        with pytest.raises(ValueError, match="Kalman"):
            call()
    with pytest.raises(ValueError, match="Kalman"):
        ssm.fused_spec(ssm.Bootstrap(ssm=m, data=[0.0, 1.0]))


# ------------------------------------------------------------------------------------------------------------------
# data-shape rules and the dimension bound (host logic of Kalman, before any device work)
# ------------------------------------------------------------------------------------------------------------------
def test_model_layout():
    dx, dy, B, _ = kalman.model_layout(kalman.LinearGauss())
    assert (dx, dy, B) == (1, 1, None)
    assert kalman.model_layout(kalman.LinearGauss(rho=np.array([0.1, 0.2, 0.3])))[2] == 3
    assert kalman.model_layout(kalman.MVLinearGauss_Guarniero_etal(dx=4))[:3] == (4, 4, None)

    class Odd:                                        # duck typing: any object with the six attributes
        F, G, covX, covY, mu0, cov0 = np.eye(2), np.ones((1, 2)), np.eye(2), 0.3, np.zeros(2), np.eye(2)
    assert kalman.model_layout(Odd())[:3] == (2, 1, None)
    Odd.G = np.ones((2, 2))
    with pytest.raises(ValueError, match="G has shape"):
        kalman.model_layout(Odd())


def test_data_layout_and_rows():
    y = np.arange(12.0)
    assert kalman.data_layout(y, None, 1) == (False, 12)
    assert kalman.data_layout(y.reshape(6, 2), None, 2) == (False, 6)
    assert kalman.data_layout(list(y.reshape(6, 1, 2)), None, 2) == (False, 6)
    assert kalman.data_layout(y.reshape(6, 2), 3, 2) == (False, 6)            # 2-D: shared even by a batch
    assert kalman.data_layout(y.reshape(3, 2, 2), 3, 2) == (True, 2)           # (B, T, dy): per model
    assert kalman.data_layout(y.reshape(3, 4, 1), None, 1) == (False, 3)       # 3-D without a batch: T rows
    with pytest.raises(ValueError, match="per-model"):
        kalman.data_layout(y.reshape(2, 3, 2), 3, 2)
    np.testing.assert_array_equal(kalman.data_rows(y.reshape(6, 2), False, 1, 3, 2), [[[2, 3], [4, 5]]])
    np.testing.assert_array_equal(kalman.data_rows(y.reshape(3, 2, 2), True, 1, 2, 2), y.reshape(3, 2, 2)[:, 1:])
    rows = [np.array([1.0]), 2.0, np.array([[3.0]])]
    np.testing.assert_array_equal(kalman.data_rows(rows, False, 0, 3, 1), [[[1.0], [2.0], [3.0]]])
    with pytest.raises(ValueError, match="hold 2"):
        kalman.data_rows(y, False, 0, 3, 2)


@pytest.mark.parametrize("dx,dy", [(33, 1), (1, 33), (40, 40)])
def test_dimension_bound_before_any_launch(dx, dy):
    m = kalman.MVLinearGauss(F=np.eye(dx), G=np.ones((dy, dx)), covX=np.eye(dx), covY=np.eye(dy))
    with pytest.raises(NotImplementedError, match="32"):
        kalman.Kalman(ssm=m, data=np.zeros((3, dy)))
