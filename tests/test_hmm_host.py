"""Host checks of the Baum-Welch test infrastructure: the NumPy oracle (tests/hmm_oracle.py) reproduces the live
reference's fixture (tests/golden/golden_hmm.npz) bit for bit, trajectory draws included, and the long-double
replay of the device algorithm (tests/hmm_replay.py) agrees with the oracle to 1e-13."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hmm_oracle as oh  # noqa: E402
import hmm_replay as rp  # noqa: E402

CASES = ("a", "b", "c", "d", "e")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_hmm.npz"))


def model(g, c):
    return g[c + "_init"], g[c + "_trans"], g[c + "_mus"], g[c + "_sigmas"], g[c + "_y"]


@pytest.mark.parametrize("c", CASES)
def test_oracle_reproduces_reference(g, c):
    init, trans, mus, sigmas, y = model(g, c)
    out = oh.run(init, trans, mus, sigmas, y)
    for k in ("logft", "pred", "filt", "logpyt", "smth"):
        np.testing.assert_array_equal(out[k], g[c + "_" + k], err_msg=k)


@pytest.mark.parametrize("c", CASES)
def test_oracle_paths_from_regenerated_uniforms(g, c):
    init, trans, mus, sigmas, y = model(g, c)
    N = int(g["N_sample"])
    last, U = oh.reference_uniforms(int(g[c + "_sample_seed"]), N, y.shape[0])
    with np.errstate(divide="ignore"):
        paths = oh.sample(trans, g[c + "_filt"], last, U)
    np.testing.assert_array_equal(paths, g[c + "_paths"])


def test_oracle_incremental_smoothing(g):
    init, trans, mus, sigmas, y = model(g, "a")
    rows = []
    for i in range(30):
        rows.append(oh.run(init, trans, mus, sigmas, y[:i + 1])["smth"])
    np.testing.assert_array_equal(np.concatenate(rows), g["a_smth_steps"])


@pytest.mark.parametrize("c", CASES)
def test_replay_agrees_with_oracle(g, c):
    init, trans, mus, sigmas, y = model(g, c)
    out = rp.run(init, trans, g[c + "_logft"])
    for k in ("pred", "filt", "logpyt", "smth"):
        np.testing.assert_allclose(out[k].astype(float), g[c + "_" + k], rtol=0, atol=1e-13, err_msg=k)


def test_replay_group_sum_order():
    v = np.arange(1, 70, dtype=np.longdouble)
    assert rp.group_sum(v) == v.sum()
    v = np.array([1e16, 1.0, -1e16] + [0.0] * 13 + [1.0], dtype=np.float64)
    # the padded lanes add exact zeros: only the fold order of the K live lanes matters
    assert rp.group_sum(v) == 2.0


def test_replay_samples_follow_cdf():
    trans = np.array([[0.5, 0.5], [0.1, 0.9]])
    filt = np.array([[0.3, 0.7], [0.6, 0.4]])
    U = np.array([[0.0, 0.999999]])
    paths, gap = rp.sample(trans, filt, np.array([0, 1]), U)
    assert paths[0, 0] == 0 and paths[0, 1] == 1 and np.all(gap[0] >= 0)
    u = rp.device_uniforms(7, 5, 3)
    assert u.shape == (2, 5) and np.all((u >= 0) & (u < 1))
