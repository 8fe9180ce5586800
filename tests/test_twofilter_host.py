"""Two-filter smoothing on the CPU: the NumPy oracle (tests/twofilter_oracle.py) against the live reference's
estimates (tests/golden/golden_twofilter.npz, written by make_golden_twofilter.py), and smoothing_worker's
method table."""
import os
import sys

import numpy as np
import pytest

from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import twofilter_oracle as otf  # noqa: E402

MU, PHI, SIGMA = 0.0, 0.9, 0.5
CASES = ("cox", "lg", "sv")


def psit(t, x, xf, mu=MU, phi=PHI, sigma=SIGMA):
    """The book's additive function (book/smoothing/offline_smoothing.py)."""
    if t == 0:
        return (-0.5 / sigma ** 2 + (0.5 * (1.0 - phi ** 2) / sigma ** 4) * (x - mu) ** 2
                + psit(1, x, xf, mu, phi, sigma))
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((xf - mu) - phi * (x - mu)) ** 2


def add_func(name):
    return psit if name == "cox" else (lambda t, x, xf: x * xf)


def oracle_model(name):
    return {"cox": lambda: orc.DiscreteCox(mu=MU, sigma=SIGMA, phi=PHI),
            "lg": lambda: orc.LinearGauss(sigmaX=1.0, sigmaY=0.5, rho=0.9),
            "sv": lambda: orc.StochVol()}[name]()


def upper_bound(name):
    m = oracle_model(name)
    sigma = m.sigmaX if name == "lg" else m.sigma
    return -0.5 * np.log(2.0 * np.pi * sigma ** 2)


@pytest.fixture(scope="module")
def gt():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_twofilter.npz"))


def _lwinfo(gt, name, ti):
    return gt[f"{name}/lwinfo"][ti] - otf.log_gamma(name, gt[f"{name}/Xinfo"][ti])


@pytest.mark.parametrize("name", CASES)
def test_oracle_on2_reproduces_reference(gt, name):
    T = int(gt["meta/T"][0])
    X, lw, Xi = gt[f"{name}/X"], gt[f"{name}/lw"], gt[f"{name}/Xinfo"]
    logpt, f = osm.px_logpt(oracle_model(name)), add_func(name)
    for t in range(T - 1):
        ti = T - 2 - t
        phi = lambda x, xf: f(t, x, xf)          # noqa: E731
        est = otf.on2(t, X[t], lw[t], Xi[ti], _lwinfo(gt, name, ti), logpt, phi, upper_bound(name))
        np.testing.assert_allclose(est, gt[f"{name}/on2"][t], rtol=1e-12, atol=0)
        rows = otf.on2_rows(t, X[t], lw[t], Xi[ti], _lwinfo(gt, name, ti), logpt, phi, chunk=37)
        np.testing.assert_allclose(rows, gt[f"{name}/on2"][t], rtol=1e-12, atol=0)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("tag", ["on", "prop"])
def test_oracle_on_given_draws_is_bit_exact(gt, name, tag):
    T = int(gt["meta/T"][0])
    X, Xi = gt[f"{name}/X"], gt[f"{name}/Xinfo"]
    logpt, f = osm.px_logpt(oracle_model(name)), add_func(name)
    for t in range(T - 1):
        ti = T - 2 - t
        mods = {}
        if tag == "prop":
            mf, mi = otf.prop_modifiers(X, Xi, t)
            mods = {"modif_forward": mf, "modif_info": mi}
        I, J = gt[f"{name}/{tag}_I"][t].astype(np.int64), gt[f"{name}/{tag}_J"][t].astype(np.int64)
        est, ess = otf.on_given(t, X[t], Xi[ti], I, J, logpt,
                                lambda x, xf: f(t, x, xf), **mods)
        assert est == gt[f"{name}/{tag}_est"][t], (t, est, gt[f"{name}/{tag}_est"][t])
        assert ess == gt[f"{name}/{tag}_ess"][t]


def test_golden_draws_fit_their_histories(gt):
    """The fixture's int16 indices cover each case's N (200 for the book's model, 100 for the others)."""
    for name, n in (("cox", 200), ("lg", 100), ("sv", 100)):
        assert gt[f"{name}/X"].shape == gt[f"{name}/Xinfo"].shape == (int(gt["meta/T"][0]), n)
        for tag in ("on", "prop"):
            for k in ("I", "J"):
                a = gt[f"{name}/{tag}_{k}"]
                assert a.dtype == np.int16 and a.min() >= 0 and a.max() < n


def test_smoothing_worker_method_table():
    """The reference's eight method names; the ones this package cannot run refuse before any device work."""
    from particles_b200 import smoothing
    assert set(smoothing.WORKER_METHODS) == {"FFBS_purereject", "FFBS_hybrid", "FFBS_MCMC", "FFBS_ON2",
                                             "FFBS_QMC", "two-filter_ON", "two-filter_ON_prop", "two-filter_ON2"}
    with pytest.raises(NotImplementedError, match="SQMC"):
        smoothing.smoothing_worker(method="FFBS_QMC", N=10)
    with pytest.raises(ValueError, match="no such method"):
        smoothing.smoothing_worker(method="two-filter_ON3", N=10)
    assert smoothing._PURE_REJECT_TRIALS == (1 << 24) - 1     # the device samplers' max_trials bound
    import inspect
    assert list(inspect.signature(smoothing.smoothing_worker).parameters) == [
        "method", "N", "fk", "fk_info", "add_func", "log_gamma"]
