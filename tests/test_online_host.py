"""On-line smoothing on the CPU: the NumPy oracle of the naive, O(N^2) and PaRIS collectors (tests/online_oracle.py)
against the live reference's output (tests/golden/golden_online.npz, written by make_golden_online.py)."""
import os

import numpy as np
import pytest

import online_oracle as oo
from oracle import smc_numpy as orc
from oracle import smoothing_numpy as osm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARIS = [("paris", 2, None), ("paris2", 3, 2)]


@pytest.fixture(scope="module")
def go():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_online.npz"))


def oracle_model(name):
    return {"lg": lambda: orc.LinearGauss(**oo.PARAMS["lg"]), "sv": lambda: orc.StochVol(),
            "cox": lambda: orc.DiscreteCox(**oo.PARAMS["cox"]),
            "mvlg2": lambda: orc.MVLinearGauss_Guarniero_etal(0.4, 2)}[name]()


@pytest.mark.parametrize("name", list(oo.SEEDS))
def test_oracle_online_smoothers_reproduce_reference(go, name):
    """Same history, same global-stream seeds -> the reference's summaries and nprop bit for bit."""
    m = oracle_model(name)
    h, f, logpt, bound = oo.history(go, name), oo.add_func(name, m), osm.px_logpt(m), oo.log_bound(name, m)
    seed = oo.SEEDS[name]
    np.random.seed(seed + 200)
    assert np.array_equal(np.array(oo.naive(h, f), dtype=float), go[f"{name}/naive"])
    np.random.seed(seed + 201)
    assert np.array_equal(np.array(oo.on2(h, f, logpt), dtype=float), go[f"{name}/on2"])
    for i, (key, Np, mt) in enumerate(PARIS):
        np.random.seed(seed + 202 + i)
        summ, nprop, Bs, noises = oo.paris(h, f, logpt, bound, Nparis=Np, max_trials=mt)
        assert np.array_equal(np.array(summ, dtype=float), go[f"{name}/{key}"])
        assert np.array_equal(np.array(nprop, dtype=float), go[f"{name}/{key}_nprop"])
        assert len(Bs) == len(h["X"]) - 1 and Bs[0].shape == (h["X"][0].shape[0], Np)
        if mt == 2:          # the exact fallback ran
            assert any(nz["u_exact"].any() for nz in noises)
