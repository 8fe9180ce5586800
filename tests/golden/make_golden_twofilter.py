"""Two-filter smoothing of the LIVE reference on small seeded problems: the data fixture that
tests/test_twofilter_host.py checks the NumPy oracle (tests/twofilter_oracle.py) against, and that
tests/test_gpu_twofilter.py runs the device estimators on.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_twofilter.py

For each case (the book's DiscreteCox with its ``psit`` and ``log_gamma``, a stationary LinearGauss, StochVol):
simulate T = 50 observations, run a seeded forward ``particles.SMC(store_history=True)`` and a seeded information
filter (the same model on the data in reverse), N = 200 particles for the book's model and 100 for the others, then
record
  - both histories (X, lw);
  - ``two_filter_smoothing`` O(N^2) at every t;
  - ``two_filter_smoothing(linear_cost=True, return_ess=True)`` at every t, without and with the book's ``_prop``
    modifiers (smoothing_worker, smoothing.py:649-660): the I and J the reference drew (captured by wrapping
    ``resampling.multinomial``, stored as int16), the estimates and the ESS;
  - for LinearGauss, the Kalman smoother means.
loggamma(Xinfo) and the modifier arrays are not stored: ``twofilter_oracle.log_gamma`` and ``prop_modifiers`` give
them bit for bit from the stored particles, and they are what the reference was fed here.
Writes tests/golden/golden_twofilter.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import twofilter_oracle as otf  # noqa: E402
import particles  # noqa: E402
from particles import kalman, smoothing  # noqa: E402
from particles import state_space_models as ssms  # noqa: E402

T = 50
MU, PHI, SIGMA = 0.0, 0.9, 0.5


def psit(t, x, xf, mu=MU, phi=PHI, sigma=SIGMA):
    """The book's additive function (book/smoothing/offline_smoothing.py): the score at theta_0."""
    if t == 0:
        return (-0.5 / sigma ** 2 + (0.5 * (1.0 - phi ** 2) / sigma ** 4) * (x - mu) ** 2
                + psit(1, x, xf, mu, phi, sigma))
    return -0.5 / sigma ** 2 + (0.5 / sigma ** 4) * ((xf - mu) - phi * (x - mu)) ** 2


class DiscreteCox_with_add_f(ssms.DiscreteCox):     # the book's model (its bound enters the ON2 shift)
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2 * np.pi * self.sigma ** 2)


class LinearGaussB(kalman.LinearGauss):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigmaX ** 2)


class StochVolB(ssms.StochVol):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigma ** 2)


def product(t, x, xf):
    return x * xf


CASES = [("cox", lambda: DiscreteCox_with_add_f(mu=MU, phi=PHI, sigma=SIGMA), psit, 200, 31),
         ("lg", lambda: LinearGaussB(sigmaX=1.0, sigmaY=0.5, rho=0.9), product, 100, 32),
         ("sv", lambda: StochVolB(), product, 100, 33)]

_draws = []
_multinomial = smoothing.rs.multinomial


def _capture(W, M=None):
    A = _multinomial(W) if M is None else _multinomial(W, M)
    _draws.append(np.asarray(A, dtype=np.int64).copy())
    return A


smoothing.rs.multinomial = _capture


def main():
    out = {}
    for name, make, add_func, N, seed in CASES:
        model = make()
        log_gamma = lambda x, name=name: otf.log_gamma(name, x)      # noqa: E731
        np.random.seed(seed)
        _, y = model.simulate(T)
        np.random.seed(seed + 100)
        pf = particles.SMC(fk=ssms.Bootstrap(ssm=model, data=y), N=N, store_history=True)
        pf.run()
        np.random.seed(seed + 200)
        info = particles.SMC(fk=ssms.Bootstrap(ssm=model, data=y[::-1]), N=N, store_history=True)
        info.run()
        h, ih = pf.hist, info.hist
        out[f"{name}/data"] = np.array([np.asarray(v, dtype=float).reshape(-1) for v in y])
        out[f"{name}/X"] = np.array(h.X)
        out[f"{name}/lw"] = np.array([w.lw for w in h.wgts])
        out[f"{name}/Xinfo"] = np.array(ih.X)
        out[f"{name}/lwinfo"] = np.array([w.lw for w in ih.wgts])
        on2 = np.zeros(T - 1)
        for t in range(T - 1):
            on2[t] = h.two_filter_smoothing(t, info, lambda x, xf: add_func(t, x, xf), log_gamma)
        out[f"{name}/on2"] = on2
        for tag in ("on", "prop"):
            est, ess = np.zeros(T - 1), np.zeros(T - 1)
            I, J = np.zeros((T - 1, N), dtype=np.int64), np.zeros((T - 1, N), dtype=np.int64)
            np.random.seed(seed + (300 if tag == "on" else 400))
            for t in range(T - 1):
                kw = {}
                if tag == "prop":           # smoothing.py:649-660
                    mf, mi = otf.prop_modifiers(np.array(h.X), np.array(ih.X), t)
                    kw = {"modif_forward": mf, "modif_info": mi}
                del _draws[:]
                est[t], ess[t] = h.two_filter_smoothing(t, info, lambda x, xf: add_func(t, x, xf), log_gamma,
                                                        linear_cost=True, return_ess=True, **kw)
                assert len(_draws) == 2
                I[t], J[t] = _draws
            out[f"{name}/{tag}_est"], out[f"{name}/{tag}_ess"] = est, ess
            out[f"{name}/{tag}_I"], out[f"{name}/{tag}_J"] = I.astype(np.int16), J.astype(np.int16)
        if name == "lg":
            kf = kalman.Kalman(ssm=model, data=y)
            kf.smoother()
            out[f"{name}/kalman_mean"] = np.array([float(np.asarray(s.mean).reshape(-1)[0]) for s in kf.smth])
        print(name, "on2[:3]", on2[:3], "on[:3]", out[f"{name}/on_est"][:3], flush=True)
    out["meta/T"] = np.array([T])
    out["meta/seeds"] = np.array([s for *_, s in CASES])
    np.savez_compressed(os.path.join(HERE, "golden_twofilter.npz"), **out)


if __name__ == "__main__":
    main()
