"""Kalman filter and smoother of the LIVE reference (particles.kalman.Kalman) on eight linear-Gaussian models: the
data fixture that tests/test_kalman_host.py checks the NumPy oracle (tests/kalman_oracle.py) and the replay
(tests/kalman_replay.py) against and tests/test_gpu_kalman.py runs the device on.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_kalman.py

Cases: (a) the book's LinearGauss(sigmaX=1, sigmaY=.2, rho=.9), T = 100; (b) LinearGauss with rho = 1 and sigma0
given, T = 50; (c) the module docstring's model (dx = 2, dy = 1), T = 50; (d) Guarniero et al. with dx = 4,
T = 100; (e) a random model with dx = 5, dy = 3, non-zero mu0, cov0 != covX and a non-symmetric F, T = 60;
(f) dx = 3, dy = 7, T = 40; (g) dx = dy = 32, T = 6; (h) dx = dy = 2, T = 1.  For each: the model's six matrices,
the data (T, dy), and pred / filt / smth means (T, dx) and covariances (T, dx, dx) and logpyt (T,).  For (a) also
the smoothing means and covariances after each of the first 10 ``next()`` calls, rows concatenated.
Writes tests/golden/golden_kalman.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get("PARTICLES_REFERENCE", "/root/reference"))
from particles import kalman  # noqa: E402

STEPS = 10


def random_model(rng, dx, dy):
    A = rng.normal(size=(dx, dx))
    F = 0.9 * A / np.max(np.abs(np.linalg.eigvals(A)))

    def spd(d, s):
        M = rng.normal(size=(d, d))
        return s * (M @ M.T / d + np.eye(d))

    return kalman.MVLinearGauss(F=F, G=rng.normal(size=(dy, dx)) / np.sqrt(dx), covX=spd(dx, 0.5),
                                covY=spd(dy, 0.3), mu0=rng.normal(size=dx), cov0=spd(dx, 2.0))


def cases():
    rng = np.random.RandomState(20261019)
    return [("a", kalman.LinearGauss(sigmaX=1.0, sigmaY=0.2, rho=0.9), 100),
            ("b", kalman.LinearGauss(sigmaX=0.5, sigmaY=0.3, rho=1.0, sigma0=1.0), 50),
            ("c", kalman.MVLinearGauss(F=np.eye(2), G=np.ones((1, 2)), covX=np.eye(2), covY=0.3), 50),
            ("d", kalman.MVLinearGauss_Guarniero_etal(alpha=0.4, dx=4), 100),
            ("e", random_model(rng, 5, 3), 60),
            ("f", random_model(rng, 3, 7), 40),
            ("g", random_model(rng, 32, 32), 6),
            ("h", random_model(rng, 2, 2), 1)]


def stack(seq, T, dx):
    return (np.array([np.asarray(s.mean, float).reshape(dx) for s in seq]).reshape(T, dx),
            np.array([np.asarray(s.cov, float).reshape(dx, dx) for s in seq]).reshape(T, dx, dx))


def main():
    rec = {}
    for i, (name, m, T) in enumerate(cases()):
        np.random.seed(300 + i)
        _, y = m.simulate(T)
        dx, dy = m.dx, m.dy
        y = np.array(y, dtype=float).reshape(T, dy)
        kf = kalman.Kalman(ssm=m, data=list(y))
        kf.smoother()
        p = name + "_"
        for k in ("F", "G", "covX", "covY", "mu0", "cov0"):
            rec[p + k] = np.array(getattr(m, k), dtype=float)
        rec[p + "y"] = y
        for k in ("pred", "filt", "smth"):
            rec[p + k + "_mean"], rec[p + k + "_cov"] = stack(getattr(kf, k), T, dx)
        rec[p + "logpyt"] = np.array([np.asarray(v, float).reshape(-1)[0] for v in kf.logpyt])
        if name == "a":
            kf = kalman.Kalman(ssm=m, data=list(y))
            means, covs = [], []
            for _ in range(STEPS):
                kf.next()
                kf.smoother()
                sm, sc = stack(kf.smth, kf.t, dx)
                means.append(sm)
                covs.append(sc)
            rec["a_smth_steps_mean"], rec["a_smth_steps_cov"] = np.concatenate(means), np.concatenate(covs)
    np.savez_compressed(os.path.join(HERE, "golden_kalman.npz"), **rec)


if __name__ == "__main__":
    main()
