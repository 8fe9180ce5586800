"""Off-line smoothing (FFBS) of the LIVE reference on small seeded problems: the data fixture that
tests/test_smoothing_host.py checks the NumPy oracle (oracle/smoothing_numpy.py) against bit-for-bit, and that
tests/test_gpu_smoothing.py runs the device samplers on.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_smoothing.py

For each case: simulate data, run a seeded forward ``particles.SMC(store_history=True)``, then under fixed seeds
``backward_sampling_ON2``, ``backward_sampling_mcmc`` (nsteps = 2), ``backward_sampling_reject`` (default
max_trials and max_trials = 2, which exercises the exact fallback), recording the INDEX arrays (the reference
returns X[t][idx[t]]; the generator captures idx at _output_backward_sampling) and acc_rate; for the linear Gaussian
cases also the reference's Kalman smoother means and covariances.  Writes tests/golden/golden_smoothing.npz."""
import os
import sys

import numpy as np

sys.path.insert(0, "/root/reference")
import particles  # noqa: E402
from particles import kalman, smoothing  # noqa: E402
from particles import state_space_models as ssms  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
T, N, M = 50, 200, 100


class LinearGaussB(kalman.LinearGauss):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigmaX ** 2)


class StochVolB(ssms.StochVol):
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigma ** 2)


class DiscreteCoxB(ssms.DiscreteCox):          # the bound of the book's smoothing scripts
    def upper_bound_log_pt(self, t):
        return -0.5 * np.log(2.0 * np.pi * self.sigma ** 2)


class GuarnieroB(kalman.MVLinearGauss_Guarniero_etal):
    def upper_bound_log_pt(self, t):          # covX = I
        return -0.5 * self.dx * np.log(2.0 * np.pi)


CASES = [("lg", lambda: LinearGaussB(sigmaX=1.0, sigmaY=0.2, rho=0.9), 11),
         ("sv", lambda: StochVolB(), 12),
         ("cox", lambda: DiscreteCoxB(mu=0.0, sigma=0.5, phi=0.9), 13),
         ("mvlg2", lambda: GuarnieroB(alpha=0.4, dx=2), 14)]

smoothing.ParticleHistory._output_backward_sampling = lambda self, idx: idx     # capture the indices


def main():
    out = {}
    for name, make, seed in CASES:
        model = make()
        np.random.seed(seed)
        _, y = model.simulate(T)
        np.random.seed(seed + 100)
        pf = particles.SMC(fk=ssms.Bootstrap(ssm=model, data=y), N=N, store_history=True)
        pf.run()
        h = pf.hist
        out[f"{name}/data"] = np.array([np.asarray(v, dtype=float).reshape(-1) for v in y])
        out[f"{name}/X"] = np.array(h.X)
        out[f"{name}/lw"] = np.array([w.lw for w in h.wgts])
        out[f"{name}/A"] = np.array([np.zeros(N, dtype=np.int64)] + [np.asarray(a, dtype=np.int64) for a in h.A[1:]])
        np.random.seed(seed + 200)
        out[f"{name}/idx_on2"] = h.backward_sampling_ON2(M)
        np.random.seed(seed + 300)
        out[f"{name}/idx_mcmc"] = h.backward_sampling_mcmc(M, nsteps=2)
        np.random.seed(seed + 400)
        out[f"{name}/idx_reject"] = h.backward_sampling_reject(M)
        out[f"{name}/acc_rate"] = h.acc_rate.copy()
        np.random.seed(seed + 500)
        out[f"{name}/idx_reject2"] = h.backward_sampling_reject(M, max_trials=2)
        out[f"{name}/acc_rate2"] = h.acc_rate.copy()
        out[f"{name}/bound"] = np.array([model.upper_bound_log_pt(t) for t in range(T)])
        if name in ("lg", "mvlg2"):
            kf = kalman.Kalman(ssm=model, data=y)
            kf.smoother()
            out[f"{name}/kalman_mean"] = np.array([np.asarray(s.mean).reshape(-1) for s in kf.smth])
            out[f"{name}/kalman_cov"] = np.array([np.atleast_2d(s.cov) for s in kf.smth])
        print(name, "acc_rate", float(np.mean(h.acc_rate)), flush=True)
    out["meta/T_N_M"] = np.array([T, N, M])
    out["meta/seeds"] = np.array([s for _, _, s in CASES])
    np.savez_compressed(os.path.join(HERE, "golden_smoothing.npz"), **out)


if __name__ == "__main__":
    main()
