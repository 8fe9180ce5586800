"""numpy restatement of the reference's particle MCMC (particles/mcmc.py; TEST INFRASTRUCTURE, see
``oracle/__init__.py``): the conditional SMC with its history, the trajectory draws, the adaptive random-walk
Metropolis of PMMH and the Gibbs loop.  Citations are relative to the reference's root.

``CSMC`` follows mcmc.py:453-475 with one correction: the pinned particle is weighted by logG(t, x*[t-1], x*[t]),
where the reference leaves Xp[0] at the discarded resampled ancestor.  For the Bootstrap kind of the models whose PY
ignores xp the two agree, so with the global stream (``noise=None``) it reproduces the reference bit for bit.  With
``InjectedNoise`` it consumes the device kernel's layout: z[t] (N,) normals, u[t] (N + 1,) spacing uniforms."""
import numpy as np
from scipy.linalg import LinAlgError, cholesky

from . import smc_numpy as orc
from .smoothing_numpy import backward_ON2  # noqa: F401  (backward_sampling_ON2, smoothing.py:291-311)


class CSMC(orc.SMC):
    """Conditional SMC: multinomial resampling, history kept in ``trace``; ``xstar`` None runs unconditionally."""

    def __init__(self, fk, N=100, ESSrmin=0.5, xstar=None, noise=None):
        orc.SMC.__init__(self, fk, N=N, resampling="multinomial", ESSrmin=ESSrmin, noise=noise, keep=True)
        self.xstar = xstar

    def step(self):
        if self.t >= self.fk.T:
            raise StopIteration
        if self.t == 0:                                    # generate_particles, mcmc.py:468-470
            self.X = self.fk.M0(self.N, self.noise.normals(0, None))
            if self.xstar is not None:
                self.X[0] = self.xstar[0]
        else:                                              # resample_move, mcmc.py:472-475
            self.setup_auxiliary_weights()
            self.resample_move()
            if self.xstar is not None:
                self.X[0] = self.xstar[self.t]
                self.A[0] = 0
                self.Xp = np.array(self.Xp, copy=True)
                self.Xp[0] = self.xstar[self.t - 1]        # the correction: the pinned path's own previous state
        self.wgts = self.wgts.add(self.fk.logG(self.t, self.Xp, self.X))
        self.compute_summaries()
        self.t += 1

    @property
    def hist(self):
        """The history in the layout of ``smoothing_numpy``: lists X, lw, A (A[0] = arange)."""
        A = [np.arange(self.N)] + [s["A"] for s in self.trace[1:]]
        return {"X": [s["X"] for s in self.trace], "lw": [s["lw"] for s in self.trace], "A": A}


def extract_one_trajectory(hist, u=None):
    """smoothing.py:256-269: one multinomial_once on W_{T-1}, then the ancestors."""
    X, A = hist["X"], hist["A"]
    T = len(X)
    n = orc.multinomial_once(orc.exp_and_normalise(hist["lw"][-1]), u)
    traj = [None] * T
    for t in reversed(range(T)):
        if t < T - 1:
            n = A[t + 1][n]
        traj[t] = X[t][n]
    return traj


def draw_trajectory(hist, logpt, u, backward):
    """The device kernel's trajectory draw: u (T,) uniforms, u[T-1] for the index at T - 1 (multinomial_once on
    W_{T-1}), u[t] for the backward draw at t from lw_t + logpt(t + 1, X_t, x_{t+1}) (smoothing.py:303-308); without
    ``backward`` the ancestors are traced.  Returns (trajectory (T,), its indices (T,))."""
    X, A, lw = hist["X"], hist["A"], hist["lw"]
    T, N = len(X), X[0].shape[0]
    n = min(orc.multinomial_once(orc.exp_and_normalise(lw[-1]), u[T - 1]), N - 1)
    traj, idx = np.empty(T), np.empty(T, dtype=np.int64)
    traj[-1], idx[-1] = X[-1][n], n
    for t in reversed(range(T - 1)):
        if backward:
            lwm = lw[t] + logpt(t + 1, X[t], traj[t + 1])
            n = min(orc.multinomial_once(orc.exp_and_normalise(lwm), u[t]), N - 1)
        else:
            n = A[t + 1][n]
        traj[t], idx[t] = X[t][n], n
    return traj, idx


class VanishCovTracker:
    """mcmc.py:188-220."""

    def __init__(self, alpha=0.6, dim=1, mu0=None, Sigma0=None):
        self.alpha, self.t = alpha, 0
        self.mu = np.zeros(dim) if mu0 is None else mu0
        if Sigma0 is None:
            self.Sigma, self.L0 = np.eye(dim), np.eye(dim)
        else:
            self.Sigma, self.L0 = Sigma0, cholesky(Sigma0, lower=True)
        self.L = self.L0.copy()

    def update(self, v):
        self.t += 1
        g = (self.t + 1) ** (-self.alpha)
        self.mu = (1.0 - g) * self.mu + g * v
        mv = v - self.mu
        self.Sigma = (1.0 - g) * self.Sigma + g * np.dot(mv[:, np.newaxis], mv[np.newaxis, :])
        try:
            self.L = cholesky(self.Sigma, lower=True)
        except LinAlgError:
            self.L = self.L0


def rwhm(logpost, theta0, z, u, adaptive=True, scale=1.0, rw_cov=None):
    """GenericRWHM.step0 / step (mcmc.py:258-294) for one chain: z (niter, d) proposal normals and u (niter,)
    acceptance uniforms (entry n used at step n).  Returns (theta (niter, d), lpost (niter,), nacc)."""
    niter, d = z.shape
    arr, lp = np.empty((niter, d)), np.empty(niter)
    arr[0], lp[0] = theta0, logpost(theta0)
    if adaptive:
        scale = scale * 2.38 / np.sqrt(d)
        tracker = VanishCovTracker(dim=d, Sigma0=rw_cov)
        L = scale * tracker.L
    else:
        L = np.eye(d) if rw_cov is None else cholesky(rw_cov, lower=True)
    nacc = 0
    for n in range(1, niter):
        prop = arr[n - 1] + np.dot(L, z[n])
        lpp = logpost(prop)
        if np.log(u[n]) < lpp - lp[n - 1]:
            arr[n], lp[n] = prop, lpp
            nacc += 1
        else:
            arr[n], lp[n] = arr[n - 1], lp[n - 1]
        if adaptive:
            tracker.update(arr[n])
            L = scale * tracker.L
    return arr, lp, nacc


def gibbs(theta0, niter, update_theta, update_states):
    """GenericGibbs in the corrected order: x_n is drawn given theta_n (the reference passes theta_{n-1},
    mcmc.py:526-529).  ``update_states(theta, x)``: x is None at n = 0."""
    theta, x = [theta0], [update_states(theta0, None)]
    for n in range(1, niter):
        theta.append(update_theta(theta[-1], x[-1]))
        x.append(update_states(theta[-1], x[-1]))
    return theta, x
