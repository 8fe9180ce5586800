"""Randomised quasi-Monte Carlo points on the device (particles/rqmc.py).

``sobol(N, d)`` restates ``rqmc.sobol``: scrambled Sobol' points of ``scipy.stats.qmc.Sobol(d)`` (30 bits, a linear
matrix scramble and a digital shift), squeezed into ``0.5 + (1 - 1e-10) * (u - 0.5)``, for d <= ``MAX_DIM`` = 4096, as
an (N, d) CUDA tensor (csrc/smcb_sqmc.cu).  Dimension j's scrambling depends on (key, j) only, so the first k columns of
a d-dimensional set equal the k-dimensional set of the same key.  The scrambling is drawn from the device Philox under
a key taken from NumPy's global generator, so ``np.random.seed`` repeats it.  Halton and Latin hypercube points have no
kernel.
"""
import numpy as np
import torch

from . import _lib
from .device import context, ptr

TOL = 1e-10
MAX_DIM = 4096


def sobol_points(N, d, seed, call=0, scramble=True, raw=False):
    """The (d, N) component-major points of ``smcb_sobol`` for key (seed, call); with ``raw``, also the (d, N) 30-bit
    integers.  Step t of ``SMC(qmc=True, seed=s)`` uses key (s, t), with d = du at t = 0 and du + 1 afterwards."""
    N, d = int(N), int(d)
    if not 1 <= d <= MAX_DIM:
        raise NotImplementedError(f"device Sobol' points exist for d = 1..{MAX_DIM} (got d={d})")
    ctx = context()
    ctx.bind_stream()
    u = torch.empty((d, N), dtype=torch.float64, device=ctx.device)
    r = torch.empty((d, N), dtype=torch.int32, device=ctx.device) if raw else None
    _lib.check(ctx.lib.smcb_sobol(ctx.handle, d, N, 1 if scramble else 0, int(seed) & (2 ** 64 - 1),
                                  int(call) & (2 ** 64 - 1), ptr(u), None if r is None else ptr(r)))
    return (u, r) if raw else u


def sobol(N, d):
    """rqmc.sobol(N, d): (N, d) scrambled Sobol' points in (0, 1), a CUDA tensor."""
    seed = int(np.random.randint(0, 2 ** 62, dtype=np.int64))
    return sobol_points(N, d, seed).t()


def halton(N, d):
    raise NotImplementedError("Halton points have no device kernel; use rqmc.sobol")


def latin(N, d):
    raise NotImplementedError("Latin hypercube points have no device kernel; use rqmc.sobol")
