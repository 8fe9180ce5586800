"""particles_b200 -- the per-step SMC hot path of nchopin/particles on an H100.

Hand-written sm_90a CUDA kernels (csrc/, C-ABI in include/smcb.h) behind the
reference's own plugin surface: ``SMC``, ``FeynmanKac``, ``state_space_models``,
``distributions``, ``resampling``, ``collectors``.  See DESIGN.md / INTEGRATION.md.
"""
from .core import SMC, FeynmanKac, multiSMC  # noqa: F401
from .device import seed  # noqa: F401
from . import hmm  # noqa: F401
from .hmm import HMM, GaussianHMM, BaumWelch  # noqa: F401
from . import kalman  # noqa: F401

__version__ = "0.1.0"


def install():
    """Make this package the engine under the reference's own entry point: after ``particles_b200.install()``
    ``particles.SMC(fk=..., N=...).run()`` (and ``particles.core.SMC``) IS ``particles_b200.SMC``.  The
    reference's model / Feynman-Kac classes stay the user-facing surface: stock models built from
    ``particles.state_space_models`` / ``particles.kalman`` are recognised by class and module name
    (``state_space_models.fused_spec``) and run on the fused kernels; their NumPy closures are never called.
    The reference's ``particles.smc_samplers.SMC2`` of a stock 1-D model runs as ``smc_samplers.SMC2`` (its inner
    filters in one device filter bank).
    Returns a function that restores the original binding."""
    import importlib
    import sys
    core_mod = importlib.import_module("particles.core")
    pkg = sys.modules["particles"]
    saved = (getattr(pkg, "SMC", None), core_mod.SMC)
    pkg.SMC = SMC
    core_mod.SMC = SMC

    def uninstall():
        pkg.SMC, core_mod.SMC = saved

    return uninstall
