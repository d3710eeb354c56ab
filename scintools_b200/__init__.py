"""scintools_b200 -- CUDA-native (H100, sm_90a) implementation of the scintools
arc-measurement hot path: Dynspec.calc_sspec / calc_acf, the ththmod
theta-theta curvature sweep and scint_sim.Simulation, behind the reference's
Python API.  Hand-written CUDA in libscint_b200.so, called through ctypes.
No CPU fallback: importing needs the built library, running needs an H100.
"""
from . import _lib  # noqa: F401  (fails loudly when the .so is missing)
from . import scint_utils  # noqa: F401
from . import ththmod  # noqa: F401
from .dynspec import BasicDyn, Dynspec  # noqa: F401

__all__ = ["ththmod", "scint_utils", "Dynspec", "BasicDyn"]
__version__ = "0.1.0"
