"""cleandiffuser_b200 -- H100-native diffusion-policy sampling engine.

Keeps CleanDiffuser's ``diffusion`` / ``nn_diffusion`` / ``nn_condition`` plugin surfaces and
runs ``sample()``'s reverse loop as hand-written sm_90a CUDA behind a C-ABI (``include/cds.h``).
"""
__version__ = "0.1.0"

from . import utils, nn_condition, nn_diffusion, diffusion  # noqa: F401
from .overlay import install, uninstall  # noqa: F401  (drop-in route A: rebind the installed reference's sampler classes)
