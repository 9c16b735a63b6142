"""advancedhmc.jl_b200 -- H100-native (sm_90a) many-chain leapfrog / HMC / NUTS engine behind
AdvancedHMC.jl's `AbstractIntegrator` / `Hamiltonian` / `AbstractMetric` plugin surface.

The directory name is not a legal Python identifier; import it as `ahmc_b200` (root-level shim).
Product path = libahmc_b200.so (CUDA kernels + C ABI) + this thin host mirror.  No CPU fallback.
"""
from . import _lib
from ._lib import (FLAG_ASYNC, FLAG_COMPAT_BREAK_ALL, FLAG_EXACT_CHECKS, FLAG_HOST_BUFFERS, FLAG_NO_REFRESH,
                   FLAG_NUTS_CLASSIC, FLAG_NUTS_SLICE_TS, FLAG_NUTS_STRICT,
                   STATUS_NONFINITE, AhmcError, InvalidArgument)
from .core import *  # noqa: F401,F403
from .core import get_context
