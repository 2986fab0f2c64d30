"""clp_b200 -- H100-native revised dual simplex behind Clp's ClpSimplex::dual() surface.

Only what the hot path needs lives here: ``csrc/`` (sm_90a CUDA kernels + the C ABI of
include/clp_b200.h), ``simplex.ClpSimplex`` (host-side mirror of the reference interface) and
``generators`` (synthetic LPs of BASELINE.json and of the reference's own tests).
"""
from .simplex import ClpSimplex, NoDeviceError, denseInvert  # noqa: F401
