"""claymore_b200 -- H100-native (sm_90a) MPM transfer engine behind claymore's GMPM/MGSP interface.

The product is the compiled library ``claymore_b200/lib/libclaymore_b200.so`` (hand-written CUDA kernels and a
C++ step driver, C ABI in ``include/claymore_b200.h``).  This package is the thin Python host layer over it:
ctypes bindings, the GmpmSimulator-shaped wrapper, the scene/material front-end and the synthetic samplers.
It fails loudly when the CUDA library is missing: there is no CPU fallback.
"""
from ._capi import (CB200Error, Config, ParticleBuffer, Partition, SimDesc, SimStats, J_FLUID, FIXED_COROTATED, SAND, NACC, lib, lib_path, build_library)
from .simulator import GmpmSimulator
from . import levelset, samplers, scene, scenes

__all__ = ["CB200Error", "Config", "ParticleBuffer", "Partition", "SimDesc", "SimStats", "J_FLUID", "FIXED_COROTATED", "SAND", "NACC", "lib", "lib_path", "build_library", "GmpmSimulator", "levelset", "samplers", "scene", "scenes"]
