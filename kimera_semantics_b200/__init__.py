"""H100-native semantic TSDF integrator: drop-in for Kimera-Semantics' `fast` / `merged` integrators.

Only the hot path lives here (SURVEY.md §8): `csrc/` holds the sm_90a CUDA kernels and the C-ABI
(`include/ksg.h`), `cpp/` the C++ host shim mirroring the reference classes, `capi.py` a ctypes
binding of the C-ABI used by tests and bench.py, `synth.py` the synthetic depth+label+pose generator.
"""
from .capi import (KsgConfig, KsgFrameStats, default_config, load_library, Integrator, library_path,
                   KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED)

__all__ = ["KsgConfig", "KsgFrameStats", "default_config", "load_library", "Integrator", "library_path",
           "KSG_INTEGRATOR_FAST", "KSG_INTEGRATOR_MERGED"]
