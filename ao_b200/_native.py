"""Loads the in-tree native libraries and fails loudly when they are missing.

``ao_b200/lib/libao_b200.so``  — C-ABI CUDA kernels (nvcc, sm_90a)
``ao_b200/lib/ao_b200_torch.so`` — TORCH_LIBRARY(ao_b200) registration (links the above)
Built by ``python -m ao_b200._build`` / ``__graft_entry__.build()``; never JIT-compiled.
"""
from __future__ import annotations

import os
from pathlib import Path

import torch

_LIB_DIR = Path(__file__).resolve().parent / "lib"
_LOADED = False


def native_lib_paths():
    return _LIB_DIR / "libao_b200.so", _LIB_DIR / "ao_b200_torch.so"


def load_native() -> None:
    global _LOADED
    if _LOADED:
        return
    cu, binding = native_lib_paths()
    missing = [str(p) for p in (cu, binding) if not p.exists()]
    if missing:
        raise ImportError(
            "ao_b200: native library not built: " + ", ".join(missing)
            + ". Run `python -m ao_b200._build` (or __graft_entry__.build()). "
            "There is no fallback path for the quantized-linear kernels."
        )
    torch.ops.load_library(str(binding))
    if not hasattr(torch.ops.ao_b200, "int4_tilepacked_linear"):
        raise ImportError("ao_b200: torch.ops.ao_b200 did not register; stale build?")
    _LOADED = True


def require_sm90(device=None) -> None:
    """Raise unless the CUDA device can run the sm_90a kernels."""
    if not torch.cuda.is_available():
        raise RuntimeError("ao_b200: a CUDA device (H100, sm_90) is required; none is visible")
    major, minor = torch.cuda.get_device_capability(device)
    if (major, minor) != (9, 0):
        raise RuntimeError(f"ao_b200: kernels are built for sm_90a only, device is sm_{major}{minor}")
