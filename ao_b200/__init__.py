"""ao_b200 — H100-native quantized-linear engine with torchao's operator surface.

Drop-in for the quantized ``nn.Linear`` forward of pytorch/ao (torchao 0.19): the same
``quantize_`` / config / tensor-subclass API, with the kernels underneath replaced by
hand-written sm_90a CUDA (``libao_b200.so``, C ABI in ``include/ao_b200.h``) registered as
``torch.ops.ao_b200.*``.  There is no CPU or eager fallback for the hot path: importing this
package without the native library raises.
"""
import os as _os
import sys as _sys

from ._native import load_native, native_lib_paths  # noqa: F401

__version__ = "0.2.0"

# `python -m ao_b200._build` imports this package before the module it runs: a fresh checkout has no native
# libraries yet (they are git-ignored build products), so the build entry point alone may import the package
# without them.  Every other import fails loudly when they are missing.
_BUILDING = "ao_b200._build" in getattr(_sys, "orig_argv", []) or _os.environ.get("AO_B200_BUILDING") == "1"

if not _BUILDING:
    load_native()
    from . import quantization  # noqa: E402,F401
    from .quantization import quantize_  # noqa: E402,F401
