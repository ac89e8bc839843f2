"""Kernel family switch carried by the quantized tensors
(reference: torchao/quantization/quantize_/common/kernel_preference.py).

On this engine AUTO resolves to the hand-written sm_90a kernels (``B200``).  ``TORCH`` keeps the
reference's library route (``torch._scaled_mm`` / ``torch._int_mm``) and ``EMULATED`` the
dequantize-then-matmul route; both exist for parity runs only and are never chosen implicitly.
"""
from enum import Enum


class KernelPreference(str, Enum):
    AUTO = "auto"
    TORCH = "torch"
    MSLK = "mslk"          # accepted for config compatibility; not available here
    EMULATED = "emulated"
    B200 = "b200"
