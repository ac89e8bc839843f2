"""Golden fixture for the 3-D (MoE expert) MX weight: the REFERENCE's CPU MXTensor.to_mx (block 32, RCEIL) on bf16
[E, N, K] weights, mxfp8 and mxfp4, with blocked (swizzled) and plain scales.  The blocked scales of a 3-D tensor are
to_blocked of its [E*N, K/32] scales viewed as [E, 32 * ceil(N/128), 16 * ceil(K/128)] (mx_tensor.py:401-407), which
exists for N % 128 == 0.  Expert 0 is scaled by 10 and the last by 1e-3, and expert 1 holds an all-zero block.
    PYTHONPATH=/root/reference python tests/golden/make_golden_mx_3d.py
-> mx_3d.npz (x_<shape>: bf16 bits [E, N, K]; q_<fmt>_<shape>: qdata bytes, the same for both layouts;
s_<fmt>_<shape>_<layout>: scale bytes; <shape> = ExNxK, <layout> = blocked | plain)."""
import os
import sys

import numpy as np
import torch

REF = os.environ.get("AO_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(3, 256, 256), (3, 128, 96)]
FMTS = {"mxfp8": torch.float8_e4m3fn, "mxfp4": torch.float4_e2m1fn_x2}


def main():
    from torchao.prototype.mx_formats.config import ScaleCalculationMode
    from torchao.prototype.mx_formats.mx_tensor import MXTensor

    torch.manual_seed(2468)
    out = {}
    for E, N, K in SHAPES:
        tag = f"{E}x{N}x{K}"
        w = torch.randn(E, N, K, dtype=torch.bfloat16)
        w[0] *= 10.0
        w[-1] *= 1e-3
        w[1, 5, 32:64] = 0.0   # an all-zero block
        out[f"x_{tag}"] = w.view(torch.int16).numpy().view(np.uint16).copy()
        for fmt, dt in FMTS.items():
            for layout, swz in (("blocked", True), ("plain", False)):
                t = MXTensor.to_mx(w, dt, 32, ScaleCalculationMode.RCEIL, is_swizzled_scales=swz)
                q = t.qdata.contiguous().view(torch.uint8).numpy().copy()
                assert np.array_equal(out.setdefault(f"q_{fmt}_{tag}", q), q)
                out[f"s_{fmt}_{tag}_{layout}"] = t.scale.contiguous().view(torch.uint8).numpy().copy()
                print(fmt, tag, layout, tuple(t.qdata.shape), tuple(t.scale.shape))
    np.savez_compressed(os.path.join(HERE, "mx_3d.npz"), **out)


if __name__ == "__main__":
    main()
