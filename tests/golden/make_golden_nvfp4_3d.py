"""Golden fixture for the 3-D (MoE expert) NVFP4 weight: the REFERENCE's CPU NVFP4Tensor.to_nvfp4 on a bf16 [E, N, K]
weight with a per-expert per_tensor_scale [E, 1, 1] (nvfp4_tensor.py:131-194, inference_workflow.py:307-319), with
blocked (swizzled) and plain scales.   PYTHONPATH=/root/reference python tests/golden/make_golden_nvfp4_3d.py
-> nvfp4_3d.npz (x: bf16 bits [E, N, K]; pts: f32 [E]; q_*: qdata bytes; s_*: scale bytes)."""
import os
import sys

import numpy as np
import torch

REF = os.environ.get("AO_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    torch.manual_seed(4321)
    from torchao.prototype.mx_formats.nvfp4_tensor import NVFP4Tensor, per_tensor_amax_to_scale

    E, N, K = 3, 128, 128
    w = torch.randn(E, N, K, dtype=torch.bfloat16)
    w[0] *= 10.0       # as the reference's test_grouped_mm_nvfp4: very different per-expert scales
    w[-1] *= 1e-3
    w[1, 5, :16] = 0.0   # an all-zero block
    pts = per_tensor_amax_to_scale(torch.amax(torch.abs(w), dim=(1, 2))).view(E, 1, 1)
    out = {"x": w.view(torch.int16).numpy().view(np.uint16).copy(), "pts": pts.reshape(-1).numpy().copy()}
    for name, swz in (("blocked", True), ("plain", False)):
        t = NVFP4Tensor.to_nvfp4(w, per_tensor_scale=pts, is_swizzled_scales=swz, use_triton_kernel=False)
        out[f"q_{name}"] = t.qdata.contiguous().view(torch.uint8).numpy().copy()
        out[f"s_{name}"] = t.scale.contiguous().view(torch.uint8).numpy().copy()
        print(name, tuple(t.qdata.shape), tuple(t.scale.shape))
    np.savez_compressed(os.path.join(HERE, "nvfp4_3d.npz"), **out)


if __name__ == "__main__":
    main()
