"""Golden fixture for [B, K, N] expert weights of torch.bmm (Llama-4 layout) from the REFERENCE on the CPU.

Float8Tensor.from_hp(w, e4m3, PerRow(1)) of bf16 weights stored [B, K, N]: one scale per (batch, output feature n),
taken over K, shape [B, 1, N].  Shapes include K and N that are not multiples of 128 and B = 1; the values mix
magnitudes across features, an all-zero feature and features whose amax sits on e4m3 ties.

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_fp8_bmm.py
-> fp8_bmm.npz: s<i>_w (bf16 bits as uint16, [B, K, N]), s<i>_wq (e4m3 codes as uint8, [B, K, N]), s<i>_ws (f32
[B, 1, N]) and s<i>_bs (the block_size), and ``shapes``, the JSON list of (B, K, N)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(3, 208, 144), (1, 128, 256), (2, 384, 48)]   # (B, K, N)


def main():
    from torchao.quantization.granularity import PerRow
    from torchao.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor

    g = torch.Generator().manual_seed(20261018)
    out = {"shapes": json.dumps(SHAPES)}
    for i, (B, K, N) in enumerate(SHAPES):
        col = torch.exp2(torch.randint(-12, 6, (B, 1, N), generator=g).float())
        w = torch.randn(B, K, N, generator=g) * col
        w[:, :, 1] = 0.0                                        # an all-zero feature: scale 0 -> clamped
        w[:, 3, 2] = 448.0 * 2.0 ** -5 * 1.0625                  # amax on a tie of amax / 448
        w = w.to(torch.bfloat16)
        t = Float8Tensor.from_hp(w, float8_dtype=torch.float8_e4m3fn, granularity=PerRow(1))
        assert tuple(t.scale.shape) == (B, 1, N), t.scale.shape
        out[f"s{i}_w"] = w.view(torch.int16).numpy().view(np.uint16)
        out[f"s{i}_wq"] = t.qdata.view(torch.uint8).numpy()
        out[f"s{i}_ws"] = t.scale.float().numpy()
        out[f"s{i}_bs"] = np.array(t.block_size, dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "fp8_bmm.npz"), **out)
    print("wrote", os.path.join(HERE, "fp8_bmm.npz"))


if __name__ == "__main__":
    main()
