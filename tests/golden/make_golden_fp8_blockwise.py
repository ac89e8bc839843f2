"""Golden fixture for blockwise fp8 (Float8DynamicActivationFloat8WeightConfig with granularity
[PerBlock([1, 128]), PerBlock([128, 128])]) from the REFERENCE on the CPU:

* its Float8Tensor.from_hp codes and scales for 128x128 weight blocks (``w_*``) and 1x128 activation blocks (``x_*``,
  a 2-D and a 3-D input).  The inputs hold an all-zero block (scale 0, codes NaN: 0/0), blocks whose scale is a
  subnormal fp32 (amax of 2^-126 and below), blocks of bf16 extremes (the largest finite bf16, the smallest subnormal)
  and ordinary random blocks over several decades;
* config_to_dict of the blockwise config (``config_json``), which carries its mm_config default, and which spellings
  of the granularity the reference's config accepts (``spellings``: the pair as a list or a tuple, the block sizes as
  lists or tuples).

The reference's GEMM is a Triton kernel and cannot run on a CPU, so the fixture holds no GEMM outputs; the tests
restate its loop in torch.

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_fp8_blockwise.py
-> fp8_blockwise.npz (bf16 inputs as uint16 bits, e4m3 codes as uint8, scales fp32; JSON strings as 0-d arrays)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
W_SHAPE = (256, 256)      # (N, K): 2 x 2 weight blocks
X_SHAPE = (6, 512)        # (M, K): 4 blocks per token
X3_SHAPE = (2, 3, 256)    # a 3-D input: the block size applies to the last dim


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def edge_blocks(x, width):
    """Rows of x rewritten block by block: block 0 of row 0 all zero, block 1 of row 0 with a subnormal scale, block 0
    of row 1 holding the largest finite bf16 and the smallest subnormal, block 1 of row 1 tiny normals."""
    x[0, :width] = 0
    x[0, width: 2 * width] = torch.randn(width) * 2.0 ** -128
    x[1, :width] = torch.randn(width)
    x[1, 0], x[1, 1], x[1, 2] = torch.finfo(torch.bfloat16).max, -torch.finfo(torch.bfloat16).max, 2.0 ** -133
    x[1, width: 2 * width] = torch.randn(width) * 2.0 ** -120
    return x


def main():
    from torchao.core.config import config_to_dict
    from torchao.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock
    from torchao.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor

    torch.manual_seed(2024)
    out = {}
    w = torch.randn(W_SHAPE) * torch.logspace(-3, 3, W_SHAPE[0])[:, None]
    w = edge_blocks(w, 128)
    w[128:, 128:] = 0   # a whole weight block of zeros
    w = w.to(torch.bfloat16)
    wt = Float8Tensor.from_hp(w, granularity=PerBlock([128, 128]))
    assert list(wt.block_size) == [128, 128] and wt.scale.shape == (W_SHAPE[0] // 128, W_SHAPE[1] // 128)
    out["w"], out["w_q"], out["w_scale"] = bits(w), wt.qdata.view(torch.uint8).numpy().copy(), wt.scale.numpy().copy()

    x = torch.randn(X_SHAPE) * torch.logspace(-2, 2, X_SHAPE[1])[None, :]
    x = edge_blocks(x, 128).to(torch.bfloat16)
    xt = Float8Tensor.from_hp(x, granularity=PerBlock([1, 128]))
    assert list(xt.block_size) == [1, 128] and xt.scale.shape == (X_SHAPE[0], X_SHAPE[1] // 128)
    out["x"], out["x_q"], out["x_scale"] = bits(x), xt.qdata.view(torch.uint8).numpy().copy(), xt.scale.numpy().copy()

    x3 = (torch.randn(X3_SHAPE) * 3).to(torch.bfloat16)
    x3t = Float8Tensor.from_hp(x3, granularity=PerBlock([1, 128]))
    assert list(x3t.block_size) == [1, 1, 128]
    out["x3"], out["x3_q"], out["x3_scale"] = bits(x3), x3t.qdata.view(torch.uint8).numpy().copy(), x3t.scale.numpy().copy()

    cfg = Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])])
    out["config_json"] = np.array(json.dumps(config_to_dict(cfg), sort_keys=True))
    spellings = {}
    for name, g in (("list_of_lists", [PerBlock([1, 128]), PerBlock([128, 128])]),
                    ("tuple_of_lists", (PerBlock([1, 128]), PerBlock([128, 128]))),
                    ("list_of_tuples", [PerBlock((1, 128)), PerBlock((128, 128))]),
                    ("tuple_of_tuples", (PerBlock((1, 128)), PerBlock((128, 128))))):
        try:
            Float8DynamicActivationFloat8WeightConfig(granularity=g)
            spellings[name] = "ok"
        except ValueError:
            spellings[name] = "ValueError"
    out["spellings"] = np.array(json.dumps(spellings, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, "fp8_blockwise.npz"), **out)
    print(spellings)
    print(json.dumps(config_to_dict(cfg))[:400])


if __name__ == "__main__":
    main()
