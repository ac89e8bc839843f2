"""Golden fixture for blockwise fp8 expert weights (3-D Float8Tensor with 128x128 blocks per expert, PerBlock([1, 128])
activations) from the REFERENCE on the CPU:

* Float8Tensor.from_hp of bf16 expert weights [E, N, K] with PerBlock([128, 128]) (from_hp, not quantize_, which checks
  for an sm_89 device first): codes ``w_q``, scales ``w_scale`` [E, N/128, K/128] and ``block_size``.  Expert 0 holds a
  block whose scale is a subnormal fp32, expert 1 an all-zero block (scale 0, codes NaN);
* the views the expert paths take: ``select`` (w[e], the eager loop's 2-D weight) and ``transpose(-2, -1)`` (how
  torch._grouped_mm receives the weight), their shapes and block sizes (``views``, JSON);
* the per-expert recipe's activation quantization: each expert's rows [offs[e-1], offs[e]) quantized on their own with
  PerBlock([1, 128]), codes ``x_q`` and scales ``x_scale`` up to offs[-1].  ``offs`` has an empty expert, and the input
  has rows past offs[-1];
* what the reference's own _grouped_mm does with this pair (``grouped_mm``, JSON: the exception type and message).

The reference's blockwise GEMM is a Triton kernel and cannot run on a CPU, so the fixture holds no GEMM outputs.

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_fp8_blockwise_3d.py
-> fp8_blockwise_3d.npz (bf16 inputs as uint16 bits, e4m3 codes as uint8, scales fp32, JSON strings as 0-d arrays)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
E, N, K = 3, 256, 384
OFFS = [5, 5, 12]      # expert 1 is empty
M = 14                 # rows 12 and 13 are past offs[-1]


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    from torchao.quantization import PerBlock
    from torchao.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor, QuantizeTensorToFloat8Kwargs

    torch.manual_seed(2025)
    out = {}
    w = torch.randn(E, N, K) * torch.logspace(-2, 2, N)[None, :, None]
    w[0, :128, 128:256] = torch.randn(128, 128) * 2.0 ** -121   # amax / 448 is a subnormal fp32
    w[1, 128:, :128] = 0                                         # an all-zero block
    w = w.to(torch.bfloat16)
    act = QuantizeTensorToFloat8Kwargs(granularity=PerBlock([1, 128]))
    wt = Float8Tensor.from_hp(w, granularity=PerBlock([128, 128]), act_quant_kwargs=act)
    out["w"], out["w_q"] = bits(w), wt.qdata.view(torch.uint8).numpy().copy()
    out["w_scale"], out["block_size"] = wt.scale.numpy().copy(), np.array(list(wt.block_size), np.int64)

    views = {"select": [], "transpose": {}}
    for e in range(E):
        s = wt[e]
        views["select"].append({"shape": list(s.shape), "qdata": list(s.qdata.shape), "scale": list(s.scale.shape),
                                "block_size": list(s.block_size)})
    t = wt.transpose(-2, -1)
    views["transpose"] = {"shape": list(t.shape), "qdata": list(t.qdata.shape), "scale": list(t.scale.shape),
                          "block_size": list(t.block_size)}
    out["views"] = np.array(json.dumps(views, sort_keys=True))

    x = torch.randn(M, K) * torch.logspace(-2, 2, K)[None, :]
    x[0, :128] = 0                       # an all-zero activation block
    x[6, 128:256] *= 2.0 ** -125         # a subnormal activation scale
    x = x.to(torch.bfloat16)
    out["x"], out["offs"] = bits(x), np.array(OFFS, np.int32)
    q, s, start = [], [], 0
    for end in OFFS:
        if end == start:   # an empty expert: the recipe's loop skips it (from_hp of no rows divides by zero)
            continue
        xt = Float8Tensor.from_hp(x[start:end], granularity=PerBlock([1, 128]))
        q.append(xt.qdata.view(torch.uint8).numpy())
        s.append(xt.scale.numpy())
        start = end
    out["x_q"], out["x_scale"] = np.concatenate(q), np.concatenate(s)

    try:
        torch._grouped_mm(x, t, offs=torch.tensor(OFFS, dtype=torch.int32))
        result = {"raised": None, "message": ""}
    except Exception as exc:   # recorded, whichever it is
        result = {"raised": type(exc).__name__, "message": str(exc)}
    out["grouped_mm"] = np.array(json.dumps(result, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, "fp8_blockwise_3d.npz"), **out)
    print(views)
    print(result)


if __name__ == "__main__":
    main()
