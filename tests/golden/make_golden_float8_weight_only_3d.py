"""Golden fixture for float8 weight-only MoE expert weights (Float8WeightOnlyConfig on 3-D [E, N, K] weights) from the
REFERENCE on the CPU: Float8Tensor.from_hp of a 3-D bf16 weight (PerRow and PerTensor, no activation quantization),
then torch._grouped_mm(x, w.transpose(-2, -1), offs=offs) through the weight-only branch of the reference's
_grouped_mm handler (torch._grouped_mm on the dequantized weight), and, per expert, F.linear(x[rows_e], w[e]) through
its select.  The cases cover:

* an empty expert and rows after offs[-1] (not stored: torch leaves them unwritten);
* N not a multiple of 128 (an N tail) and K not a multiple of 128 (a K tail);
* an all-zero weight row (expert 0, row 1): its scale is 0 and its codes NaN (0 / 0), which the output carries, next
  to stored rows of the same 128-row tile;
* per-expert weight magnitudes that span decades (expert e times 10^(2e - 3)), and rows over two decades.

Two inputs per shape: ``x`` random bf16 and ``xe`` one-hot rows (+-2^j at one column per row: every output is one
product w~[e, n, k] * 2^j, exact in fp32, so it is determined bit for bit).  The reference's select fails for a
per-tensor scale [1, 1, 1] past expert 0 (scale[index]), so F.linear outputs are recorded for PerRow only.

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_float8_weight_only_3d.py
-> float8_weight_only_3d.npz (bf16 arrays as uint16 bits, e4m3 codes as uint8): s<shape>_<field> (weight, inputs,
offs; qdata, scale and outputs per granularity) and ``cases``, a JSON list describing each shape."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
# (E, K, N, rows of each expert, rows after offs[-1])
SHAPES = [(4, 160, 200, [5, 0, 9, 3], 4), (3, 256, 128, [17, 0, 33], 0), (2, 48, 40, [1, 6], 2)]
ZERO_ROW = 1


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    import torch.nn.functional as F
    from torchao.quantization import PerRow, PerTensor
    from torchao.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor

    out, cases = {}, []
    for si, (E, K, N, rows, tail) in enumerate(SHAPES):
        torch.manual_seed(300 + si)
        w = torch.randn(E, N, K) * torch.logspace(-1, 1, N)[None, :, None]
        w = w * torch.pow(10.0, 2.0 * torch.arange(E) - 3)[:, None, None]   # experts over decades
        w[0, ZERO_ROW] = 0
        w = w.to(torch.bfloat16)
        M = sum(rows) + tail
        offs = torch.tensor(np.cumsum(rows), dtype=torch.int32)
        x = (torch.randn(M, K) * 1.5).to(torch.bfloat16)
        xe = torch.zeros(M, K)
        cols = torch.randint(0, K, (M,))
        xe[torch.arange(M), cols] = torch.pow(2.0, torch.randint(-3, 4, (M,)).float()) * (torch.randint(0, 2, (M,)) * 2 - 1)
        xe = xe.to(torch.bfloat16)
        out[f"s{si}_w"], out[f"s{si}_x"], out[f"s{si}_xe"] = bits(w), bits(x), bits(xe)
        out[f"s{si}_offs"] = offs.numpy().copy()
        end = int(offs[-1])
        for gname, gran in (("PerRow", PerRow()), ("PerTensor", PerTensor())):
            wq = Float8Tensor.from_hp(w, float8_dtype=torch.float8_e4m3fn, granularity=gran)
            assert wq.act_quant_kwargs is None and wq.scale.dtype == torch.float32 and wq.dtype == torch.bfloat16
            out[f"s{si}_{gname}_q"] = wq.qdata.view(torch.uint8).numpy().copy()
            out[f"s{si}_{gname}_scale"] = wq.scale.numpy().copy()
            out[f"s{si}_{gname}_block_size"] = np.array(wq.block_size)
            with torch.no_grad():
                for name, inp in (("y", x), ("ye", xe)):
                    y = torch._grouped_mm(inp, wq.transpose(-2, -1), offs=offs)
                    out[f"s{si}_{gname}_{name}"] = bits(y[:end])
                    if gname == "PerRow":
                        lin, start = [], 0
                        for e in range(E):
                            lin.append(F.linear(inp[start:int(offs[e])], wq[e]))
                            start = int(offs[e])
                        out[f"s{si}_{gname}_{name}_linear"] = bits(torch.cat(lin))
        cases.append(dict(shape=si, E=E, K=K, N=N, rows=rows, tail=tail, M=M))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "float8_weight_only_3d.npz"), **out)
    print("wrote", len(cases), "shapes")


if __name__ == "__main__":
    main()
