"""Golden fixture for float8 weight-only (Float8WeightOnlyConfig, version 2) from the REFERENCE on the CPU: for a few
small linears, quantize_(nn.Linear(K, N).bfloat16(), Float8WeightOnlyConfig(granularity=g)) and F.linear through the
weight-only branch of the reference's Float8Tensor handler (torch.matmul on the dequantized weight, then + bias).
Shapes include K not a multiple of 128 and N not a multiple of 128; PerRow and PerTensor; with and without bias.  The
weight rows span four decades and row 1 is all zero: its per-row scale is 0 and its codes NaN (0 / 0), which the
reference's output carries.  Two inputs per linear:

* ``x``: random bf16 (fp32 sums round, so the accumulation order can show in the last bf16 bit);
* ``xe``: one-hot rows, +-2^j at one column per row: every output is one product w~[n, k] * 2^j, exact in fp32, so it
  is determined bit for bit: bf16(bf16(w~ * 2^j) + bias).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_float8_weight_only.py
-> float8_weight_only.npz (bf16 arrays as uint16 bits, e4m3 codes as uint8): s<shape>_<field> (weight, bias, inputs;
qdata and scale per granularity), c<case>_y / c<case>_ye (outputs) and ``cases``, a JSON list describing each case."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(5, 160, 72), (33, 256, 128), (3, 400, 40)]   # (M, K, N)
ZERO_ROW = 1


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    import torch.nn.functional as F
    from torchao.quantization import Float8WeightOnlyConfig, PerRow, PerTensor, quantize_
    from torchao.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor

    out, cases = {}, []
    for si, (M, K, N) in enumerate(SHAPES):
        torch.manual_seed(200 + si)
        base = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
        with torch.no_grad():
            base.weight.mul_(torch.logspace(-2, 2, N)[:, None].to(torch.bfloat16))   # rows over four decades
            base.weight[ZERO_ROW] = 0
        x = (torch.randn(M, K) * 1.5).to(torch.bfloat16)
        xe = torch.zeros(M, K)
        cols = torch.randint(0, K, (M,))
        xe[torch.arange(M), cols] = torch.pow(2.0, torch.randint(-3, 4, (M,)).float()) * (torch.randint(0, 2, (M,)) * 2 - 1)
        xe = xe.to(torch.bfloat16)
        out[f"s{si}_w"], out[f"s{si}_b"], out[f"s{si}_x"], out[f"s{si}_xe"] = bits(base.weight), bits(base.bias), bits(x), bits(xe)
        for gname, gran in (("PerRow", PerRow()), ("PerTensor", PerTensor())):
            lin = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
            lin.load_state_dict(base.state_dict())
            quantize_(lin, Float8WeightOnlyConfig(granularity=gran, set_inductor_config=False))
            w = lin.weight
            assert isinstance(w, Float8Tensor) and w.act_quant_kwargs is None and w.scale.dtype == torch.float32
            out[f"s{si}_{gname}_q"] = w.qdata.view(torch.uint8).numpy().copy()
            out[f"s{si}_{gname}_scale"] = w.scale.numpy().copy()
            for bias in (True, False):
                b = lin.bias if bias else None
                with torch.no_grad():
                    out[f"c{len(cases)}_y"] = bits(F.linear(x, w, b))
                    out[f"c{len(cases)}_ye"] = bits(F.linear(xe, w, b))
                cases.append(dict(shape=si, M=M, K=K, N=N, granularity=gname, bias=bias, block_size=list(w.block_size)))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "float8_weight_only.npz"), **out)
    print("wrote", len(cases), "cases")


if __name__ == "__main__":
    main()
