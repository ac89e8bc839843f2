"""Golden fixture for int8 weight-only (Int8WeightOnlyConfig, version 2) from the REFERENCE on the CPU: for a few small
linears, quantize_(nn.Linear(K, N).bfloat16(), Int8WeightOnlyConfig(granularity)) and F.linear through the weight-only
branch of the reference's Int8Tensor handler.  Shapes include K not a multiple of 128 and N not a multiple of 128;
PerRow and PerTensor; with and without bias.  Two inputs per linear:

* ``x``: random bf16 (fp32 sums round, so the accumulation order can show in the last bf16 bit);
* ``xe``: integers -8..8 times 2^-3 (every product x * q is a multiple of 2^-3 and the sums stay below 2^24 of them:
  fp32 accumulates exactly in any order, the output is determined bit for bit).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_int8_weight_only.py
-> int8_weight_only.npz (bf16 arrays as uint16 bits): s<shape>_<field> (weight, bias, inputs; qdata and scale per
granularity), c<case>_y / c<case>_ye (outputs) and ``cases``, a JSON list describing each case."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(5, 160, 72), (33, 256, 128), (3, 400, 40)]   # (M, K, N)


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    import torch.nn.functional as F
    from torchao.quantization import Int8WeightOnlyConfig, PerRow, PerTensor, quantize_
    from torchao.quantization.quantize_.workflows.int8.int8_tensor import Int8Tensor

    out, cases = {}, []
    for si, (M, K, N) in enumerate(SHAPES):
        torch.manual_seed(100 + si)
        base = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
        with torch.no_grad():
            base.weight.mul_(torch.logspace(-2, 2, N)[:, None].to(torch.bfloat16))   # scales over four decades
        x = (torch.randn(M, K) * 1.5).to(torch.bfloat16)
        xe = (torch.randint(-8, 9, (M, K)).float() * 2.0**-3).to(torch.bfloat16)
        out[f"s{si}_w"], out[f"s{si}_b"], out[f"s{si}_x"], out[f"s{si}_xe"] = bits(base.weight), bits(base.bias), bits(x), bits(xe)
        for gname, gran in (("PerRow", PerRow()), ("PerTensor", PerTensor())):
            lin = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
            lin.load_state_dict(base.state_dict())
            quantize_(lin, Int8WeightOnlyConfig(granularity=gran, set_inductor_config=False))
            w = lin.weight
            assert isinstance(w, Int8Tensor) and w.act_quant_kwargs is None and w.scale.dtype == torch.float32
            out[f"s{si}_{gname}_q"] = w.qdata.numpy().copy()
            out[f"s{si}_{gname}_scale"] = w.scale.numpy().copy()
            for bias in (True, False):
                b = lin.bias if bias else None
                with torch.no_grad():
                    out[f"c{len(cases)}_y"] = bits(F.linear(x, w, b))
                    out[f"c{len(cases)}_ye"] = bits(F.linear(xe, w, b))
                cases.append(dict(shape=si, M=M, K=K, N=N, granularity=gname, bias=bias, block_size=list(w.block_size)))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "int8_weight_only.npz"), **out)
    print("wrote", len(cases), "cases")


if __name__ == "__main__":
    main()
