"""Golden fixture for int8 MoE expert weights (the three int8 configs on 3-D [E, N, K] weights) from the REFERENCE on
the CPU: Int8Tensor.from_hp of a 3-D bf16 weight, then, per expert, F.linear(x[rows_e], w[e]) through its select, the
per-expert recipe torch._grouped_mm on an int8 expert weight must reproduce (the reference's Int8Tensor has no
transpose and no _grouped_mm handler).  Variants:

* ``wo_PerRow`` and ``wo_PerTensor``: weight-only (Int8WeightOnlyConfig), per-row and per-tensor weight scales;
* ``dyn_PerRow``: per-row weights with dynamic symmetric PerRow int8 activations
  (Int8DynamicActivationInt8WeightConfig);
* ``static_PerTensor``: per-row weights with a calibrated PerTensor [1, 1] activation scale and a bf16
  ``act_pre_scale`` (Int8StaticActivationInt8WeightConfig with SmoothQuant-style pre-scales).

The reference's select takes ``scale[index]``, which fails past expert 0 for a per-tensor scale [1, 1, 1], so
outputs are recorded for the per-row weights only.  The cases cover:

* an empty expert and rows after offs[-1] (not stored: torch leaves them unwritten);
* N not a multiple of 128 (an N tail) and K not a multiple of 128 (a K tail, K % 16 == 0);
* an all-zero weight row (expert 0, row 1): scale 0, codes 0, outputs 0;
* per-expert weight magnitudes that span decades (expert e times 10^(2e - 3)), and rows over two decades.

Two inputs per shape: ``x`` random bf16 and ``xe`` one-hot rows (+-2^j at one column per row: every weight-only output
is one product q * 2^j, exact in fp32, so it is determined bit for bit).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_int8_3d.py
-> int8_3d.npz (bf16 arrays as uint16 bits, codes as int8): s<shape>_<field> (weight, inputs, offs, the static
activation scale and pre-scale; qdata, scale and block_size per weight granularity, PerRow or PerTensor, stored once
because the three per-row variants quantize the weight identically; outputs per variant) and ``cases``, a JSON list
describing each shape."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
# (E, K, N, rows of each expert, rows after offs[-1])
SHAPES = [(4, 160, 136, [5, 0, 9, 3], 4), (3, 128, 128, [17, 0, 33], 0), (2, 48, 40, [1, 6], 2)]
ZERO_ROW = 1
VARIANTS = ("wo_PerRow", "wo_PerTensor", "dyn_PerRow", "static_PerTensor")


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    import torch.nn.functional as F
    from torchao.quantization import PerRow, PerTensor
    from torchao.quantization.quantize_.workflows.int8.int8_tensor import Int8Tensor, QuantizeTensorToInt8Kwargs

    out, cases = {}, []
    for si, (E, K, N, rows, tail) in enumerate(SHAPES):
        torch.manual_seed(400 + si)
        w = torch.randn(E, N, K) * torch.logspace(-1, 1, N)[None, :, None]
        w = w * torch.pow(10.0, 2.0 * torch.arange(E) - 3)[:, None, None]   # experts over decades
        w[0, ZERO_ROW] = 0
        w = w.to(torch.bfloat16)
        M = sum(rows) + tail
        offs = torch.tensor(np.cumsum(rows), dtype=torch.int32)
        x = (torch.randn(M, K) * torch.logspace(-1, 1, M)[:, None]).to(torch.bfloat16)   # rows over two decades
        xe = torch.zeros(M, K)
        cols = torch.randint(0, K, (M,))
        xe[torch.arange(M), cols] = torch.pow(2.0, torch.randint(-3, 4, (M,)).float()) * (torch.randint(0, 2, (M,)) * 2 - 1)
        xe = xe.to(torch.bfloat16)
        pre = (torch.rand(K) + 0.5).to(torch.bfloat16)
        act_scale = ((x.float() * pre.float()).abs().amax() / 127).reshape(1, 1)
        out[f"s{si}_w"], out[f"s{si}_x"], out[f"s{si}_xe"] = bits(w), bits(x), bits(xe)
        out[f"s{si}_offs"] = offs.numpy().copy()
        out[f"s{si}_pre"], out[f"s{si}_act_scale"] = bits(pre), act_scale.numpy().copy()
        for v in VARIANTS:
            kind, gname = v.split("_")
            gran = PerRow() if gname == "PerRow" or kind == "static" else PerTensor()
            kw = dict()
            if kind == "dyn":
                kw = dict(act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow()))
            elif kind == "static":
                kw = dict(act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerTensor()),
                          act_quant_scale=act_scale, act_pre_scale=pre)
            wq = Int8Tensor.from_hp(w, gran, **kw)
            assert wq.scale.dtype == torch.float32 and wq.dtype == torch.bfloat16
            wname = "PerTensor" if v == "wo_PerTensor" else "PerRow"
            fields = dict(q=wq.qdata.numpy().copy(), scale=wq.scale.numpy().copy(), block_size=np.array(wq.block_size))
            for f, arr in fields.items():
                key = f"s{si}_{wname}_{f}"
                if key in out:   # the activation settings do not change the weight's quantization
                    assert np.array_equal(out[key], arr), (key, v)
                out[key] = arr
            if v == "wo_PerTensor":
                continue
            with torch.no_grad():
                for name, inp in (("y", x), ("ye", xe)):
                    lin, start = [], 0
                    for e in range(E):
                        if int(offs[e]) > start:   # the reference's quantizer fails on an empty expert's 0 rows
                            lin.append(F.linear(inp[start:int(offs[e])], wq[e]))
                        start = int(offs[e])
                    out[f"s{si}_{v}_{name}"] = bits(torch.cat(lin))
        cases.append(dict(shape=si, E=E, K=K, N=N, rows=rows, tail=tail, M=M))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "int8_3d.npz"), **out)
    print("wrote", len(cases), "shapes")


if __name__ == "__main__":
    main()
