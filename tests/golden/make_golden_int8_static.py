"""Golden fixture for static int8 activations (Int8StaticActivationInt8WeightConfig) from the REFERENCE on the CPU: for a
few small linears, quantize_(nn.Linear(K, N).bfloat16(), Int8StaticActivationInt8WeightConfig(...)) with a calibrated
activation scale, then F.linear through the reference's Int8Tensor handler.  K and N are not multiples of 128.  Every
case crosses PerTensor / PerRow activation scales, SYMMETRIC / ASYMMETRIC mappings, reduce_range off / on and an
``act_pre_scale`` of None, bf16 [K] or fp32 [K] (SmoothQuant's 1 / smoothing_factor, set on the weight as the reference's
SmoothQuant flow sets it); bias alternates.

The activations are bf16(v * s_row) with v mostly in {-127.5, -127, ..., 127.5}: with a power-of-two scale, x * (1 / s)
is exactly k + 0.5 for half of them (round half to even decides), and a few elements lie far past the clamp.  Rows
alternate power-of-two scales and scales with full mantissas; the zero points include -128, 127 and non-zero values.

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_int8_static.py
-> int8_static.npz: s<shape>_{w,b,x} (bf16 as uint16 bits), c<case>_{scale,zp,pre,q,y} (the calibrated scale f32, the
zero point int8, the pre-scale as bf16 bits or f32, the reference's activation codes Int8Tensor.from_hp(x * pre, ...,
scale=, zero_point=).qdata and the linear's output as bf16 bits; zp / pre only where the case has them) and ``cases``,
a JSON list describing each case."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(5, 160, 72), (16, 272, 40), (3, 400, 104)]   # (M, K, N)


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def activations(M, K, g):
    s_row = torch.tensor([2.0 ** -(3 + m % 4) if m % 2 == 0 else 0.0173 * (1 + m) for m in range(M)])
    v = torch.randint(-255, 256, (M, K), generator=g).float() / 2
    far = torch.rand(M, K, generator=g) < 0.04
    v = torch.where(far, torch.randint(-3000, 3000, (M, K), generator=g).float(), v)
    return (v * s_row[:, None]).to(torch.bfloat16), s_row


def main():
    import torch.nn.functional as F
    from torchao.quantization import Int8StaticActivationInt8WeightConfig, MappingType, PerRow, PerTensor, quantize_
    from torchao.quantization.quantize_.workflows.int8.int8_tensor import Int8Tensor

    out, cases = {}, []
    for si, (M, K, N) in enumerate(SHAPES):
        g = torch.Generator().manual_seed(200 + si)
        torch.manual_seed(200 + si)
        base = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
        with torch.no_grad():
            base.weight.mul_(torch.logspace(-2, 1, N)[:, None].to(torch.bfloat16))
        x, s_row = activations(M, K, g)
        out[f"s{si}_w"], out[f"s{si}_b"], out[f"s{si}_x"] = bits(base.weight), bits(base.bias), bits(x)
        pow2 = 2.0 ** torch.randint(-2, 3, (K,), generator=g).float()
        pre_f32 = torch.where(torch.arange(K) % 2 == 0, pow2, 1.0 / (0.3 + 2 * torch.rand(K, generator=g)))
        pres = {"none": None, "bf16": pre_f32.to(torch.bfloat16), "f32": pre_f32}
        for gname, gran in (("PerTensor", PerTensor()), ("PerRow", PerRow())):
            scale = (torch.tensor([[2.0 ** -4]]) if gname == "PerTensor" else s_row[:, None].clone()).float()
            for mapping in (MappingType.SYMMETRIC, MappingType.ASYMMETRIC):
                zp = None
                if mapping == MappingType.ASYMMETRIC:
                    zp = (torch.tensor([[5]]) if gname == "PerTensor"
                          else torch.tensor([[[-128, 127, 5, 0, -7][m % 5]] for m in range(M)])).to(torch.int8)
                for reduce_range in (False, True):
                    for pname, pre in pres.items():
                        bias = len(cases) % 2 == 0
                        lin = torch.nn.Linear(K, N, bias=bias).to(torch.bfloat16)
                        with torch.no_grad():
                            lin.weight.copy_(base.weight)
                            if bias:
                                lin.bias.copy_(base.bias)
                        quantize_(lin, Int8StaticActivationInt8WeightConfig(
                            act_quant_scale=scale, act_quant_zero_point=zp, granularity=gran, act_mapping_type=mapping,
                            set_inductor_config=False, reduce_range=reduce_range))
                        w = lin.weight
                        assert isinstance(w, Int8Tensor) and w.act_quant_scale is not None
                        w.act_pre_scale = pre
                        c = len(cases)
                        xp = x if pre is None else x * pre
                        xt = Int8Tensor.from_hp(xp, gran, mapping_type=mapping, scale=scale, zero_point=zp,
                                                reduce_range=reduce_range)
                        out[f"c{c}_scale"] = scale.numpy().copy()
                        if zp is not None:
                            out[f"c{c}_zp"] = zp.numpy().copy()
                        if pre is not None:
                            out[f"c{c}_pre"] = bits(pre) if pre.dtype == torch.bfloat16 else pre.numpy().copy()
                        out[f"c{c}_q"] = xt.qdata.numpy().copy()
                        with torch.no_grad():
                            out[f"c{c}_y"] = bits(F.linear(x, w, lin.bias))
                        cases.append(dict(shape=si, M=M, K=K, N=N, granularity=gname, mapping=mapping.name,
                                          reduce_range=reduce_range, pre=pname, bias=bias))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "int8_static.npz"), **out)
    print("wrote", len(cases), "cases")


if __name__ == "__main__":
    main()
