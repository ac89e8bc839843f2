"""Golden fixture for static e4m3 activations (Float8StaticActivationFloat8WeightConfig) from the REFERENCE on the CPU.

* Weights: PrototypeFloat8Tensor.from_hp(w, e4m3, PerTensor() / PerRow()) of a few small bf16 linears (K and N not
  multiples of 128): the codes and scales.
* Activation codes: PrototypeFloat8Tensor.from_hp(x, e4m3, granularity, scale=s) (the reference's
  _quantize_affine_float8 with the calibrated scale) for PerTensor [1, 1] and PerRow [M, 1] scales.  The inputs mix
  values that land exactly halfway between two e4m3 codes (round half to even decides), values past +-448 s, +-0,
  +-inf and NaN; the scales include 0, a subnormal (1e-40), a huge one (3e38) and full-mantissa ones.
* Linears: quantize_(nn.Linear(K, N).bfloat16(), Float8StaticActivationFloat8WeightConfig(act_quant_scale=s,
  granularity=PerTensor(), output_act_quant_scale=s_o)) and F.linear through the reference's handler, with and
  without bias and with and without the output fake-quant (s_o chosen so that part of the outputs saturate).  PerRow
  linears do not run on the CPU (torch._scaled_mm rowwise is CUDA-only).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_fp8_static.py
-> fp8_static.npz: s<shape>_{w,b,x} (bf16 as uint16 bits), s<shape>_{PerTensor,PerRow}_{wq,ws} (weight codes as
uint8, scales f32), q<case>_{x,scale,q} (quantizer cases: bf16 bits, f32 scale, e4m3 codes as uint8),
c<case>_{scale,oscale,y} (linear cases: the scales f32 and the output as bf16 bits; oscale only where the case has one)
and ``qcases`` / ``cases``, JSON lists describing each case."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(5, 160, 48), (16, 272, 80), (3, 400, 112)]   # (M, K, N)
SCALES = [2.0 ** -4, 0.0173, 0.0, 1e-40, 3e38, 1.0]


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def codes(t):
    return t.detach().contiguous().view(torch.uint8).numpy().copy()


def activations(M, K, g):
    s_row = torch.tensor([2.0 ** -(3 + m % 4) if m % 2 == 0 else 0.0173 * (1 + m) for m in range(M)])
    v = torch.randn(M, K, generator=g) * 40
    far = torch.rand(M, K, generator=g) < 0.04
    v = torch.where(far, torch.randint(-3000, 3000, (M, K), generator=g).float(), v)
    return (v * s_row[:, None]).to(torch.bfloat16), s_row


def special_activations(K, g):
    """Rows of e4m3 midpoints (times 2^-4, the PerTensor test scale), values past the clamp, and +-0, +-inf, NaN."""
    e4m3 = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).float()
    e4m3 = e4m3[torch.isfinite(e4m3)].unique()
    mids = (e4m3[1:] + e4m3[:-1]) / 2   # exact in bf16: e4m3 has 3 mantissa bits, a midpoint 4
    rows = []
    for r in range(4):
        v = mids[torch.randint(0, len(mids), (K,), generator=g)] * 2.0 ** -4
        if r % 2:
            v = torch.where(torch.rand(K, generator=g) < 0.2, v * 300, v)   # past +-448 s
        rows.append(v)
    sp = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -3e38, 448 * 2.0 ** -4])
    edge = torch.randn(K, generator=g)
    edge[: len(sp)] = sp
    rows.append(edge)
    return torch.stack(rows).to(torch.bfloat16)


def main():
    import torch.nn.functional as F
    from torchao.prototype.quantization.float8_static_quant.prototype_float8_tensor import PrototypeFloat8Tensor
    from torchao.prototype.quantization.quant_api import Float8StaticActivationFloat8WeightConfig
    from torchao.quantization import PerRow, PerTensor, quantize_

    out, qcases, cases = {}, [], []

    def quant_case(x, scale, gname, si):
        t = PrototypeFloat8Tensor.from_hp(x, torch.float8_e4m3fn, PerTensor() if gname == "PerTensor" else PerRow(),
                                          scale=scale)
        q = len(qcases)
        out[f"q{q}_x"], out[f"q{q}_scale"], out[f"q{q}_q"] = bits(x), scale.numpy().copy(), codes(t.qdata)
        qcases.append(dict(shape=si, granularity=gname, M=x.shape[0], K=x.shape[1]))

    for si, (M, K, N) in enumerate(SHAPES):
        g = torch.Generator().manual_seed(300 + si)
        torch.manual_seed(300 + si)
        base = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
        with torch.no_grad():
            base.weight.mul_(torch.logspace(-2, 1, N)[:, None].to(torch.bfloat16))
        x, s_row = activations(M, K, g)
        out[f"s{si}_w"], out[f"s{si}_b"], out[f"s{si}_x"] = bits(base.weight), bits(base.bias), bits(x)
        for gname, gran in (("PerTensor", PerTensor()), ("PerRow", PerRow())):
            wt = PrototypeFloat8Tensor.from_hp(base.weight, torch.float8_e4m3fn, gran)
            out[f"s{si}_{gname}_wq"], out[f"s{si}_{gname}_ws"] = codes(wt.qdata), wt.scale.detach().numpy().copy()
        # quantizer cases: the linear's activations, then the special rows, with every scale
        quant_case(x, torch.tensor([[2.0 ** -4]]), "PerTensor", si)
        quant_case(x, s_row[:, None].clone().float(), "PerRow", si)
        xs = special_activations(K, g)
        for s in SCALES:
            quant_case(xs, torch.tensor([[s]], dtype=torch.float32), "PerTensor", si)
        quant_case(xs, torch.tensor([[SCALES[m % len(SCALES)]] for m in range(xs.shape[0])], dtype=torch.float32),
                   "PerRow", si)
        # PerTensor linears
        scale = torch.tensor([[2.0 ** -4]])
        with torch.no_grad():
            y0 = F.linear(x, base.weight, base.bias).float()
        for qdq in (False, True):
            for bias in (True, False):
                oscale = (y0.abs().amax() / 448 * 0.5).reshape(1, 1) if qdq else None
                lin = torch.nn.Linear(K, N, bias=bias).to(torch.bfloat16)
                with torch.no_grad():
                    lin.weight.copy_(base.weight)
                    if bias:
                        lin.bias.copy_(base.bias)
                quantize_(lin, Float8StaticActivationFloat8WeightConfig(
                    act_quant_scale=scale, granularity=PerTensor(), set_inductor_config=False,
                    output_act_quant_scale=oscale))
                assert isinstance(lin.weight, PrototypeFloat8Tensor)
                c = len(cases)
                out[f"c{c}_scale"] = scale.numpy().copy()
                if oscale is not None:
                    out[f"c{c}_oscale"] = oscale.detach().float().numpy().copy()
                with torch.no_grad():
                    out[f"c{c}_y"] = bits(F.linear(x, lin.weight, lin.bias))
                cases.append(dict(shape=si, M=M, K=K, N=N, bias=bias, qdq=qdq))
    out["qcases"] = np.array(json.dumps(qcases))
    out["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "fp8_static.npz"), **out)
    print("wrote", len(qcases), "quantizer cases and", len(cases), "linear cases")


if __name__ == "__main__":
    main()
