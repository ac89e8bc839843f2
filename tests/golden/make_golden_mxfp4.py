"""Golden fixture for mxfp4 (MXTensor with float4_e2m1fn_x2 elements, block 32, RCEIL) from the REFERENCE on the CPU:

* to_mx codes (uint8 [M, K/2], even k in the low nibble), plain and blocked e8m0 scales and dequantize() of a 130 x 256
  bf16 input whose rows span 1e-3..1e3, with one all-zero block and one outlier;
* the e2m1 decode table (f4_unpacked_to_f32 of the 16 codes);
* quantize_ of an nn.Linear(256, 192, bias) with MXDynamicActivationMXWeightConfig(float4_e2m1fn_x2, EMULATED): its
  weight qdata and blocked scales, an input and the output;
* the safetensors wire form of one mxfp4 MXTensor (flatten_tensor_state_dict metadata and tensor bytes).

    PYTHONPATH=/root/reference python tests/golden/make_golden_mxfp4.py
-> mxfp4.npz (bf16 arrays as uint16 bits; the wire metadata as a JSON string)."""
import json
import os
import sys

import numpy as np
import torch

REF = os.environ.get("AO_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
FP4 = torch.float4_e2m1fn_x2


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def u8(t):
    return t.detach().contiguous().view(torch.uint8).numpy().copy()


def main():
    from torchao.prototype.mx_formats.config import ScaleCalculationMode
    from torchao.prototype.mx_formats.inference_workflow import MXDynamicActivationMXWeightConfig
    from torchao.prototype.mx_formats.kernels import f4_unpacked_to_f32
    from torchao.prototype.mx_formats.mx_tensor import MXTensor, QuantizeTensorToMXKwargs, to_mx
    from torchao.prototype.safetensors.safetensors_support import flatten_tensor_state_dict
    from torchao.quantization import quantize_
    from torchao.quantization.quantize_.common import KernelPreference

    out = {}
    torch.manual_seed(5)
    M, K = 130, 256
    x = torch.randn(M, K) * torch.logspace(-3, 3, M)[:, None]
    x[3, 32:64] = 0.0          # a zero block
    x[7, 100] = 3.0e4          # an outlier
    x = x.to(torch.bfloat16)
    out["x"] = bits(x)
    s, q = to_mx(x, FP4, 32, ScaleCalculationMode.RCEIL, False)
    out["q"], out["scale"] = u8(q), u8(s)
    sb, qb = to_mx(x, FP4, 32, ScaleCalculationMode.RCEIL, True)
    assert torch.equal(qb.view(torch.uint8), q.view(torch.uint8))
    out["scale_blocked"] = u8(sb)
    t = MXTensor.to_mx(x, FP4, 32, ScaleCalculationMode.RCEIL)
    assert t.shape == x.shape and t.qdata.shape == (M, K // 2)
    out["dequant"] = bits(t.dequantize(torch.bfloat16))
    out["dequant_f32"] = t.dequantize(torch.float32).numpy().copy()
    out["e2m1_table"] = f4_unpacked_to_f32(torch.arange(16, dtype=torch.uint8)).numpy().copy()

    torch.manual_seed(6)
    lin = torch.nn.Linear(256, 192, bias=True).to(torch.bfloat16)
    out["lin_w"], out["lin_b"] = bits(lin.weight), bits(lin.bias)
    quantize_(lin, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4,
                                                     kernel_preference=KernelPreference.EMULATED))
    w = lin.weight
    assert w.elem_dtype == FP4 and w.is_swizzled_scales
    out["lin_q"], out["lin_scale"] = u8(w.qdata), u8(w.scale)
    xin = (torch.randn(9, 256) * 2.0).to(torch.bfloat16)
    out["lin_x"] = bits(xin)
    with torch.no_grad():
        out["lin_y"] = bits(lin(xin))

    torch.manual_seed(8)
    wv = (torch.randn(64, 128) * 0.05).to(torch.bfloat16)
    wire = MXTensor.to_mx(wv, FP4, 32, act_quant_kwargs=QuantizeTensorToMXKwargs(elem_dtype=FP4, block_size=32))
    flat, meta = flatten_tensor_state_dict({"m.weight": wire})
    out["wire_meta"] = np.array(json.dumps(meta, sort_keys=True))
    out["wire_keys"] = np.array(json.dumps(sorted(flat)))
    for i, k in enumerate(sorted(flat)):
        out[f"wire_{i}"] = u8(flat[k])
    out["wire_dequant"] = bits(wire.dequantize(torch.bfloat16))
    np.savez_compressed(os.path.join(HERE, "mxfp4.npz"), **out)
    print("wrote", sorted(out), meta)


if __name__ == "__main__":
    main()
