"""Golden fixture for NF4 weights (NF4Tensor / NF4WeightOnlyConfig) from the REFERENCE on the CPU: for a few small bf16
linears, NF4Tensor.from_tensor(weight, block_size, scaler_block_size), its get_original_weight() and F.linear through
the reference's NF4 override (F.linear on the dequantized weight, then + bias).  The cases cover N not a multiple of
128, block sizes 64 and 128, scaler block sizes 256 and 64, and with and without bias.  Two inputs per linear:

* ``x``: random bf16 (fp32 sums round, so the accumulation order can show in the last bf16 bit);
* ``xe``: one-hot rows, +-2^j at one column per row: every output is one product w~[n, k] * 2^j, exact in fp32, so it
  is determined bit for bit: bf16(bf16(w~ * 2^j) + bias).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_nf4.py
-> nf4.npz (bf16 arrays as uint16 bits, codes uint8, scalers int8): c<case>_<field> and ``cases``, a JSON list of
(M, K, N, block_size, scaler_block_size, bias)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(5, 256, 192, 64, 256, True), (3, 256, 160, 128, 64, False), (4, 512, 64, 64, 256, True)]


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def main():
    import torch.nn.functional as F
    from torchao.quantization import NF4Tensor

    out = {}
    for ci, (M, K, N, bs, sbs, has_bias) in enumerate(CASES):
        torch.manual_seed(300 + ci)
        lin = torch.nn.Linear(K, N, bias=has_bias).to(torch.bfloat16)
        with torch.no_grad():
            lin.weight.mul_(torch.logspace(-1, 1, N)[:, None].to(torch.bfloat16))   # rows over two decades
        w = lin.weight.detach()
        t = NF4Tensor.from_tensor(w, bs, sbs)
        x = (torch.randn(M, K) * 1.5).to(torch.bfloat16)
        xe = torch.zeros(M, K)
        cols = torch.randint(0, K, (M,))
        xe[torch.arange(M), cols] = torch.pow(2.0, torch.randint(-3, 4, (M,)).float()) * (torch.randint(0, 2, (M,)) * 2 - 1)
        xe = xe.to(torch.bfloat16)
        b = lin.bias.detach() if has_bias else None
        out[f"c{ci}_w"], out[f"c{ci}_x"], out[f"c{ci}_xe"] = bits(w), bits(x), bits(xe)
        if has_bias:
            out[f"c{ci}_b"] = bits(b)
        out[f"c{ci}_quantized_data"] = t.quantized_data.numpy().copy()
        out[f"c{ci}_quantized_scalers"] = t.quantized_scalers.numpy().copy()
        out[f"c{ci}_quantization_factor"] = bits(t.quantization_factor)
        out[f"c{ci}_scaler_mean"] = bits(t.scaler_mean.reshape(1))
        out[f"c{ci}_nf4"] = bits(t.nf4)
        out[f"c{ci}_orig"] = bits(t.get_original_weight())
        out[f"c{ci}_y"] = bits(F.linear(x, t, b))
        out[f"c{ci}_ye"] = bits(F.linear(xe, t, b))
    out["cases"] = np.array(json.dumps(CASES))
    np.savez_compressed(os.path.join(HERE, "nf4.npz"), **out)


if __name__ == "__main__":
    main()
