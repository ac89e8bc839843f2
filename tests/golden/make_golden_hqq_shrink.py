"""Golden fixture for HQQ int4 qparams where the solver's shrinkage step is active, and at g = 256, from the REFERENCE
on CPU (fp32 solver path), as make_golden_hqq.py does for int4_hqq.npz.
    PYTHONPATH=<reference checkout> python tests/golden/make_golden_hqq_shrink.py
Writes int4_hqq_shrink.npz: per case the bf16 weight bits, the reference's codes, scale and zero (bf16 bits), g.
The archive is written with fixed member timestamps, so a rerun gives the same bytes.

Weights of std 1 and 2 put a group's quantisation error past the point where relu(|d| - |d|^-0.3 / beta) is nonzero
(thousands of active elements per iteration); std 0.02 at g = 256 is the LLM-scale case of the widest group."""
import io
import os
import sys
import zipfile

import numpy as np
import torch

REF = os.environ.get("AO_REFERENCE")
if REF:
    sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))

# name: (N, K, g, seed, std)
CASES = {"s002_g256": (32, 2048, 256, 21, 0.02), "s1_g32": (64, 1024, 32, 22, 1.0),
         "s1_g256": (32, 2048, 256, 23, 1.0), "s2_g128": (32, 2048, 128, 24, 2.0)}


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def save_npz(path, arrays):
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    from torchao.quantization.quant_primitives import _choose_qparams_and_quantize_affine_hqq

    out = {}
    for name, (N, K, g, seed, std) in CASES.items():
        torch.manual_seed(seed)
        w = (torch.randn(N, K) * std).to(torch.bfloat16)
        q, s, z, _ = _choose_qparams_and_quantize_affine_hqq(w, nbits=4, group_size=g, axis=1, compute_dtype=torch.bfloat16,
                                                             device="cpu", verbose=False, raw_output=False)
        out[f"{name}__w"] = bits(w)
        out[f"{name}__q"] = q.numpy().copy()
        out[f"{name}__s"] = bits(s).reshape(N, K // g)
        out[f"{name}__z"] = bits(z).reshape(N, K // g)
        out[f"{name}__g"] = np.array(g)
    save_npz(os.path.join(HERE, "int4_hqq_shrink.npz"), out)
    print("wrote", sorted(out))


if __name__ == "__main__":
    main()
