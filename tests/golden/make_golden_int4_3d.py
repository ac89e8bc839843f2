"""Golden fixture for 3-D (MoE expert) int4 tile-packed weights: the REFERENCE's CPU primitives on bf16 [E, N, K]
weights padded as Int4TilePackedTo4dTensor.from_hp pads them (int4_tile_packed_to_4d_tensor.py:128-217):
_choose_qparams_affine_tinygemm, _quantize_affine_tinygemm and pack_tinygemm_scales_and_zeros of the [E, N, K/g] scales,
and one HQQ call on a whole 3-D weight.  N not a multiple of 8 and K not a multiple of 1024 exercise the padding.
    PYTHONPATH=/root/reference python tests/golden/make_golden_int4_3d.py
-> int4_3d.npz, per case: w (bf16 bits [E, N, K], unpadded), g, q (the codes two per byte as from_hp packs them, even k
in the high nibble: uint8 [E, N_pad, K_pad/2]), sz (scale_and_zero bf16 bits [E, K_pad/g, N_pad, 2]); HQQ case: q, s,
z (bf16 bits [E, N_pad, K_pad/g])."""
import os
import sys

import numpy as np
import torch

REF = os.environ.get("AO_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))

# name: (E, N, K, g, seed)
TINYGEMM = {"e3_n20_k768_g32": (3, 20, 768, 32, 11), "e2_n40_k1024_g128": (2, 40, 1024, 128, 12),
            "e4_n13_k1000_g256": (4, 13, 1000, 256, 13)}
HQQ = {"hqq_e3_n20_k768_g64": (3, 20, 768, 64, 14)}


def bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def pairs(q):
    q = q.to(torch.int32)
    return (q[..., ::2] << 4 | q[..., 1::2]).to(torch.uint8).numpy().copy()


def padded(E, N, K, seed):
    torch.manual_seed(seed)
    w = (torch.randn(E, N, K) * 0.02).to(torch.bfloat16)
    w[0] *= 8.0   # experts of very different magnitudes
    Np, Kp = -(-N // 8) * 8, -(-K // 1024) * 1024
    return w, torch.nn.functional.pad(w, (0, Kp - K, 0, Np - N))


def main():
    from torchao.quantization.quant_primitives import (
        MappingType, _choose_qparams_affine_tinygemm, _choose_qparams_and_quantize_affine_hqq, _quantize_affine_tinygemm)
    from torchao.quantization.utils import pack_tinygemm_scales_and_zeros

    out = {}
    for name, (E, N, K, g, seed) in TINYGEMM.items():
        w, wp = padded(E, N, K, seed)
        bs = (1, 1, g)
        s, z = _choose_qparams_affine_tinygemm(wp, MappingType.ASYMMETRIC, bs, torch.int32, 0, 15,
                                               scale_dtype=torch.bfloat16, zero_point_dtype=torch.bfloat16)
        q = _quantize_affine_tinygemm(wp, bs, s, z, torch.int32, 0, 15)
        sz = pack_tinygemm_scales_and_zeros(s.reshape(E, wp.shape[1], -1), z.reshape(E, wp.shape[1], -1), s.dtype)
        out.update({f"{name}__w": bits(w), f"{name}__g": np.array(g), f"{name}__q": pairs(q),
                    f"{name}__sz": bits(sz)})
        print(name, tuple(q.shape), tuple(sz.shape))
    for name, (E, N, K, g, seed) in HQQ.items():
        w, wp = padded(E, N, K, seed)
        q, s, z, _ = _choose_qparams_and_quantize_affine_hqq(wp, nbits=4, group_size=g, axis=1,
                                                             compute_dtype=torch.bfloat16, device="cpu", verbose=False,
                                                             raw_output=False)
        Np, Kp = wp.shape[1:]
        out.update({f"{name}__w": bits(w), f"{name}__g": np.array(g),
                    f"{name}__q": pairs(q.reshape(E, Np, Kp)),
                    f"{name}__s": bits(s).reshape(E, Np, Kp // g), f"{name}__z": bits(z).reshape(E, Np, Kp // g)})
        print(name, tuple(q.shape), tuple(s.shape))
    np.savez_compressed(os.path.join(HERE, "int4_3d.npz"), **out)


if __name__ == "__main__":
    main()
