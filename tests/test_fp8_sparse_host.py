"""2:4-sparse fp8 (Float8DynamicActivationFloat8WeightConfig, packing_format SPARSE_2D_DATA_2D_METADATA) without a GPU:
the config, the packing-format enum and its alias against the reference's (golden/fp8_sparse.npz), the 2:4 compressor's
round trip, shapes and metadata, the handler's rejections and skips, torch.save / load, clone, fusion, the C ABI's
argument checks, the op's meta kernel, and the registers, stack and shared memory of every
ts_gemm_kernel<SparseF8Fmt, N>."""
import ctypes
import json
import logging
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import streamk_model as sk
from test_decode_residency import RESERVED_PER_CTA, SMEM_PER_SM, resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fp8_sparse.npz")
VALID_NIBBLES = {0b0100, 0b1000, 0b1100, 0b1001, 0b1101, 0b1110}


def mod():
    from ao_b200.quantization.quantize_.workflows.float8 import float8_sparse_2x4_2d_data_2d_metadata_tensor as m

    return m


def sparse_config(**kw):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8PackingFormat, PerRow

    kw.setdefault("granularity", PerRow())
    return Float8DynamicActivationFloat8WeightConfig(packing_format=Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA, **kw)


def pruned(N, K, seed=0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g)
    idx = torch.rand(N, K // 4, 4, generator=g).argsort(-1)[..., :2]
    mask = torch.zeros(N, K // 4, 4, dtype=torch.bool).scatter_(-1, idx, True).reshape(N, K)
    return (w * mask).to(dtype)


def codes(N, K, seed=0):
    """2:4 e4m3 codes with empty groups, single codes at every position and -0.0"""
    q = pruned(N, K, seed, torch.float32).mul(3).to(torch.float8_e4m3fn)
    u = q.view(torch.uint8).reshape(N, K // 4, 4)
    u[:, 0] = 0
    if K >= 24:
        for p in range(4):
            one = torch.zeros(4, dtype=torch.uint8)
            one[p] = 0x40 + p
            u[:, 1 + p] = one
        u[:, 5] = torch.tensor([0x80, 0x44, 0x80, 0xC0], dtype=torch.uint8)
    return q


def plain(q):
    """codes with -0.0 as +0 (the compressor never stores -0.0)"""
    u = q.view(torch.uint8)
    return torch.where((u & 0x7F) == 0, torch.zeros_like(u), u)


# ---------------------------------------------------------------- config and enum
def test_config_enum_and_json_match_the_reference():
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.quantization import Float8PackingFormat

    g = dict(np.load(GOLDEN))
    want = json.loads(str(g["config_json"]))
    got = config_to_dict(sparse_config())
    assert got == want
    assert config_from_dict(want) == sparse_config()
    members = json.loads(str(g["packing_formats"]))
    for name, value in members.items():
        assert Float8PackingFormat[name].value == value
    assert Float8PackingFormat.OPAQUE.value == "opaque"   # this engine's extra member
    name, value = json.loads(str(g["sparse_cutlass"]))
    assert Float8PackingFormat.SPARSE_CUTLASS is Float8PackingFormat[name] and Float8PackingFormat.SPARSE_CUTLASS == value


# ---------------------------------------------------------------- the compressor
@pytest.mark.parametrize("N,K", [(64, 128), (80, 160), (16, 192), (200, 224), (128, 4096), (48, 32), (130, 96)])
def test_compressor_round_trip_shapes_and_nibbles(N, K):
    m = mod()
    q = codes(N, K, seed=N + K)
    qd, meta = m.compress_2x4_e4m3(q)
    assert qd.dtype == torch.float8_e4m3fn and tuple(qd.shape) == (N, K // 2)
    assert meta.dtype == torch.uint8 and tuple(meta.shape) == ((N + 63) // 64 * 64, (K + 127) // 128 * 16)
    assert torch.equal(m.decompress_2x4_e4m3(qd, meta).view(torch.uint8), plain(q))
    rows = m.metadata_rows(meta)
    nib = torch.stack([rows & 0xF, rows >> 4], -1).reshape(rows.shape[0], -1)
    live = nib[:N, : K // 4]
    empty = (plain(q).reshape(N, K // 4, 4) == 0).all(-1)
    assert set(live[~empty].unique().tolist()) <= VALID_NIBBLES
    assert bool((live[empty] == 0).all())   # the reference's compressor writes 0b0000 for an all-zero group
    pad = torch.ones_like(nib, dtype=torch.bool)
    pad[:N, : K // 4] = False
    assert bool((nib[pad] == 0).all())


def test_single_codes_are_placed_as_the_reference_places_them():
    m = mod()
    q = torch.zeros(64, 128, dtype=torch.uint8)
    q[0, :4] = torch.tensor([0x38, 0, 0, 0])
    q[0, 4:8] = torch.tensor([0, 0, 0, 0x38])
    q[0, 8:12] = torch.tensor([0, 0x38, 0x40, 0])
    qd, meta = m.compress_2x4_e4m3(q.view(torch.float8_e4m3fn))
    assert qd.view(torch.uint8)[0, :6].tolist() == [0x38, 0, 0, 0x38, 0x38, 0x40]
    # groups 0 / 1: (0, 3) = 0b1100, group 2: (1, 2) = 0b1001, group 3 empty: 0b0000
    assert m.metadata_rows(meta)[0, :2].tolist() == [0b1100_1100, 0b0000_1001]


def test_a_group_with_three_codes_raises_naming_it():
    q = pruned(64, 128).to(torch.float8_e4m3fn)
    u = q.view(torch.uint8)
    u[5, 36:40] = torch.tensor([0x38, 0x38, 0x38, 0])
    with pytest.raises(ValueError, match="row 5, group 9"):
        mod().compress_2x4_e4m3(q)


# ---------------------------------------------------------------- the handler
def test_quantize_makes_a_sparse_weight_with_the_dense_codes():
    from ao_b200.quantization import Float8Sparse2x4_2DData2DMetadataTensor, Float8Tensor, PerRow, quantize_

    lin = nn.Linear(256, 128, bias=False).to(torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(pruned(128, 256))
    w0 = lin.weight.detach().clone()
    quantize_(lin, sparse_config())
    w = lin.weight
    assert isinstance(w, Float8Sparse2x4_2DData2DMetadataTensor) and tuple(w.shape) == (128, 256)
    assert w.dtype == torch.bfloat16 and list(w.block_size) == [1, 256] and tuple(w.scale.shape) == (128, 1)
    assert w.act_quant_kwargs.granularity == PerRow()
    dense = Float8Tensor.from_hp(w0, granularity=PerRow())
    assert torch.equal(mod().decompress_2x4_e4m3(w.qdata, w.sparse_metadata).view(torch.uint8), plain(dense.qdata))
    assert torch.equal(w.scale, dense.scale)
    want = (plain(dense.qdata).view(torch.float8_e4m3fn).float() * dense.scale).to(torch.bfloat16)
    assert torch.equal(w.dequantize(), want)
    assert torch.equal(w.to(torch.float), want.float())
    assert torch.equal(w.dequantize(torch.float32), want.float())


def test_rejections():
    from ao_b200.quantization import Float8PackingFormat, PerTensor, quantize_

    lin = lambda: nn.Linear(128, 64).to(torch.bfloat16)
    dense = nn.Linear(128, 64).to(torch.bfloat16)
    with pytest.raises(ValueError, match="not 2:4 sparse"):
        quantize_(dense, sparse_config())
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow

    with pytest.raises(NotImplementedError, match="ROCm"):
        quantize_(lin(), Float8DynamicActivationFloat8WeightConfig(
            granularity=PerRow(), packing_format=Float8PackingFormat.SPARSE_1D_DATA_1D_METADATA))
    with pytest.raises(AssertionError, match="per-row"):
        quantize_(lin(), sparse_config(granularity=PerTensor()))
    with pytest.raises(AssertionError, match="e4m3"):
        quantize_(lin(), sparse_config(weight_dtype=torch.float8_e5m2))
    with pytest.raises(NotImplementedError, match="bf16 weights only"):
        quantize_(nn.Linear(128, 64), sparse_config())
    with pytest.raises(AssertionError, match="hp_value_lb"):
        mod().Float8Sparse2x4_2DData2DMetadataTensor.from_hp(pruned(64, 128), hp_value_lb=1e-3)


def test_k_not_a_multiple_of_32_is_skipped_with_a_log_line(caplog):
    from ao_b200.quantization import quantize_

    lin = nn.Linear(144, 64).to(torch.bfloat16)   # K % 16 == 0, K % 32 != 0
    w0 = lin.weight.detach().clone()
    with caplog.at_level(logging.INFO):
        quantize_(lin, sparse_config())
    assert type(lin.weight.data) is torch.Tensor and torch.equal(lin.weight.detach(), w0)
    assert "in_features=144 is not a multiple of 32" in caplog.text


def test_save_load_clone_and_fusion_skip(tmp_path):
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.quantization import Float8Sparse2x4_2DData2DMetadataTensor, quantize_

    lin = nn.Linear(256, 128).to(torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(pruned(128, 256, seed=3))
    quantize_(lin, sparse_config())
    torch.save(lin.state_dict(), tmp_path / "w.pt")
    sd = torch.load(tmp_path / "w.pt", weights_only=True)
    w, v = lin.weight, sd["weight"]
    assert type(v) is Float8Sparse2x4_2DData2DMetadataTensor
    c = w.clone()
    for a in (v, c):
        assert all(torch.equal(getattr(a, n).view(torch.uint8) if getattr(a, n).dtype != torch.float32 else getattr(a, n),
                               getattr(w, n).view(torch.uint8) if getattr(w, n).dtype != torch.float32 else getattr(w, n))
                   for n in ("qdata", "sparse_metadata", "scale"))
        assert a.act_quant_kwargs == w.act_quant_kwargs and list(a.block_size) == list(w.block_size)
    assert c.qdata.data_ptr() != w.qdata.data_ptr()

    class Attn(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj, self.v_proj = (nn.Linear(256, 128, bias=False).to(torch.bfloat16) for _ in range(3))

    m = Attn()
    with torch.no_grad():
        for i, l in enumerate((m.q_proj, m.k_proj, m.v_proj)):
            l.weight.copy_(pruned(128, 256, seed=10 + i))
    quantize_(m, sparse_config())
    assert fuse_parallel_linears(m) == 0
    assert all(isinstance(l.weight, Float8Sparse2x4_2DData2DMetadataTensor) for l in (m.q_proj, m.k_proj, m.v_proj))


# ---------------------------------------------------------------- op surface
def test_meta_kernel_and_schema():
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    xq = torch.empty(130, 512, dtype=torch.float8_e4m3fn, device="meta")
    wq = torch.empty(192, 256, dtype=torch.float8_e4m3fn, device="meta")
    y = ops.fp8_sparse_linear(xq, torch.empty(130, device="meta"), wq, torch.empty(192, 64, dtype=torch.uint8, device="meta"),
                              torch.empty(192, device="meta"), None)
    assert y.shape == (130, 192) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(ops.fp8_sparse_linear.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_meta, Tensor w_scale, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    lin = lambda M, K, N, x=None, s=None, w=None, m=None, p=None: lib.ao_fp8_sparse_linear(
        ctypes.c_void_p(x), ctypes.c_void_p(s), M, K, ctypes.c_void_p(w), ctypes.c_void_p(m), ctypes.c_void_p(p), N,
        None, ctypes.c_void_p(p), None, z, None)
    assert lin(4, 4112, 256) == -1 and b"K=4112 must be a multiple of 32" in lib.ao_b200_last_error()
    assert lin(4, 4096, 200) == -1 and b"N=200 must be a multiple of 16" in lib.ao_b200_last_error()
    assert lin(4, 0, 256) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    assert lin(4, 4096, 256) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert lin(0, 4096, 256) == 0   # M == 0: nothing to do, no CUDA call (this process has no device)
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15
    assert lin(4, 4096, 256, x=a + 8, s=a, w=a, m=a, p=a) == -1 and b"xq must be 16-byte" in lib.ao_b200_last_error()
    assert lin(4, 4096, 256, x=a, s=a, w=a + 4, m=a, p=a) == -1 and b"wq must be 16-byte" in lib.ao_b200_last_error()
    assert lin(4, 4096, 256, x=a, s=a, w=a, m=a + 8, p=a) == -1 and b"w_meta must be 16-byte" in lib.ao_b200_last_error()


# ---------------------------------------------------------------- the budget of the format
# Cfg<SparseF8Fmt, N> is streamk_model.ring("fp8_sparse", N): a stage is 8 KiB of compressed codes, the 2 KiB metadata
# slot and N x 128 activation bytes; two CTAs per SM at decode tiles (DECODE_2CTA), else a 200 KB ring
@pytest.mark.parametrize("n_mma", [16, 32, 64, 128])
def test_tiles_registers_stack_and_shared_memory(n_mma):
    src = open(os.path.join(ROOT, "ao_b200", "csrc", "lowp_linear.cu")).read()
    body = src[src.index("struct SparseF8Fmt"):]
    body = body[:body.index("\n};\n")]
    assert "DECODE_2CTA = true;" in body and "MAX_N_MMA = 128;" in body and "PROMOTE = false;" in body
    usage = resource_usage()
    assert ("SparseF8Fmt", n_mma) in usage, f"ts_gemm_kernel<SparseF8Fmt, {n_mma}> not built"
    reg, stack = usage[("SparseF8Fmt", n_mma)]
    stage, ctas, stages, _ = sk.ring("fp8_sparse", n_mma)
    assert stage == 8192 + 2048 + n_mma * 128 and ctas == (2 if n_mma <= 32 else 1)
    # two CTAs per SM: 80 registers per thread at launch (the consumers grow to 104 with setmaxnreg)
    assert stack == 0 and reg <= (80 if ctas == 2 else 168), (reg, stack)
    smem = sk.ring_smem("fp8_sparse", n_mma)
    assert stages >= 2 and ctas * (smem + RESERVED_PER_CTA) <= SMEM_PER_SM
