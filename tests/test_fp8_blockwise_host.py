"""Blockwise fp8 (Float8DynamicActivationFloat8WeightConfig with [PerBlock([1, 128]), PerBlock([128, 128])]) without a
GPU: the config against the reference's (golden/fp8_blockwise.npz: defaults, accepted spellings, JSON), the package's
weight and activation quantizers bit for bit against the reference's codes and scales, the shape rules, slicing,
torch.save / safetensors, fusion, the C ABI's argument checks, the ops' meta kernels, and the registers, stack and
shared memory of every ts_gemm_kernel<BlockwiseF8Fmt, N>."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import streamk_model as sk
from test_decode_residency import RESERVED_PER_CTA, SMEM_PER_SM, resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fp8_blockwise.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def bf16(bits):
    return torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16)


def blockwise_config(**kw):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock

    return Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])], **kw)


def blockwise_weight(n=256, k=256, seed=0, scale=0.05):
    from ao_b200.quantization import Float8Tensor, PerBlock
    from ao_b200.quantization.quantize_.workflows.float8.float8_tensor import QuantizeTensorToFloat8Kwargs

    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, k, generator=g) * scale).to(torch.bfloat16)
    return Float8Tensor.from_hp(w, granularity=PerBlock([128, 128]),
                                act_quant_kwargs=QuantizeTensorToFloat8Kwargs(granularity=PerBlock([1, 128])))


def same(a, b):
    return (type(a) is type(b) and torch.equal(a.qdata.view(torch.uint8), b.qdata.view(torch.uint8))
            and torch.equal(a.scale, b.scale) and list(a.block_size) == list(b.block_size)
            and a.act_quant_kwargs == b.act_quant_kwargs and a.mm_config == b.mm_config and a.dtype == b.dtype)


# ---------------------------------------------------------------- config
def test_config_defaults_spellings_and_json(golden):
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.float8.inference import Float8MMConfig
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock, PerRow

    c = blockwise_config()
    assert c.mm_config == Float8MMConfig(use_fast_accum=False)
    assert Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()).mm_config.use_fast_accum   # unchanged
    assert config_to_dict(c) == json.loads(str(golden["config_json"]))
    assert config_from_dict(json.loads(str(golden["config_json"]))) == c
    spellings = {"list_of_lists": [PerBlock([1, 128]), PerBlock([128, 128])],
                 "tuple_of_lists": (PerBlock([1, 128]), PerBlock([128, 128])),
                 "list_of_tuples": [PerBlock((1, 128)), PerBlock((128, 128))],
                 "tuple_of_tuples": (PerBlock((1, 128)), PerBlock((128, 128)))}
    want = json.loads(str(golden["spellings"]))
    for name, g in spellings.items():
        try:
            Float8DynamicActivationFloat8WeightConfig(granularity=g)
            got = "ok"
        except ValueError:
            got = "ValueError"
        assert got == want[name], name


@pytest.mark.parametrize("gran", [
    "a1x128_wrow", "arow_w128", "a1x64", "w64x64", "w128x128_only"])
def test_mixed_and_other_block_pairs_raise(gran):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock, PerRow

    g = {"a1x128_wrow": [PerBlock([1, 128]), PerRow()], "arow_w128": [PerRow(), PerBlock([128, 128])],
         "a1x64": [PerBlock([1, 64]), PerBlock([128, 128])], "w64x64": [PerBlock([1, 128]), PerBlock([64, 64])],
         "w128x128_only": PerBlock([128, 128])}[gran]
    with pytest.raises(ValueError):
        Float8DynamicActivationFloat8WeightConfig(granularity=g)


def test_kernel_preference_and_version_rules():
    from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference

    for kp in (KernelPreference.AUTO, KernelPreference.TORCH):
        assert blockwise_config(kernel_preference=kp).kernel_preference == kp
    with pytest.raises(AssertionError):
        blockwise_config(kernel_preference=KernelPreference.MSLK)
    with pytest.raises(AssertionError):
        blockwise_config(version=1)


# ---------------------------------------------------------------- quantizers against the reference
def test_weight_codes_and_scales_match_the_reference(golden):
    from ao_b200.quantization import Float8Tensor, PerBlock

    w = Float8Tensor.from_hp(bf16(golden["w"]), granularity=PerBlock([128, 128]))
    assert list(w.block_size) == [128, 128] and w.scale.dtype == torch.float32
    assert np.array_equal(w.qdata.view(torch.uint8).numpy(), golden["w_q"])
    assert np.array_equal(w.scale.numpy().view(np.uint32), golden["w_scale"].view(np.uint32))


@pytest.mark.parametrize("name", ["x", "x3"])
def test_activation_codes_and_scales_match_the_reference(golden, name):
    from ao_b200.quantization import Float8Tensor, PerBlock

    x = bf16(golden[name])
    t = Float8Tensor.from_hp(x, granularity=PerBlock([1, 128]))
    assert list(t.block_size) == [1] * (x.dim() - 1) + [128]
    assert np.array_equal(t.qdata.view(torch.uint8).numpy(), golden[f"{name}_q"])
    assert np.array_equal(t.scale.numpy().view(np.uint32), golden[f"{name}_scale"].view(np.uint32))


def test_fixture_holds_the_edge_blocks(golden):
    """All-zero blocks have scale 0 and NaN codes, some activation scales are subnormal fp32, and a weight block holds
    the largest finite bf16: the fixture covers them."""
    s = golden["x_scale"]
    assert s[0, 0] == 0 and (golden["x_q"][0, :128] & 0x7F == 0x7F).all()
    assert ((s > 0) & (s < np.finfo(np.float32).tiny)).any()
    assert golden["w_scale"][1, 1] == 0 and (golden["w_q"][128:, 128:] & 0x7F == 0x7F).all()
    assert golden["w_scale"][0, 0] > 1e35   # the largest finite bf16 / 448


# ---------------------------------------------------------------- shapes through quantize_
@pytest.mark.parametrize("k,n", [(256, 144), (144, 256)])
def test_n_or_k_not_a_multiple_of_128_raises(k, n):
    from ao_b200.quantization import quantize_

    lin = nn.Linear(k, n).to(torch.bfloat16)
    with pytest.raises(AssertionError):
        quantize_(lin, blockwise_config())


def test_fp8_incompatible_shapes_are_skipped():
    from ao_b200.quantization import quantize_

    lin = nn.Linear(136, 256).to(torch.bfloat16)   # K % 16 != 0: _fp8_mm_compat skips the layer
    w0 = lin.weight.detach().clone()
    quantize_(lin, blockwise_config())
    assert type(lin.weight.data) is torch.Tensor and torch.equal(lin.weight.detach(), w0)


def test_quantize_makes_a_blockwise_weight():
    from ao_b200.quantization import Float8Tensor, PerBlock, quantize_

    lin = nn.Linear(384, 256).to(torch.bfloat16)
    quantize_(lin, blockwise_config())
    w = lin.weight
    assert isinstance(w, Float8Tensor) and list(w.block_size) == [128, 128] and tuple(w.scale.shape) == (2, 3)
    assert w.act_quant_kwargs.granularity == PerBlock([1, 128]) and w.mm_config.use_fast_accum is False


def test_get_block_size_pads_a_shorter_block_with_leading_ones():
    from ao_b200.quantization import PerBlock
    from ao_b200.quantization.utils import get_block_size

    assert get_block_size((2, 3, 256), PerBlock([1, 128])) == (1, 1, 128)
    assert get_block_size((256, 512), PerBlock([128, 128])) == (128, 128)


# ---------------------------------------------------------------- slicing, saving, fusion
def test_slice_by_whole_blocks():
    w = blockwise_weight(384, 256)
    full = w.dequantize()
    rows = w[128:384]
    assert tuple(rows.scale.shape) == (2, 2) and torch.equal(rows.dequantize(), full[128:384])
    cols = w.narrow(1, 128, 128)
    assert tuple(cols.scale.shape) == (3, 1) and torch.equal(cols.dequantize(), full[:, 128:256])
    assert list(cols.block_size) == [128, 128]
    for bad in ((0, 64, 192), (0, 0, 100), (1, 32, 256)):
        dim, lo, hi = bad
        with pytest.raises(ValueError, match="not aligned"):
            torch.ops.aten.slice.Tensor(w, dim, lo, hi)


def test_narrow_and_copy_write_through():
    dst, src = blockwise_weight(256, 256, seed=1), blockwise_weight(256, 256, seed=2)
    for lo in (0, 128):
        dst.narrow(0, lo, 128).copy_(src.narrow(0, lo, 128))
    assert same(dst, src)


def test_torch_save_safetensors_and_to(tmp_path):
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import quantize_

    lin = nn.Linear(256, 384).to(torch.bfloat16)
    quantize_(lin, blockwise_config())
    torch.save(lin.state_dict(), tmp_path / "w.pt")
    back = torch.load(tmp_path / "w.pt", weights_only=True)["weight"]
    assert same(back, lin.weight)
    flat, meta = flatten_tensor_state_dict({"m.weight": lin.weight.data})
    assert json.loads(meta["m.weight"])["_data"]["block_size"] == [128, 128]
    assert all(type(v) is torch.Tensor for v in flat.values())
    sd, leftover = unflatten_tensor_state_dict(flat, meta)
    assert leftover == {} and same(sd["m.weight"], lin.weight)
    moved = lin.weight.to("cpu")
    assert same(moved, lin.weight)


def test_fusion_concatenates_or_declines():
    from ao_b200.fusion import cat_out_features
    from ao_b200.quantization import Float8Tensor

    ws = [blockwise_weight(n, seed=i) for i, n in enumerate((512, 128, 128))]   # q|k|v-like
    cat = cat_out_features(ws)
    assert cat is not None and list(cat.block_size) == [128, 128] and tuple(cat.scale.shape) == (6, 2)
    assert torch.equal(cat.dequantize(), torch.cat([w.dequantize() for w in ws], 0))
    assert same(cat[512:640], ws[1])
    # a member whose N is not a multiple of 128 (built directly: from_hp refuses one) is declined
    odd = Float8Tensor(ws[1].qdata[:64], ws[1].scale, [128, 128], ws[1].mm_config, ws[1].act_quant_kwargs,
                       ws[1].kernel_preference, ws[1].dtype)
    assert cat_out_features([ws[0], odd]) is None


# ---------------------------------------------------------------- op surface
def test_meta_shapes_and_schemas():
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    x = torch.empty(130, 512, dtype=torch.bfloat16, device="meta")
    q, s = ops.fp8_quantize_1x128(x)
    assert q.shape == (130, 512) and q.dtype == torch.float8_e4m3fn and s.shape == (4, 132) and s.dtype == torch.float32
    wq = torch.empty(256, 512, dtype=torch.float8_e4m3fn, device="meta")
    y = ops.fp8_blockwise_linear(q, s, wq, torch.empty(2, 4, device="meta"), None)
    assert y.shape == (130, 256) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(ops.fp8_quantize_1x128.default._schema).endswith("(Tensor x) -> (Tensor, Tensor)")
    assert str(ops.fp8_blockwise_linear.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    lin = lambda M, K, N, x=None, s=None, p=None: lib.ao_fp8_blockwise_linear(
        ctypes.c_void_p(x), ctypes.c_void_p(s), M, K, ctypes.c_void_p(p), ctypes.c_void_p(p), N, None, ctypes.c_void_p(p),
        None, z, None)
    assert lin(4, 4160, 256) == -1 and b"K=4160 must be a multiple of 128" in lib.ao_b200_last_error()
    assert lin(4, 4096, 200) == -1 and b"N=200 must be a multiple of 128" in lib.ao_b200_last_error()
    assert lin(4, 0, 256) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    assert lin(4, 4096, 256) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert lin(0, 4096, 256) == 0   # M == 0: nothing to do, no CUDA call (this process has no device)
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15
    assert lin(4, 4096, 256, x=a + 8, s=a, p=a) == -1 and b"xq must be 16-byte aligned" in lib.ao_b200_last_error()
    assert lin(4, 4096, 256, x=a, s=a + 4, p=a) == -1 and b"x_scale must be 16-byte aligned" in lib.ao_b200_last_error()
    quant = lambda ldx, M, K, x=None, p=None: lib.ao_fp8_quantize_1x128_ld(
        ctypes.c_void_p(x), ldx, M, K, ctypes.c_void_p(p), ctypes.c_void_p(p), None)
    assert quant(192, 4, 192) == -1 and b"K%128==0" in lib.ao_b200_last_error()
    assert quant(4096, 4, 4096) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert quant(4100, 4, 4096, x=a, p=a) == -1 and b"multiple of 8" in lib.ao_b200_last_error()
    assert quant(4088, 4, 4096, x=a, p=a) == -1 and b"ldx" in lib.ao_b200_last_error()
    assert quant(4096, 4, 4096, x=a + 8, p=a) == -1 and b"16-byte aligned" in lib.ao_b200_last_error()
    assert quant(4096, 0, 4096) == 0
    assert lib.ao_fp8_quantize_1x128(None, 4, 100, None, None, None) == -1


# ---------------------------------------------------------------- the budget of the format
# Cfg<BlockwiseF8Fmt, N> is streamk_model.ring("fp8_blockwise", N): a stage is the 16 KiB weight tile, the 1 KiB aux
# slot (256 bytes of token scales) and N x 128 activation bytes; one CTA per SM (PROMOTE), a 200 KB ring
@pytest.mark.parametrize("n_mma", [16, 32, 64])
def test_tiles_registers_stack_and_shared_memory(n_mma):
    src = open(os.path.join(ROOT, "ao_b200", "csrc", "lowp_linear.cu")).read()
    body = src[src.index("struct BlockwiseF8Fmt"):]
    body = body[:body.index("\n};\n")]
    assert "X_AUX_BYTES = MAX_N_MMA * 4;" in body and "AUX_BYTES = X_AUX_BYTES;" in body
    usage = resource_usage()
    assert ("BlockwiseF8Fmt", n_mma) in usage, f"ts_gemm_kernel<BlockwiseF8Fmt, {n_mma}> not built"
    assert ("BlockwiseF8Fmt", 128) not in usage   # MAX_N_MMA = 64, as SsFmt<KIND_F8>
    reg, stack = usage[("BlockwiseF8Fmt", n_mma)]
    assert reg <= 168 and stack == 0, (reg, stack)
    stage, ctas, stages, staging = sk.ring("fp8_blockwise", n_mma)
    assert stage == 16384 + 1024 + n_mma * 128 and ctas == 1 and not staging
    smem = sk.ring_smem("fp8_blockwise", n_mma)
    assert stages >= 2 and smem + RESERVED_PER_CTA <= SMEM_PER_SM
