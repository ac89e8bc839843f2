"""mxfp4 (MXTensor with float4_e2m1fn_x2 elements) without a GPU: the torch restatement of the quantizer against the
reference's fixture, Meta shapes and op schemas, C-ABI rejections, config validation, tensor metadata, the safetensors
wire form, and the register budget of the GEMM's decode tiles."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from test_block_quantizers_gpu import e2m1_codes, e8m0_rceil, e8m0_reciprocal, pack_e2m1, to_blocked
from test_decode_residency import resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FP4 = torch.float4_e2m1fn_x2
E2M1 = [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, -0.0, -0.5, -1.0, -1.5, -2.0, -3.0, -4.0, -6.0]


# ---------------------------------------------------------------- the restatement (shared with test_mxfp4_gpu.py)
def mxfp4_ref(x):
    """to_mx(x, float4_e2m1fn_x2, 32, RCEIL) on bf16 x [M, K], with torch ops as the reference writes them (max_abs *
    (1 / 6), so a multiply by the fp32 reciprocal on either device): (packed codes [M, K/2], e8m0 bytes [M, K/32]).
    The codes of a NaN block (scale byte 0xFF) are not restated."""
    M, K = x.shape
    blocks = x.reshape(M, K // 32, 32)
    max_abs = torch.amax(torch.abs(blocks), -1, keepdim=True).to(torch.float32)
    e8 = e8m0_rceil(max_abs * (1.0 / 6.0))
    scaled = torch.clamp(blocks.to(torch.float32) * e8m0_reciprocal(e8), -6.0, 6.0)
    return pack_e2m1(e2m1_codes(scaled.reshape(M, K))), e8.reshape(M, K // 32)


def mxfp4_dequant(q, s):
    """codes [M, K/2] x e8m0 bytes [M, K/32] -> float32 [M, K], as MXTensor.dequantize computes it (NaN for 0xFF)."""
    lut = torch.tensor(E2M1, dtype=torch.float32, device=q.device)
    v = lut[torch.stack([q & 15, q >> 4], dim=-1).reshape(q.shape[0], -1).long()]
    e = torch.pow(2.0, s.to(torch.float32) - 127.0)
    e = torch.where(s == 255, torch.full_like(e, float("nan")), e)
    return v * e.repeat_interleave(32, dim=1)


def bf16(a):
    return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "mxfp4.npz"))


def test_restatement_reproduces_the_reference(golden):
    x = bf16(golden["x"])
    q, s = mxfp4_ref(x)
    assert np.array_equal(q.numpy(), golden["q"]) and np.array_equal(s.numpy(), golden["scale"])
    assert np.array_equal(to_blocked(s).numpy(), golden["scale_blocked"].reshape(-1))
    assert np.array_equal(np.array(E2M1, dtype=np.float32), golden["e2m1_table"])
    assert torch.equal(mxfp4_dequant(q, s), torch.from_numpy(golden["dequant_f32"]))
    # the fixture has the cases it claims: a zero block, 1e-3 .. 1e3 rows, an outlier
    assert (s[3, 1] == 0).item() and s.min().item() < 110 and s.max().item() > 130


def test_mxtensor_dequantize_matches_the_reference(golden):
    from ao_b200.prototype.mx_formats import MXTensor

    q = torch.from_numpy(golden["q"].copy())
    s = torch.from_numpy(golden["scale"].copy()).view(torch.float8_e8m0fnu)
    t = MXTensor(q, s, FP4, 32, torch.bfloat16, None, None, False)
    assert tuple(t.shape) == (130, 256) and t.dtype == torch.bfloat16
    assert np.array_equal(t.dequantize().view(torch.int16).numpy().view(np.uint16), golden["dequant"])
    sb = torch.from_numpy(golden["scale_blocked"].copy()).view(torch.float8_e8m0fnu)
    tb = MXTensor(q, sb, FP4, 32, torch.bfloat16, None, None, True)
    assert torch.equal(tb.dequantize(torch.float32), torch.from_numpy(golden["dequant_f32"]))


def test_every_finite_code_and_byte_is_exact_in_bf16():
    """2034 finite (code, byte) products: each is a bf16 value (the exactness the GEMM relies on); the overflowing
    ones are exactly |code| >= 4 at byte 253 and |code| >= 2 at byte 254."""
    codes = torch.tensor(E2M1[:8], dtype=torch.float64)   # the magnitudes; the sign bit only negates
    e = torch.arange(255, dtype=torch.float64)
    p = codes[:, None] * torch.pow(2.0, e - 127.0)[None, :]
    f32 = p.to(torch.float32)
    finite = torch.isfinite(f32)
    assert int(finite.sum()) == 2034
    assert torch.equal(f32[finite].to(torch.bfloat16).to(torch.float64), p[finite])
    assert torch.equal(f32[finite].to(torch.float64), p[finite])
    over = sorted((E2M1[int(c)], int(b)) for c, b in zip(*torch.nonzero(~finite, as_tuple=True)))
    assert over == [(2.0, 254), (3.0, 254), (4.0, 253), (4.0, 254), (6.0, 253), (6.0, 254)]


def test_meta_shapes_and_schemas():
    import ao_b200  # noqa: F401

    x = torch.empty(130, 256, dtype=torch.bfloat16, device="meta")
    q, s = torch.ops.ao_b200.mxfp4_quantize(x, False)
    assert q.shape == (130, 128) and q.dtype == torch.uint8 and s.shape == (130, 8) and s.dtype == torch.uint8
    q, s = torch.ops.ao_b200.mxfp4_quantize(x, True)
    assert s.shape == (64, 32)
    w = torch.empty(200, 128, dtype=torch.uint8, device="meta")
    y = torch.ops.ao_b200.mxfp4_linear(q, s, w, torch.empty(512, dtype=torch.uint8, device="meta"), None)
    assert y.shape == (130, 200) and y.dtype == torch.bfloat16
    assert str(torch.ops.ao_b200.mxfp4_quantize.default._schema).endswith("(Tensor x, bool swizzled) -> (Tensor, Tensor)")
    assert str(torch.ops.ao_b200.mxfp4_linear.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    rc = lib.ao_mxfp4_linear(None, None, 4, 4112, None, None, 128, None, None, None, z, None)
    assert rc == -1 and b"multiple of 32" in lib.ao_b200_last_error()
    rc = lib.ao_mxfp4_linear(None, None, 4, 4096, None, None, 128, None, None, None, z, None)
    assert rc == -1 and b"null pointer" in lib.ao_b200_last_error()
    rc = lib.ao_mxfp4_quantize(None, 4, 48, None, None, 1, None)
    assert rc == -1 and b"multiple of 32" in lib.ao_b200_last_error()
    rc = lib.ao_mxfp4_quantize(None, 4, 64, None, None, 1, None)
    assert rc == -1 and b"null pointer" in lib.ao_b200_last_error()
    # M == 0: nothing to do, no CUDA call (this process has no device)
    assert lib.ao_mxfp4_linear(None, None, 0, 4096, None, None, 128, None, None, None, z, None) == 0
    assert lib.ao_mxfp4_quantize(None, 0, 64, None, None, 1, None) == 0
    assert lib.ao_mxfp4_quantize_ld(None, 64, 0, 64, None, None, 0, None) == 0


def test_config_validation():
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.prototype.mx_formats.mx_tensor import ScaleCalculationMode

    c = MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4)
    assert c.weight_dtype == FP4
    with pytest.raises(AssertionError):
        MXDynamicActivationMXWeightConfig(activation_dtype=torch.float8_e4m3fn, weight_dtype=FP4)
    for bad in (dict(block_size=16), dict(scaling_mode=ScaleCalculationMode.FLOOR),
                dict(activation_dtype=torch.float8_e5m2, weight_dtype=torch.float8_e5m2)):
        kw = dict(activation_dtype=FP4, weight_dtype=FP4)
        kw.update(bad)
        with pytest.raises(NotImplementedError, match="implemented"):
            MXDynamicActivationMXWeightConfig(**kw)


def test_to_mx_rejects_other_elements_and_modes():
    from ao_b200.prototype.mx_formats import MXTensor
    from ao_b200.prototype.mx_formats.mx_tensor import ScaleCalculationMode

    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="float4_e2m1fn_x2"):
        MXTensor.to_mx(x, torch.float8_e5m2)
    with pytest.raises(NotImplementedError):
        MXTensor.to_mx(x, FP4, 16)
    with pytest.raises(NotImplementedError):
        MXTensor.to_mx(x, FP4, 32, ScaleCalculationMode.FLOOR)


def test_fp4_metadata_slicing_and_save(tmp_path):
    from ao_b200.prototype.mx_formats import MXTensor

    q = torch.randint(0, 256, (256, 64), dtype=torch.uint8)
    s = torch.randint(100, 140, (256 * 4,), dtype=torch.uint8).view(torch.float8_e8m0fnu)   # blocked, 2 x 1 tiles
    t = MXTensor(q, s.reshape(64, 16), FP4, 32, torch.bfloat16, None, None, True)
    assert tuple(t.shape) == (256, 128) and t.dtype == torch.bfloat16 and t.qdata.dtype == torch.uint8
    full = t.dequantize(torch.float32)
    rows = t[128:256]
    assert tuple(rows.shape) == (128, 128) and torch.equal(rows.dequantize(torch.float32), full[128:])
    p = MXTensor(q, torch.randint(100, 140, (256, 4), dtype=torch.uint8).view(torch.float8_e8m0fnu), FP4, 32,
                 torch.bfloat16, None, None, False)
    cols = p.narrow(1, 32, 64)
    assert tuple(cols.shape) == (256, 64) and torch.equal(cols.dequantize(torch.float32), p.dequantize(torch.float32)[:, 32:96])
    with pytest.raises(RuntimeError, match="even"):
        p.narrow(1, 1, 64)
    torch.save({"w": t}, tmp_path / "w.pt")
    back = torch.load(tmp_path / "w.pt", weights_only=True)["w"]
    assert type(back) is MXTensor and back.elem_dtype == FP4 and tuple(back.shape) == (256, 128)
    assert torch.equal(back.qdata, q) and torch.equal(back.dequantize(torch.float32), full)


def test_safetensors_wire_fixture_loads_into_an_equal_tensor(golden):
    import ao_b200  # noqa: F401
    from ao_b200.prototype.mx_formats import MXTensor
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict

    meta = json.loads(str(golden["wire_meta"]))
    keys = json.loads(str(golden["wire_keys"]))
    dtypes = {"qdata": (torch.uint8, (64, 64)), "scale": (torch.float8_e8m0fnu, (64, 4))}
    flat = {}
    for i, k in enumerate(keys):
        dt, shape = dtypes[k.rsplit("_", 1)[-1]]
        flat[k] = torch.from_numpy(golden[f"wire_{i}"].copy()).view(dt).reshape(shape)
    sd, leftover = unflatten_tensor_state_dict(flat, meta)
    assert leftover == {}
    w = sd["m.weight"]
    assert type(w) is MXTensor and w.elem_dtype is FP4 and tuple(w.shape) == (64, 128)
    assert np.array_equal(w.dequantize(torch.bfloat16).view(torch.int16).numpy().view(np.uint16), golden["wire_dequant"])
    flat2, meta2 = flatten_tensor_state_dict(sd)
    assert sorted(flat2) == keys and all(torch.equal(flat2[k].view(torch.uint8), flat[k].view(torch.uint8)) for k in keys)
    assert {k: json.loads(v) for k, v in meta2.items()} == {k: json.loads(v) for k, v in meta.items()}
    assert json.loads(meta2["m.weight"])["_data"]["elem_dtype"] == {"_type": "torch.dtype", "_data": "float4_e2m1fn_x2"}


@pytest.mark.parametrize("n_mma", [16, 32])
def test_decode_tiles_registers_and_stack(n_mma):
    """ts_gemm_kernel<Mxfp4Fmt, 16 | 32> against the residency Mxfp4Fmt declares: with DECODE_2CTA, at most 80
    registers (two 384-thread CTAs per SM); without, at most 168 (one CTA); never any stack."""
    src = open(os.path.join(ROOT, "ao_b200", "csrc", "lowp_linear.cu")).read()
    body = src[src.index("struct Mxfp4Fmt"):]
    two = "static constexpr bool DECODE_2CTA = true;" in body[:body.index("};")]
    usage = resource_usage()
    assert ("Mxfp4Fmt", n_mma) in usage, f"ts_gemm_kernel<Mxfp4Fmt, {n_mma}> not built"
    reg, stack = usage[("Mxfp4Fmt", n_mma)]
    assert reg <= (80 if two else 168), (reg, two)
    assert stack == 0, f"ts_gemm_kernel<Mxfp4Fmt, {n_mma}>: {stack} bytes of stack"
