"""float8 weight-only (Float8WeightOnlyConfig, Float8Tensor without act_quant_kwargs) without a GPU: a restatement of
the weight quantization and of the recipe against the reference's fixture, the package's quantizer on the fixture's
weights, the config's rules and JSON round trip, the PerGroup / e5m2 / version rejections and the skip rule, Meta shapes
and the op schema, C-ABI rejections, the tensor plumbing of a weight-only instance, and the register and shared-memory
budget of the GEMM's format policy."""
import ctypes
import json
import logging
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import streamk_model as sk
from test_decode_residency import SMEM_PER_SM, RESERVED_PER_CTA, resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ---------------------------------------------------------------- the restatement (shared with the GPU tests)
def bf16_round(a):
    """float32 array -> the nearest bf16 (ties to even), as float32."""
    from oracle import oracle as o

    return o.bf16_to_f32(o.f32_to_bf16(np.asarray(a, np.float32)))


def f32(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32)


def e4m3_values():
    """float32 value of every e4m3fn byte 0x00..0xFF (0x7F and 0xFF are NaN)."""
    from oracle import oracle as o

    return o.e4m3_to_f32(np.arange(256, dtype=np.uint8))


def to_e4m3(v):
    """float32 array with |v| <= 448 or NaN -> e4m3fn bytes, round to nearest, ties to the even code; the sign bit is
    kept for zeros and NaNs (a NaN gives 0x7F or 0xFF)."""
    v = np.asarray(v, np.float32)
    mag = e4m3_values()[:127]   # codes 0x00..0x7E, increasing
    a = np.abs(np.nan_to_num(v, nan=0.0))
    hi = np.clip(np.searchsorted(mag, a, side="left"), 0, 126)
    lo = np.maximum(hi - 1, 0)
    d_hi, d_lo = mag[hi] - a, a - mag[lo]
    code = np.where(d_lo < d_hi, lo, np.where(d_hi < d_lo, hi, np.where(hi % 2 == 0, hi, lo)))
    code = np.where(np.isnan(v), 0x7F, code).astype(np.uint8)
    return code | np.where(np.signbit(v), 0x80, 0).astype(np.uint8)


def quantize_ref(w, per_tensor):
    """The reference's torch path of Float8Tensor.from_hp on bf16 values held in float32 w [N, K]: scale = bf16(amax /
    448) over the row (or the tensor; the division is a bf16 operation, the result is stored as fp32, no lower bound),
    q = e4m3(clamp(w / scale, -448, 448)).  An all-zero row gets scale 0 and NaN codes.  Returns (q uint8, scale)."""
    w = np.asarray(w, np.float32)
    amax = np.abs(w).max() if per_tensor else np.abs(w).max(axis=1, keepdims=True)
    scale = bf16_round(amax / np.float32(448.0)).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = to_e4m3(np.clip(w / scale, -448.0, 448.0))
    return q, np.asarray(scale, np.float32).reshape(-1)


def dequantize_ref(q, scale):
    """w~ = bf16(fp32(e4m3(q)) * scale), the reference's dequantize: q uint8 [N, K], scale N or 1 fp32 values."""
    s = np.broadcast_to(np.asarray(scale, np.float32).reshape(-1), (q.shape[0],))
    with np.errstate(invalid="ignore", over="ignore"):
        return bf16_round(e4m3_values()[q] * s[:, None])


def weight_only_ref(x, q, scale, bias=None):
    """The recipe on float32 arrays holding bf16 values: x [M, K], e4m3 bytes q [N, K], fp32 scale, bf16 bias [N] or
    None.  torch.matmul(x, w~.t()) returns bf16(the fp32 sum), the bias add is a bf16 operation.  The sum is taken in
    fp64 and rounded to fp32: the fp32 sum itself wherever that one is exact."""
    wt = dequantize_ref(q, scale)
    with np.errstate(invalid="ignore", over="ignore"):
        acc = (x.astype(np.float64) @ wt.astype(np.float64).T).astype(np.float32)
        y = bf16_round(acc)
        return y if bias is None else bf16_round(y + bias[None, :])


def same_codes(a, b):
    """e4m3 bytes equal, a NaN code (0x7F, 0xFF) matching either: the sign of 0 / 0 is the platform's (the reference on
    the CPU gives 0xFF, the package's CUDA quantizer 0x7F); both decode to NaN."""
    a, b = np.asarray(a, np.uint8), np.asarray(b, np.uint8)
    nan_a, nan_b = (a & 0x7F) == 0x7F, (b & 0x7F) == 0x7F
    return a.shape == b.shape and bool((nan_a == nan_b).all() and (a[~nan_a] == b[~nan_a]).all())


def same_bits_or_both_nan(got_bits, ref_bits):
    nan_g = np.isnan(f32(got_bits))
    return bool((nan_g == np.isnan(f32(ref_bits))).all() and (got_bits[~nan_g] == ref_bits[~nan_g]).all())


def within_one_step_of_the_sum(got_bits, ref_bits, x, q, scale, bias=None):
    """Where the fp32 sums round, two correct implementations differ by their accumulation order: bf16(sum) may fall on
    either neighbour, one bf16 step (at most 2^-7 of the sum) apart, and the fp32 sums themselves by far less.  The
    bias add rounds again and can cancel most of the sum, so the outputs are compared in absolute terms:
    |y - y_ref| <= 2^-6 (sum_k |x w~| + |bias|), and nine outputs in ten are identical.  NaNs (the reference's zero
    rows) must be NaN on both sides."""
    g, r = f32(got_bits).astype(np.float64), f32(ref_bits).astype(np.float64)
    if not (np.isnan(g) == np.isnan(r)).all():
        return False
    ok = ~np.isnan(r)
    mag = np.abs(x.astype(np.float64)) @ np.abs(np.nan_to_num(dequantize_ref(q, scale).astype(np.float64))).T
    if bias is not None:
        mag = mag + np.abs(bias.astype(np.float64))[None, :]
    return bool((np.abs(g - r)[ok] <= 2.0**-6 * mag[ok]).all()) and float((got_bits == ref_bits)[ok].mean()) >= 0.9


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "float8_weight_only.npz"))


def golden_cases(d):
    for i, c in enumerate(json.loads(str(d["cases"]))):
        s, g = c["shape"], c["granularity"]
        yield i, c, dict(w=d[f"s{s}_w"], b=d[f"s{s}_b"] if c["bias"] else None, x=d[f"s{s}_x"], xe=d[f"s{s}_xe"],
                         q=d[f"s{s}_{g}_q"], scale=d[f"s{s}_{g}_scale"], y=d[f"c{i}_y"], ye=d[f"c{i}_ye"])


def test_restatement_reproduces_the_reference(golden):
    from oracle import oracle as o

    seen = set()
    for i, c, a in golden_cases(golden):
        per_tensor = c["granularity"] == "PerTensor"
        q, s = quantize_ref(f32(a["w"]), per_tensor)
        assert same_codes(q, a["q"]) and np.array_equal(s, a["scale"].reshape(-1)), c
        assert a["scale"].shape == ((1, 1) if per_tensor else (c["N"], 1))
        assert c["block_size"] == ([c["N"], c["K"]] if per_tensor else [1, c["K"]])
        if not per_tensor:   # the zero row: scale 0, NaN codes, as the oracle's per-token rule gives them
            assert a["scale"][1, 0] == 0.0 and (a["q"][1] & 0x7F == 0x7F).all()
            qo, so = o.fp8_quantize_rowwise(a["w"])
            assert same_codes(qo, a["q"]) and np.array_equal(so, a["scale"].reshape(-1))
        bias = None if a["b"] is None else f32(a["b"])
        # one-hot inputs: every output is one exact product, determined bit for bit
        ye = o.f32_to_bf16(weight_only_ref(f32(a["xe"]), a["q"], a["scale"], bias))
        assert same_bits_or_both_nan(ye, a["ye"]), c
        assert np.isnan(f32(a["ye"])[:, 1]).all() != per_tensor   # the zero row's NaN reaches every token
        # random inputs: the reference's fp32 sums round in its own order
        got = o.f32_to_bf16(weight_only_ref(f32(a["x"]), a["q"], a["scale"], bias))
        assert within_one_step_of_the_sum(got, a["y"], f32(a["x"]), a["q"], a["scale"], bias), c
        seen.add((c["K"] % 128 != 0, c["N"] % 128 != 0, per_tensor, c["bias"]))
    assert len(seen) >= 8


def test_encoder_round_trips_every_code():
    v = e4m3_values()
    codes = np.arange(256, dtype=np.uint8)
    assert same_codes(to_e4m3(v), codes)
    nan = np.float32(np.nan)
    assert to_e4m3(np.array([nan, -nan]))[0] == 0x7F and to_e4m3(np.array([nan, -nan]))[1] == 0xFF   # NaN keeps its sign
    mid = (v[1:126] + v[2:127]) / 2   # every tie between neighbours 0x01..0x7E goes to the even code
    assert np.array_equal(to_e4m3(mid), np.where(np.arange(1, 126) % 2 == 0, np.arange(1, 126), np.arange(2, 127)))


def test_package_quantizer_matches_the_fixture(golden):
    from ao_b200.quantization import Float8Tensor, PerRow, PerTensor

    for i, c, a in golden_cases(golden):
        w = torch.from_numpy(a["w"].view(np.int16).copy()).view(torch.bfloat16)
        t = Float8Tensor.from_hp(w, torch.float8_e4m3fn, PerTensor() if c["granularity"] == "PerTensor" else PerRow())
        assert t.act_quant_kwargs is None and list(t.block_size) == c["block_size"]
        assert same_codes(t.qdata.view(torch.uint8).numpy(), a["q"]) and np.array_equal(t.scale.numpy(), a["scale"])


# ---------------------------------------------------------------- config
def test_config_defaults_rules_and_json_round_trip():
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.quantization import Float8WeightOnlyConfig, PerGroup, PerRow, PerTensor, PerToken

    c = Float8WeightOnlyConfig()
    assert (c.weight_dtype, c.set_inductor_config, c.version, c.granularity) == (torch.float8_e4m3fn, True, 2, PerRow())
    with pytest.raises(AssertionError, match="granularity must be"):
        Float8WeightOnlyConfig(granularity=PerToken())
    for gran in (PerRow(), PerTensor(), PerGroup(64)):
        for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
            c = Float8WeightOnlyConfig(weight_dtype=dt, granularity=gran, set_inductor_config=False)
            d = config_to_dict(c)
            assert d["_type"] == "Float8WeightOnlyConfig" and d["_version"] == 2
            assert d["_data"]["granularity"]["_type"] == type(gran).__name__
            assert config_from_dict(json.loads(json.dumps(d))) == c


def test_rejections_and_incompatible_k_skipped(caplog):
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, PerGroup, PerTensor, quantize_

    lin = nn.Linear(64, 32).to(torch.bfloat16)
    with pytest.raises(NotImplementedError, match="PerGroup"):
        quantize_(lin, Float8WeightOnlyConfig(granularity=PerGroup(32)))
    with pytest.raises(NotImplementedError, match="float8_e5m2"):
        quantize_(lin, Float8WeightOnlyConfig(weight_dtype=torch.float8_e5m2))
    with pytest.raises(AssertionError, match="Unexpected version"):
        quantize_(lin, Float8WeightOnlyConfig(version=1))
    assert type(lin.weight.data) is torch.Tensor
    odd = nn.Linear(40, 32).to(torch.bfloat16)   # K % 16 != 0
    with caplog.at_level(logging.INFO):
        quantize_(odd, Float8WeightOnlyConfig())
    assert "Skipping float8 weight only quantization" in caplog.text and "(32, 40)" in caplog.text
    assert not isinstance(odd.weight, Float8Tensor)
    quantize_(lin, Float8WeightOnlyConfig(granularity=PerTensor()))
    w = lin.weight
    assert isinstance(w, Float8Tensor) and w.act_quant_kwargs is None and w.scale.shape == (1, 1)
    assert w.qdata.dtype == torch.float8_e4m3fn and "Float8Tensor" in repr(lin)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_weights_that_are_not_bf16(caplog, dtype):
    """The reference dequantizes into the weight's own dtype and multiplies in it; the kernel computes in bf16.  The
    handler leaves such a layer unquantized, and a Float8Tensor of such a weight (a checkpoint of an fp16 / fp32 model)
    has no linear here."""
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, PerRow, quantize_

    lin = nn.Linear(64, 32).to(dtype)
    with caplog.at_level(logging.INFO):
        quantize_(lin, Float8WeightOnlyConfig())
    assert "Skipping float8 weight only quantization" in caplog.text and str(dtype) in caplog.text
    assert type(lin.weight.data) is torch.Tensor and lin.weight.dtype == dtype
    w = Float8Tensor.from_hp(torch.randn(32, 64).to(dtype), torch.float8_e4m3fn, PerRow())
    assert w.dtype == dtype and w.act_quant_kwargs is None
    for xd in (dtype, torch.bfloat16):
        with pytest.raises(NotImplementedError, match=f"quantized from {dtype}"):
            torch.nn.functional.linear(torch.zeros(2, 64, dtype=xd), w)


def test_torch_load_of_a_dynamic_activation_instance(tmp_path):
    """torch.load restores a Float8Tensor with act_quant_kwargs as well (its dtype is the wrapper's own attribute, not
    instance state)."""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8Tensor, PerRow, quantize_

    lin = nn.Linear(128, 64).to(torch.bfloat16)
    quantize_(lin, Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()))
    torch.save(lin.state_dict(), tmp_path / "w.pt")
    back = torch.load(tmp_path / "w.pt", weights_only=True)["weight"]
    w = lin.weight
    assert type(back) is Float8Tensor and back.dtype == torch.bfloat16 and back.act_quant_kwargs == w.act_quant_kwargs
    assert torch.equal(back.qdata.view(torch.uint8), w.qdata.view(torch.uint8)) and torch.equal(back.scale, w.scale)
    assert list(back.block_size) == list(w.block_size) and back.mm_config == w.mm_config


def test_fqn_to_config_reaches_the_named_module():
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, FqnToConfig, quantize_

    m = nn.Sequential(nn.Linear(32, 32), nn.Linear(32, 16)).to(torch.bfloat16)
    quantize_(m, FqnToConfig({"1": Float8WeightOnlyConfig()}), filter_fn=None)
    assert type(m[0].weight.data) is torch.Tensor
    assert isinstance(m[1].weight, Float8Tensor) and m[1].weight.act_quant_kwargs is None


def test_linear_without_a_kernel_raises():
    """CPU tensors reach the CUDA-only op and fail in the dispatcher; weights the kernel does not serve (group scales,
    3-D) fail before it."""
    from ao_b200.quantization import Float8Tensor, PerGroup, PerRow, PerTensor

    x = torch.zeros(2, 64, dtype=torch.bfloat16)
    for gran in (PerRow(), PerTensor()):
        w = Float8Tensor.from_hp(torch.randn(32, 64).to(torch.bfloat16), torch.float8_e4m3fn, gran)
        with pytest.raises(NotImplementedError):
            torch.nn.functional.linear(x, w)
    w = Float8Tensor.from_hp(torch.randn(32, 64).to(torch.bfloat16), torch.float8_e4m3fn, PerGroup(32))
    with pytest.raises(NotImplementedError, match="no sm_90a kernel"):
        torch.nn.functional.linear(x, w)
    w3 = Float8Tensor.from_hp(torch.randn(2, 32, 64).to(torch.bfloat16), torch.float8_e4m3fn, PerRow())
    with pytest.raises(NotImplementedError, match="no sm_90a kernel"):
        torch.nn.functional.linear(x, w3)


# ---------------------------------------------------------------- op surface
def test_meta_shapes_and_schema():
    import ao_b200  # noqa: F401

    x = torch.empty(130, 256, dtype=torch.bfloat16, device="meta")
    wq = torch.empty(200, 256, dtype=torch.float8_e4m3fn, device="meta")
    y = torch.ops.ao_b200.fp8_weight_linear(x, wq, torch.empty(200, device="meta"), None)
    assert y.shape == (130, 200) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(torch.ops.ao_b200.fp8_weight_linear.default._schema).endswith(
        "(Tensor x, Tensor wq, Tensor w_scale, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    call = lambda ldx, M, K, N, x=None, s=None, p=None: lib.ao_fp8_weight_linear(
        ctypes.c_void_p(x), ldx, M, K, ctypes.c_void_p(p), ctypes.c_void_p(s), N, None, ctypes.c_void_p(p), None, z, None)
    assert call(4104, 4, 4104, 128) == -1 and b"multiple of 16" in lib.ao_b200_last_error()
    assert call(4096, 4, 0, 128) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    assert call(4100, 4, 4096, 128) == -1 and b"multiple of 8" in lib.ao_b200_last_error()   # misaligned row pitch
    assert call(4088, 4, 4096, 128) == -1 and b"ldx" in lib.ao_b200_last_error()            # pitch below K
    assert call(4096, 4, 4096, 130) == -1 and b"null pointer" in lib.ao_b200_last_error()   # any N is a valid size
    assert call(4096, 0, 4096, 128) == 0   # M == 0: nothing to do, no CUDA call (this process has no device)
    # host addresses stand in for device ones: both alignment checks come before any CUDA call
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15
    assert call(4096, 4, 4096, 128, x=a + 8, s=a, p=a) == -1 and b"x must be 16-byte aligned" in lib.ao_b200_last_error()
    assert call(4096, 4, 4096, 128, x=a, s=a + 4, p=a) == -1 and b"w_scale must be 16-byte aligned" in lib.ao_b200_last_error()


# ---------------------------------------------------------------- tensor plumbing of the weight-only instance
def _weight(n=64, k=128, gran=None, seed=0):
    from ao_b200.quantization import Float8Tensor, PerRow

    g = torch.Generator().manual_seed(seed)
    return Float8Tensor.from_hp((torch.randn(n, k, generator=g) * 0.1).to(torch.bfloat16), torch.float8_e4m3fn,
                                gran or PerRow())


def _same(a, b):
    return (type(a) is type(b) and torch.equal(a.qdata.view(torch.uint8), b.qdata.view(torch.uint8))
            and torch.equal(a.scale, b.scale) and list(a.block_size) == list(b.block_size)
            and a.act_quant_kwargs is None and b.act_quant_kwargs is None and a.dtype == b.dtype)


def test_slice_and_copy():
    from ao_b200.quantization import PerTensor

    w = _weight()
    full = w.dequantize()
    rows = w.narrow(0, 16, 32)
    assert rows.act_quant_kwargs is None and tuple(rows.shape) == (32, 128) and rows.scale.shape == (32, 1)
    assert torch.equal(rows.dequantize(), full[16:48])
    cols = w[:, 32:96]
    assert tuple(cols.shape) == (64, 64) and list(cols.block_size) == [1, 64] and torch.equal(cols.dequantize(), full[:, 32:96])
    pt = _weight(gran=PerTensor())
    assert pt[8:24].scale.shape == (1, 1) and torch.equal(pt[8:24].dequantize(), pt.dequantize()[8:24])
    # a loader's narrow + copy_ writes through into the parameter
    dst, src = _weight(seed=1), _weight(seed=2)
    for lo in (0, 32):
        dst.narrow(0, lo, 32).copy_(src.narrow(0, lo, 32))
    assert _same(dst, src)


def test_torch_save_and_safetensors_round_trip(tmp_path):
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Float8WeightOnlyConfig, PerTensor, quantize_

    for gran in (None, PerTensor()):
        lin = nn.Linear(128, 64).to(torch.bfloat16)
        quantize_(lin, Float8WeightOnlyConfig(granularity=gran))
        torch.save(lin.state_dict(), tmp_path / "w.pt")
        back = torch.load(tmp_path / "w.pt", weights_only=True)["weight"]
        assert _same(back, lin.weight)
        flat, meta = flatten_tensor_state_dict({"m.weight": lin.weight.data})
        assert json.loads(meta["m.weight"])["_data"]["act_quant_kwargs"] is None
        assert all(type(v) is torch.Tensor for v in flat.values())
        sd, leftover = unflatten_tensor_state_dict(flat, meta)
        assert leftover == {} and _same(sd["m.weight"], lin.weight)


def test_cat_out_features_serves_the_weight_only_instance():
    """fuse_parallel_linears needs nothing new: the weight-only members agree in every attribute (act_quant_kwargs is
    None in each), so their qdata and per-row scales concatenate; per-tensor scales differ per member and do not."""
    from ao_b200.fusion import cat_out_features
    from ao_b200.quantization import PerTensor

    ws = [_weight(n, seed=i) for i, n in enumerate((64, 16, 16))]
    cat = cat_out_features(ws)
    assert cat is not None and cat.act_quant_kwargs is None and tuple(cat.shape) == (96, 128)
    assert torch.equal(cat.dequantize(), torch.cat([w.dequantize() for w in ws], 0))
    assert _same(cat[64:80], ws[1])
    assert cat_out_features([_weight(gran=PerTensor(), seed=3), _weight(gran=PerTensor(), seed=4)]) is None


# ---------------------------------------------------------------- the budget the format policy declares
def _policy():
    src = open(os.path.join(ROOT, "ao_b200", "csrc", "lowp_linear.cu")).read()
    body = src[src.index("struct Fp8WoFmt"):]
    return body[:body.index("struct Raw")]


@pytest.mark.parametrize("n_mma", [16, 32, 64, 128])
def test_tiles_registers_stack_and_shared_memory(n_mma):
    """ts_gemm_kernel<Fp8WoFmt, N> against the residency Fp8WoFmt declares (DECODE_2CTA): with two CTAs per SM the 16-
    and 32-token tiles would need at most 80 registers and a ring that fits twice into the SM; with one, every tile at
    most 168 registers and a 200 KB ring; never any stack."""
    body = _policy()
    assert "W_BYTES = ROWS * KCHUNK;" in body and "AUX_BYTES = ROWS * 4;" in body and "X_ELEM_BYTES = 2;" in body
    two = "static constexpr bool DECODE_2CTA = true;" in body and n_mma <= 32
    usage = resource_usage()
    assert ("Fp8WoFmt", n_mma) in usage, f"ts_gemm_kernel<Fp8WoFmt, {n_mma}> not built"
    reg, stack = usage[("Fp8WoFmt", n_mma)]
    assert reg <= (80 if two else 168), (reg, two)
    assert stack == 0, f"ts_gemm_kernel<Fp8WoFmt, {n_mma}>: {stack} bytes of stack"
    _, ctas, stages, _ = sk.ring("fp8wo", n_mma)
    smem = sk.ring_smem("fp8wo", n_mma)
    assert ctas == (2 if two else 1)
    assert stages >= 2
    assert (2 if two else 1) * (smem + RESERVED_PER_CTA) <= SMEM_PER_SM
