"""int8 weight-only (Int8WeightOnlyConfig, Int8Tensor without act_quant_kwargs) without a GPU: the restatement of the
recipe against the reference's fixture, the config's rules and JSON round trip, Meta shapes and the op schema, C-ABI
rejections, the tensor plumbing of a weight-only instance, the PerGroup rejection and the skip rule, and the register
and shared-memory budget of the GEMM's format policy."""
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
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ---------------------------------------------------------------- the restatement (shared with the GPU tests)
def bf16_round(a):
    """float32 array -> the nearest bf16 (ties to even), as float32."""
    from oracle import oracle as o

    return o.bf16_to_f32(o.f32_to_bf16(np.asarray(a, np.float32)))


def weight_only_ref(x, q, scale, bias=None):
    """The weight-only recipe on float32 arrays holding bf16 values: x [M, K], int8 q [N, K], fp32 scale (N or 1
    values), bf16 bias [N] or None.  torch.mm of bf16 operands returns bf16(the fp32 sum), the scale is cast to bf16,
    the multiply and the bias add are bf16 operations (an fp32 operation rounded to bf16).  The sum is taken in fp64
    and rounded to fp32: the fp32 sum itself wherever that one is exact."""
    acc = (x.astype(np.float64) @ q.astype(np.float64).T).astype(np.float32)
    s = bf16_round(np.broadcast_to(np.asarray(scale, np.float32).reshape(-1), (q.shape[0],)))
    y = bf16_round(bf16_round(acc) * s[None, :])
    return y if bias is None else bf16_round(y + bias[None, :])


def quantize_ref(w, per_tensor):
    """Symmetric int8 weight quantization of bf16 values held in float32 w [N, K]: scale = max(bf16(amax / 127.5), fp32
    eps) over the row (or the tensor; the division is a bf16 operation, the result is stored as fp32),
    q = clamp(round(w * (1 / scale)), -128, 127).  Returns (q int8, scale fp32)."""
    w = np.asarray(w, np.float32)
    amax = np.abs(w).max() if per_tensor else np.abs(w).max(axis=1, keepdims=True)
    scale = np.maximum(bf16_round(amax / np.float32(127.5)), np.finfo(np.float32).eps).astype(np.float32)
    q = np.clip(np.rint(w * (np.float32(1.0) / scale)), -128, 127).astype(np.int8)
    return q, scale.reshape(-1)


def f32(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32)


def within_one_step_of_the_sum(got_bits, ref_bits, x, q, scale, bias=None):
    """Where the fp32 sums round, two correct implementations differ by their accumulation order: bf16(sum) may fall on
    either neighbour, one bf16 step (at most 2^-7 of the sum) apart.  The multiply carries that step through and rounds
    again, and the bias add can cancel most of the product, so the outputs are compared in absolute terms:
    |y - y_ref| <= 2^-6 (|sum * scale| + |bias|), and nine outputs in ten are identical."""
    mag = np.abs((x.astype(np.float64) @ q.astype(np.float64).T) * np.asarray(scale, np.float64).reshape(1, -1))
    if bias is not None:
        mag = mag + np.abs(bias.astype(np.float64))[None, :]
    diff = np.abs(f32(got_bits).astype(np.float64) - f32(ref_bits).astype(np.float64))
    return bool((diff <= 2.0**-6 * mag).all()) and float((got_bits == ref_bits).mean()) >= 0.9


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "int8_weight_only.npz"))


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
        assert np.array_equal(q, a["q"]) and np.array_equal(s, a["scale"].reshape(-1)), c
        assert a["scale"].shape == ((1, 1) if per_tensor else (c["N"], 1))
        assert c["block_size"] == ([c["N"], c["K"]] if per_tensor else [1, c["K"]])
        if not per_tensor:   # the per-row rule is the oracle's per-token one
            qo, so = o.int8_quantize_rowwise(a["w"])
            assert np.array_equal(qo, a["q"]) and np.array_equal(so, a["scale"].reshape(-1))
        bias = None if a["b"] is None else f32(a["b"])
        # exact operands: every fp32 sum is exact, so the output is determined bit for bit
        assert np.array_equal(o.f32_to_bf16(weight_only_ref(f32(a["xe"]), a["q"], a["scale"], bias)), a["ye"]), c
        # random operands: the reference's fp32 sums round in its own order
        got = o.f32_to_bf16(weight_only_ref(f32(a["x"]), a["q"], a["scale"], bias))
        assert within_one_step_of_the_sum(got, a["y"], f32(a["x"]), a["q"], a["scale"], bias), c
        seen.add((c["K"] % 128 != 0, c["N"] % 128 != 0, per_tensor, c["bias"]))
    assert len(seen) >= 8
    # a bf16 weight gives a bf16-representable scale, so the fixture cannot pin the recipe's cast of the scale to bf16;
    # scales with more bits reach the kernel through checkpoints of fp32 models and are covered on the GPU
    assert all(np.array_equal(bf16_round(a["scale"]), a["scale"]) for _, _, a in golden_cases(golden))


def test_package_quantizer_and_dequantize_match_the_fixture(golden):
    from ao_b200.quantization import Int8Tensor, PerRow, PerTensor

    for i, c, a in golden_cases(golden):
        w = torch.from_numpy(a["w"].view(np.int16).copy()).view(torch.bfloat16)
        t = Int8Tensor.from_hp(w, PerTensor() if c["granularity"] == "PerTensor" else PerRow())
        assert t.act_quant_kwargs is None and list(t.block_size) == c["block_size"]
        assert np.array_equal(t.qdata.numpy(), a["q"]) and np.array_equal(t.scale.numpy(), a["scale"])


# ---------------------------------------------------------------- config
def test_config_defaults_rules_and_json_round_trip():
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.quantization import Int8WeightOnlyConfig, PerGroup, PerRow, PerTensor, PerToken

    c = Int8WeightOnlyConfig()
    assert (c.group_size, c.granularity, c.set_inductor_config, c.version) == (None, PerRow(), True, 2)
    with pytest.raises(ValueError, match="version 1"):
        Int8WeightOnlyConfig(version=1)
    with pytest.raises(AssertionError, match="group_size=None"):
        Int8WeightOnlyConfig(group_size=32)
    with pytest.raises(AssertionError, match="granularity must be"):
        Int8WeightOnlyConfig(granularity=PerToken())
    for gran in (PerRow(), PerTensor(), PerGroup(64)):
        c = Int8WeightOnlyConfig(granularity=gran, set_inductor_config=False)
        d = config_to_dict(c)
        assert d["_type"] == "Int8WeightOnlyConfig" and d["_version"] == 2
        assert d["_data"]["granularity"]["_type"] == type(gran).__name__
        assert config_from_dict(json.loads(json.dumps(d))) == c


def test_per_group_rejected_and_incompatible_k_skipped(caplog):
    from ao_b200.quantization import Int8Tensor, Int8WeightOnlyConfig, PerGroup, PerTensor, quantize_

    lin = nn.Linear(64, 32).to(torch.bfloat16)
    with pytest.raises(NotImplementedError, match="PerGroup"):
        quantize_(lin, Int8WeightOnlyConfig(granularity=PerGroup(32)))
    assert type(lin.weight.data) is torch.Tensor
    odd = nn.Linear(40, 32).to(torch.bfloat16)   # K % 16 != 0
    with caplog.at_level(logging.INFO):
        quantize_(odd, Int8WeightOnlyConfig())
    assert "Skipping int8 weight only quantization" in caplog.text and "(32, 40)" in caplog.text
    assert not isinstance(odd.weight, Int8Tensor)
    quantize_(lin, Int8WeightOnlyConfig(granularity=PerTensor()))
    w = lin.weight
    assert isinstance(w, Int8Tensor) and w.act_quant_kwargs is None and w.scale.shape == (1, 1)
    assert "Int8Tensor" in repr(lin)


def test_fqn_to_config_reaches_the_named_module():
    from ao_b200.quantization import FqnToConfig, Int8Tensor, Int8WeightOnlyConfig, quantize_

    m = nn.Sequential(nn.Linear(32, 32), nn.Linear(32, 16)).to(torch.bfloat16)
    quantize_(m, FqnToConfig({"1": Int8WeightOnlyConfig()}), filter_fn=None)
    assert type(m[0].weight.data) is torch.Tensor
    assert isinstance(m[1].weight, Int8Tensor) and m[1].weight.act_quant_kwargs is None


def test_per_group_tensor_has_no_linear():
    from ao_b200.quantization import Int8Tensor, PerGroup

    w = Int8Tensor.from_hp(torch.randn(32, 64).to(torch.bfloat16), PerGroup(32))
    with pytest.raises(NotImplementedError, match="neither per-row nor per-tensor"):
        torch.nn.functional.linear(torch.zeros(2, 64, dtype=torch.bfloat16), w)


# ---------------------------------------------------------------- op surface
def test_meta_shapes_and_schema():
    import ao_b200  # noqa: F401

    x = torch.empty(130, 256, dtype=torch.bfloat16, device="meta")
    wq = torch.empty(200, 256, dtype=torch.int8, device="meta")
    y = torch.ops.ao_b200.int8_weight_linear(x, wq, torch.empty(200, device="meta"), None)
    assert y.shape == (130, 200) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(torch.ops.ao_b200.int8_weight_linear.default._schema).endswith(
        "(Tensor x, Tensor wq, Tensor w_scale, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    call = lambda ldx, M, K, N: lib.ao_int8_weight_linear(None, ldx, M, K, None, None, N, None, None, None, z, None)
    assert call(4104, 4, 4104, 128) == -1 and b"multiple of 16" in lib.ao_b200_last_error()
    assert call(4096, 4, 0, 128) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    assert call(4100, 4, 4096, 128) == -1 and b"multiple of 8" in lib.ao_b200_last_error()   # misaligned row pitch
    assert call(4088, 4, 4096, 128) == -1 and b"ldx" in lib.ao_b200_last_error()            # pitch below K
    assert call(4096, 4, 4096, 130) == -1 and b"null pointer" in lib.ao_b200_last_error()   # any N is a valid size
    assert call(4096, 0, 4096, 128) == 0   # M == 0: nothing to do, no CUDA call (this process has no device)


# ---------------------------------------------------------------- tensor plumbing of the weight-only instance
def _weight(n=64, k=128, gran=None, seed=0):
    from ao_b200.quantization import Int8Tensor, PerRow

    g = torch.Generator().manual_seed(seed)
    return Int8Tensor.from_hp((torch.randn(n, k, generator=g) * 0.1).to(torch.bfloat16), gran or PerRow())


def _same(a, b):
    return (type(a) is type(b) and torch.equal(a.qdata, b.qdata) and torch.equal(a.scale, b.scale)
            and list(a.block_size) == list(b.block_size) and a.act_quant_kwargs is None and b.act_quant_kwargs is None
            and a.dtype == b.dtype)


def test_slice_select_and_copy():
    from ao_b200.quantization import Int8Tensor, PerRow, PerTensor

    w = _weight()
    full = w.dequantize()
    rows = w.narrow(0, 16, 32)
    assert rows.act_quant_kwargs is None and tuple(rows.shape) == (32, 128) and rows.scale.shape == (32, 1)
    assert torch.equal(rows.dequantize(), full[16:48])
    cols = w[:, 32:96]
    assert tuple(cols.shape) == (64, 64) and list(cols.block_size) == [1, 64] and torch.equal(cols.dequantize(), full[:, 32:96])
    pt = _weight(gran=PerTensor())
    assert pt[8:24].scale.shape == (1, 1) and torch.equal(pt[8:24].dequantize(), pt.dequantize()[8:24])
    t3 = Int8Tensor.from_hp(torch.randn(3, 16, 32).to(torch.bfloat16), PerRow())
    assert t3.act_quant_kwargs is None and torch.equal(t3[1].dequantize(), t3.dequantize()[1])
    # a loader's narrow + copy_ writes through into the parameter
    dst, src = _weight(seed=1), _weight(seed=2)
    for lo in (0, 32):
        dst.narrow(0, lo, 32).copy_(src.narrow(0, lo, 32))
    assert _same(dst, src)


def test_torch_save_and_safetensors_round_trip(tmp_path):
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Int8WeightOnlyConfig, PerTensor, quantize_

    for gran in (None, PerTensor()):
        lin = nn.Linear(128, 64).to(torch.bfloat16)
        quantize_(lin, Int8WeightOnlyConfig() if gran is None else Int8WeightOnlyConfig(granularity=gran))
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
    body = src[src.index("struct Int8WoFmt"):]
    return body[:body.index("struct Raw")]


@pytest.mark.parametrize("n_mma", [16, 32, 64, 128])
def test_tiles_registers_stack_and_shared_memory(n_mma):
    """ts_gemm_kernel<Int8WoFmt, N> against the residency Int8WoFmt declares (DECODE_2CTA): the 16- and 32-token tiles
    at most 80 registers and a ring that fits twice into the SM, the wider ones at most 168 registers and a 200 KB
    ring; never any stack."""
    body = _policy()
    assert "W_BYTES = ROWS * KCHUNK;" in body and "AUX_BYTES = 0;" in body and "X_ELEM_BYTES = 2;" in body
    two = "static constexpr bool DECODE_2CTA = true;" in body and n_mma <= 32
    usage = resource_usage()
    assert ("Int8WoFmt", n_mma) in usage, f"ts_gemm_kernel<Int8WoFmt, {n_mma}> not built"
    reg, stack = usage[("Int8WoFmt", n_mma)]
    assert reg <= (80 if two else 168), (reg, two)
    assert stack == 0, f"ts_gemm_kernel<Int8WoFmt, {n_mma}>: {stack} bytes of stack"
    _, ctas, stages, _ = sk.ring("int8wo", n_mma)
    smem = sk.ring_smem("int8wo", n_mma)
    assert ctas == (2 if two else 1)
    assert stages >= 2 and (not two or stages == {16: 5, 32: 4}[n_mma])
    assert (2 if two else 1) * (smem + RESERVED_PER_CTA) <= SMEM_PER_SM
