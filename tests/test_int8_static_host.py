"""Static int8 activations (Int8StaticActivationInt8WeightConfig) without a GPU: the config's fields, defaults and rules,
the quantize handler (shape skip, missing scale, device move, FqnToConfig), the op's Meta shapes and the C ABI's
argument checks, the activation attributes through select / slice / torch.save / safetensors, and a numpy restatement
of the quantization contract against the reference's codes in tests/golden/int8_static.npz."""
import ctypes
import json
import logging
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def f32_of_bf16(b):
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16_rne(a):
    """fp32 -> the fp32 value of its bf16 rounding (round to nearest even; NaN kept)."""
    u = np.asarray(a, dtype=np.float32).view(np.uint32)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return np.where(np.isnan(a), np.float32(np.nan), r.view(np.float32))


def static_codes_ref(x_bits, scale, zp=None, pre=None, reduce_range=False):
    """The contract restated in numpy: q = int8(clamp(rne(x_f * (1 / s)) + zp, qmin, qmax)); x_f = x * pre in fp32,
    rounded to bf16 when pre is bf16 (given as uint16 bits); NaN -> 0."""
    x = f32_of_bf16(x_bits)
    if pre is not None:
        if pre.dtype == np.uint16:
            x = bf16_rne(x * f32_of_bf16(pre)[None, :])
        else:
            x = (x * pre.astype(np.float32)[None, :]).astype(np.float32)
    s = np.asarray(scale, dtype=np.float32).reshape(-1, 1)
    inv = (np.float32(1.0) / s).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        t = np.rint((x * inv).astype(np.float32))
        if zp is not None:
            t = t + np.asarray(zp, dtype=np.float32).reshape(-1, 1)
        qmin, qmax = (-64, 63) if reduce_range else (-128, 127)
        t = np.clip(t, qmin, qmax)
    return np.where(np.isnan(t), 0, t).astype(np.int8)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "int8_static.npz"))


def golden_cases(d):
    return json.loads(str(d["cases"]))


# ---------------------------------------------------------------- the contract against the reference's codes
def test_restatement_reproduces_the_reference_codes(golden):
    cases = golden_cases(golden)
    assert len(cases) == 72
    ties = clamped = 0
    for c, case in enumerate(cases):
        x = golden[f"s{case['shape']}_x"]
        zp = golden[f"c{c}_zp"] if f"c{c}_zp" in golden else None
        pre = golden[f"c{c}_pre"] if f"c{c}_pre" in golden else None
        got = static_codes_ref(x, golden[f"c{c}_scale"], zp, pre, case["reduce_range"])
        assert np.array_equal(got, golden[f"c{c}_q"]), case
        if case["pre"] == "none" and not case["reduce_range"] and case["mapping"] == "SYMMETRIC":
            v = f32_of_bf16(x) * (np.float32(1) / golden[f"c{c}_scale"].reshape(-1, 1).astype(np.float32))
            ties += int(np.sum(np.abs(v - np.trunc(v)) == 0.5))
            clamped += int(np.sum(np.abs(v) > 128))
    assert ties > 500 and clamped > 50   # the fixture exercises round-half-to-even and the clamp
    q = np.concatenate([golden[f"c{c}_q"].ravel() for c in range(len(cases))])
    assert {-128, -64, 63, 127} <= set(np.unique(q).tolist())


# ---------------------------------------------------------------- config
def test_config_fields_defaults_and_rules():
    import dataclasses

    from ao_b200.quantization import (Int8StaticActivationInt8WeightConfig, MappingType, PerGroup, PerRow, PerTensor,
                                      QuantizeTensorToInt8Kwargs)

    c = Int8StaticActivationInt8WeightConfig()
    assert [f.name for f in dataclasses.fields(c)] == [
        "act_quant_scale", "act_quant_zero_point", "granularity", "act_mapping_type", "set_inductor_config", "version",
        "reduce_range"]
    assert (c.act_quant_scale, c.act_quant_zero_point, c.granularity, c.act_mapping_type, c.set_inductor_config,
            c.version, c.reduce_range) == (None, None, PerRow(), MappingType.SYMMETRIC, True, 1, False)
    with pytest.raises(ValueError, match=r"PerRow\(dim=-1\)"):
        Int8StaticActivationInt8WeightConfig(granularity=PerRow(dim=0))
    with pytest.raises(ValueError):
        Int8StaticActivationInt8WeightConfig(granularity=PerGroup(32))
    with pytest.raises(ValueError):
        Int8StaticActivationInt8WeightConfig(granularity=[PerRow(), PerGroup(32)])
    with pytest.raises(AssertionError):
        Int8StaticActivationInt8WeightConfig(act_mapping_type=MappingType.SYMMETRIC_NO_CLIPPING_ERR)
    kw = Int8StaticActivationInt8WeightConfig(granularity=[PerTensor(), PerRow()], act_mapping_type=MappingType.ASYMMETRIC,
                                              reduce_range=True).get_act_quant_kwargs()
    assert kw == QuantizeTensorToInt8Kwargs(granularity=PerTensor(), mapping_type=MappingType.ASYMMETRIC, reduce_range=True)


# ---------------------------------------------------------------- handler
def _static(**kw):
    from ao_b200.quantization import Int8StaticActivationInt8WeightConfig

    return Int8StaticActivationInt8WeightConfig(**kw)


def test_handler_needs_a_scale_and_skips_unservable_shapes(caplog):
    from ao_b200.quantization import Int8Tensor, PerTensor, quantize_

    with pytest.raises(ValueError, match="act_quant_scale"):
        quantize_(nn.Linear(128, 64).to(torch.bfloat16), _static())
    s = torch.tensor([[0.05]])
    for k, n in ((120, 64), (128, 60)):
        lin = nn.Linear(k, n).to(torch.bfloat16)
        with caplog.at_level(logging.INFO, logger="ao_b200.quantization.quant_api"):
            quantize_(lin, _static(act_quant_scale=s, granularity=PerTensor()))
        assert type(lin.weight.data) is torch.Tensor
        assert "Skipping int8 static quantization" in caplog.text
    lin = nn.Linear(128, 64).to(torch.bfloat16)
    quantize_(lin, _static(act_quant_scale=s, granularity=[PerTensor(), PerTensor()]))
    w = lin.weight
    assert isinstance(w, Int8Tensor) and w.act_quant_scale is not None and torch.equal(w.act_quant_scale, s)
    assert w.act_quant_zero_point is None and w.act_pre_scale is None
    assert w.act_quant_kwargs.granularity == PerTensor() and w.scale.numel() == 1


def test_handler_moves_the_calibrated_tensors_to_the_weight_device():
    from ao_b200.quantization import MappingType, PerTensor
    from ao_b200.quantization.quant_api import _int8_static_activation_int8_weight_quantize_tensor

    w = torch.empty(64, 128, dtype=torch.bfloat16, device="meta")
    cfg = _static(act_quant_scale=torch.tensor([[0.05]]), act_quant_zero_point=torch.tensor([[3]], dtype=torch.int8),
                  granularity=PerTensor(), act_mapping_type=MappingType.ASYMMETRIC)
    q = _int8_static_activation_int8_weight_quantize_tensor(w, cfg)
    assert q.act_quant_scale.device.type == "meta" and q.act_quant_zero_point.device.type == "meta"
    assert cfg.act_quant_scale.device.type == "cpu"   # the config keeps its own tensors


def test_fqn_to_config_reaches_the_named_module_and_parameter():
    from ao_b200.quantization import FqnToConfig, Int8Tensor, PerTensor, quantize_

    s = torch.tensor([[0.02]])
    for key in ("a", "a.weight"):
        m = nn.Sequential()
        m.add_module("a", nn.Linear(128, 64).to(torch.bfloat16))
        m.add_module("b", nn.Linear(64, 32).to(torch.bfloat16))
        quantize_(m, FqnToConfig({key: _static(act_quant_scale=s, granularity=PerTensor())}), filter_fn=None)
        assert isinstance(m.a.weight, Int8Tensor) and torch.equal(m.a.weight.act_quant_scale, s), key
        assert type(m.b.weight.data) is torch.Tensor, key


# ---------------------------------------------------------------- op and C ABI
def test_meta_shapes_and_schema():
    import ao_b200  # noqa: F401

    op = torch.ops.ao_b200.int8_quantize_static
    x = torch.empty(130, 256, dtype=torch.bfloat16, device="meta")
    q, s, z = op(x, torch.empty(1, 1, device="meta"), None, torch.empty(256, device="meta"), -128, 127)
    assert (q.shape, q.dtype, s.shape, s.dtype, z.shape, z.dtype) == (
        (130, 256), torch.int8, (130,), torch.float32, (130,), torch.int8)
    assert all(t.device.type == "meta" for t in (q, s, z))
    assert str(op.default._schema).endswith(
        "(Tensor x, Tensor scale, Tensor? zero_point, Tensor? pre_scale, int qmin, int qmax) -> (Tensor, Tensor, Tensor)")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    dummy = ctypes.c_void_p(4096)   # never dereferenced: every call below fails its checks or returns before a launch

    def call(ldx=4096, M=4, K=4096, pre=None, pre_dtype=0, scale=dummy, qmin=-128, qmax=127, x=dummy, q=dummy):
        return lib.ao_int8_quantize_static(x, ldx, M, K, pre, pre_dtype, scale, 0, None, 0, qmin, qmax, q, dummy, None,
                                           None)

    def err():
        return lib.ao_b200_last_error()

    assert call(K=4100) == -1 and b"bad sizes" in err()
    assert call(K=0) == -1 and b"bad sizes" in err()
    assert call(pre_dtype=3) == -1 and b"pre_scale_dtype" in err()
    assert call(pre_dtype=1) == -1 and b"exactly when" in err()
    assert call(pre=dummy) == -1 and b"exactly when" in err()
    assert call(qmin=-129) == -1 and b"bad range" in err()
    assert call(qmin=5, qmax=4) == -1 and b"bad range" in err()
    assert call(scale=None) == -1 and b"null pointer" in err()
    assert call(q=None) == -1 and b"null pointer" in err()
    assert call(pre=ctypes.c_void_p(4100), pre_dtype=2) == -1 and b"16-byte aligned" in err()
    assert call(ldx=4100) == -1 and b"multiple of 8" in err()
    assert call(ldx=4088) == -1 and b"ldx" in err()
    assert call(x=ctypes.c_void_p(4104)) == -1 and b"16-byte aligned" in err()
    assert call(M=0, x=None, scale=None, q=None) == 0   # M == 0: nothing to do, no CUDA call


# ---------------------------------------------------------------- the activation attributes travel with the weight
def _static_weight(e=None, n=64, k=128):
    from ao_b200.quantization import Int8Tensor, MappingType, PerRow, QuantizeTensorToInt8Kwargs

    torch.manual_seed(0)
    shape = (n, k) if e is None else (e, n, k)
    w = Int8Tensor.from_hp(
        torch.randn(*shape).to(torch.bfloat16), PerRow(),
        act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow(), mapping_type=MappingType.ASYMMETRIC),
        act_quant_scale=torch.rand(4, 1) + 0.01, act_quant_zero_point=torch.tensor([[1], [-2], [3], [0]], dtype=torch.int8),
        act_pre_scale=torch.rand(k) + 0.5)
    return w


def _same_act_attrs(a, b):
    return all(getattr(a, n) is getattr(b, n) for n in ("act_quant_scale", "act_quant_zero_point", "act_pre_scale",
                                                       "act_quant_kwargs"))


def test_select_and_slice_keep_the_activation_attributes():
    w3 = _static_weight(e=3)
    for e in range(3):
        we = w3[e]
        assert _same_act_attrs(we, w3) and torch.equal(we.qdata, w3.qdata[e]) and torch.equal(we.scale, w3.scale[e])
        assert list(we.block_size) == list(w3.block_size[1:])
    w = _static_weight()
    for sl in (w[:32], w[:, :64], w.narrow(0, 16, 16)):
        assert _same_act_attrs(sl, w)


def test_torch_save_and_safetensors_round_trip(tmp_path):
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict

    w = _static_weight()

    def same(a, b):
        return all(torch.equal(getattr(a, n), getattr(b, n)) for n in (
            "qdata", "scale", "zero_point", "act_quant_scale", "act_quant_zero_point", "act_pre_scale")) and (
            a.act_quant_kwargs == b.act_quant_kwargs and list(a.block_size) == list(b.block_size))

    torch.save({"weight": w}, tmp_path / "w.pt")
    assert same(torch.load(tmp_path / "w.pt", weights_only=True)["weight"], w)
    flat, meta = flatten_tensor_state_dict({"m.weight": w})
    assert all(type(v) is torch.Tensor for v in flat.values())
    sd, leftover = unflatten_tensor_state_dict(flat, meta)
    assert leftover == {} and same(sd["m.weight"], w)
