"""Static e4m3 activations (Float8StaticActivationFloat8WeightConfig) without a GPU: the config's fields, defaults and
rules, its JSON round trip, the quantize handler (missing scale, observer steps, shape skip, device move, FqnToConfig),
the ops' Meta shapes and schemas and the C ABI's argument checks, the calibrated scales through select / slice /
transpose / torch.save, the scale-shape rule of the linear, and a numpy restatement of the quantization contract
against the reference's codes in tests/golden/fp8_static.npz."""
import ctypes
import dataclasses
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


# the finite non-negative e4m3 values in code order (codes 0x00 .. 0x7E)
E4M3 = torch.arange(127, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).float().numpy()


def e4m3_codes_ref(x_bits, scale):
    """The contract restated in numpy: e4m3(clamp(fp32(x) / s, -448, 448)) with an IEEE float32 division and round half
    to even onto the e4m3 grid (quantum 2^(e-3), subnormals 2^-9); NaN gives 0x7F (its sign is not part of the
    contract: see is_nan_code)."""
    x = f32_of_bf16(x_bits)
    s = np.asarray(scale, dtype=np.float32).reshape(-1, 1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        v = np.clip((x / s).astype(np.float32), -448, 448)
        a = np.abs(v)
        e = np.floor(np.log2(np.where(a > 0, a, 1))).astype(np.int32)
        quantum = np.exp2(np.maximum(e, -6) - 3).astype(np.float32)
        r = np.rint(a / quantum) * quantum
    idx = np.searchsorted(E4M3, np.where(np.isnan(r), 0, r)).astype(np.uint8)
    code = idx | np.where(np.signbit(v), 0x80, 0).astype(np.uint8)
    return np.where(np.isnan(v), np.uint8(0x7F), code).astype(np.uint8)


def is_nan_code(c):
    return (np.asarray(c) & 0x7F) == 0x7F


def same_codes(a, b):
    """Equal codes, where a NaN code equals any NaN code: the sign of a NaN quotient is the division's choice (x86 gives
    0/0 a negative NaN, the GPU a positive one)."""
    na, nb = is_nan_code(a), is_nan_code(b)
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a), np.where(nb, 0, b))


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "fp8_static.npz"))


# ---------------------------------------------------------------- the contract against the reference's codes
def test_restatement_reproduces_the_reference_codes(golden):
    qcases = json.loads(str(golden["qcases"]))
    assert len(qcases) == 27
    ties = clamped = nans = zero_scale = 0
    for q, case in enumerate(qcases):
        x, s, want = golden[f"q{q}_x"], golden[f"q{q}_scale"], golden[f"q{q}_q"]
        assert same_codes(e4m3_codes_ref(x, s), want), case
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            v = np.abs(f32_of_bf16(x) / s.reshape(-1, 1).astype(np.float32))
            clamped += int(np.sum(v > 448))
            fin = np.isfinite(v) & (v <= 448) & (v >= 2.0 ** -6)
            v = np.where(fin, v, 1)
            ties += int(np.sum(fin & (np.mod(v / np.exp2(np.floor(np.log2(v)) - 3), 1) == 0.5)))
        nans += int(np.sum(is_nan_code(want)))
        zero_scale += int(np.sum(s == 0))
    assert ties > 1000 and clamped > 500 and nans > 20 and zero_scale >= 6   # ties, the clamp, NaN, 0/0 and x/0


# ---------------------------------------------------------------- config
def test_config_fields_defaults_and_rules():
    from ao_b200.float8.inference import Float8MMConfig
    from ao_b200.quantization import (Float8StaticActivationFloat8WeightConfig, KernelPreference, PerRow, PerTensor,
                                      QuantizeTensorToFloat8Kwargs)

    c = Float8StaticActivationFloat8WeightConfig()
    assert [f.name for f in dataclasses.fields(c)] == [
        "step", "act_quant_scale", "activation_dtype", "weight_dtype", "granularity", "mm_config", "kernel_preference",
        "set_inductor_config", "quantize_and_dequantize_output", "output_act_quant_scale"]
    assert (c.step, c.act_quant_scale, c.activation_dtype, c.weight_dtype, c.granularity, c.mm_config,
            c.kernel_preference, c.set_inductor_config, c.quantize_and_dequantize_output, c.output_act_quant_scale) == (
        None, None, torch.float8_e4m3fn, torch.float8_e4m3fn, None, Float8MMConfig(use_fast_accum=True),
        KernelPreference.AUTO, True, False, None)
    assert Float8StaticActivationFloat8WeightConfig(step="PREPARE").step == "prepare"
    assert Float8StaticActivationFloat8WeightConfig(step="Convert").step == "convert"
    with pytest.raises(ValueError, match="is not one of"):
        Float8StaticActivationFloat8WeightConfig(step="calibrate")
    mm = Float8MMConfig(use_fast_accum=False)
    assert Float8StaticActivationFloat8WeightConfig(mm_config=mm).mm_config is mm
    assert c.get_act_quant_kwargs() == QuantizeTensorToFloat8Kwargs(
        float8_dtype=torch.float8_e4m3fn, granularity=PerTensor(), mm_config=Float8MMConfig(use_fast_accum=True))
    assert Float8StaticActivationFloat8WeightConfig(granularity=PerRow()).get_act_quant_kwargs().granularity == PerRow()


def test_config_json_round_trip_as_int8_static():
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.quantization import (Float8StaticActivationFloat8WeightConfig, Int8StaticActivationInt8WeightConfig,
                                      PerRow)

    c = Float8StaticActivationFloat8WeightConfig(granularity=PerRow(), step="prepare")
    d = config_to_dict(c)
    assert d["_type"] == "Float8StaticActivationFloat8WeightConfig"
    assert config_from_dict(json.loads(json.dumps(d))) == c
    # a calibrated tensor in the config: whatever the int8 static config does, this one does too
    def outcome(cfg):
        try:
            return type(config_from_dict(config_to_dict(cfg)))
        except Exception as e:  # noqa: BLE001
            return type(e)

    s = torch.tensor([[0.5]])
    assert outcome(Float8StaticActivationFloat8WeightConfig(act_quant_scale=s)) in (
        outcome(Int8StaticActivationInt8WeightConfig(act_quant_scale=s)), Float8StaticActivationFloat8WeightConfig)
    i8, f8 = (outcome(Int8StaticActivationInt8WeightConfig(act_quant_scale=s)),
              outcome(Float8StaticActivationFloat8WeightConfig(act_quant_scale=s)))
    assert (i8 is Int8StaticActivationInt8WeightConfig) == (f8 is Float8StaticActivationFloat8WeightConfig), (i8, f8)


# ---------------------------------------------------------------- handler
def _static(**kw):
    from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig

    return Float8StaticActivationFloat8WeightConfig(**kw)


def test_handler_errors_and_shape_skip(caplog):
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import PerBlock, PerRow, PerTensor, quantize_

    with pytest.raises(ValueError, match="act_quant_scale must be provided for direct quantization"):
        quantize_(nn.Linear(128, 64).to(torch.bfloat16), _static())
    for step in ("prepare", "convert"):
        with pytest.raises(NotImplementedError, match="observer flow"):
            quantize_(nn.Linear(128, 64).to(torch.bfloat16), _static(step=step, act_quant_scale=torch.tensor([[1.0]])))
    with pytest.raises(NotImplementedError, match="PerTensor or PerRow"):
        quantize_(nn.Linear(128, 64).to(torch.bfloat16),
                  _static(act_quant_scale=torch.tensor([[1.0]]), granularity=PerBlock([1, 128])))
    s = torch.tensor([[0.05]])
    for k, n in ((120, 64), (128, 60)):
        lin = nn.Linear(k, n).to(torch.bfloat16)
        with caplog.at_level(logging.INFO, logger="ao_b200.quantization.quant_api"):
            quantize_(lin, _static(act_quant_scale=s))
        assert type(lin.weight.data) is torch.Tensor
        assert "Skipping float8 quantization" in caplog.text
    for gran, wscale in ((None, (1, 1)), (PerTensor(), (1, 1)), (PerRow(), (64, 1))):
        lin = nn.Linear(128, 64).to(torch.bfloat16)
        so = torch.tensor([[0.5]])
        quantize_(lin, _static(act_quant_scale=s, granularity=gran, output_act_quant_scale=so))
        w = lin.weight
        assert isinstance(w, PrototypeFloat8Tensor) and tuple(w.scale.shape) == wscale
        assert torch.equal(w.act_quant_scale, s) and torch.equal(w.output_act_quant_scale, so)
        assert w.act_quant_kwargs == w.output_act_quant_kwargs == _static(granularity=gran).get_act_quant_kwargs()
        assert w.qdata.dtype == torch.float8_e4m3fn and w.dtype == torch.bfloat16
    lin = nn.Linear(128, 64).to(torch.bfloat16)
    quantize_(lin, _static(act_quant_scale=s))
    assert lin.weight.output_act_quant_scale is None and lin.weight.output_act_quant_kwargs is None
    assert "PrototypeFloat8Tensor" in repr(lin)


def test_handler_moves_the_calibrated_tensors_to_the_weight_device():
    from ao_b200.prototype.quantization.quant_api import _float8_static_activation_float8_weight_quantize_tensor

    w = torch.empty(64, 128, dtype=torch.bfloat16, device="meta")
    cfg = _static(act_quant_scale=torch.tensor([[0.05]]), output_act_quant_scale=torch.tensor([[0.5]]))
    q = _float8_static_activation_float8_weight_quantize_tensor(w, cfg)
    assert q.act_quant_scale.device.type == "meta" and q.output_act_quant_scale.device.type == "meta"
    assert cfg.act_quant_scale.device.type == "cpu" and cfg.output_act_quant_scale.device.type == "cpu"


def test_fqn_to_config_reaches_the_named_module_and_parameter():
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import FqnToConfig, quantize_

    s = torch.tensor([[0.02]])
    for key in ("a", "a.weight"):
        m = nn.Sequential()
        m.add_module("a", nn.Linear(128, 64).to(torch.bfloat16))
        m.add_module("b", nn.Linear(64, 32).to(torch.bfloat16))
        quantize_(m, FqnToConfig({key: _static(act_quant_scale=s)}), filter_fn=None)
        assert isinstance(m.a.weight, PrototypeFloat8Tensor) and torch.equal(m.a.weight.act_quant_scale, s), key
        assert type(m.b.weight.data) is torch.Tensor, key


def test_fixture_weights_match_from_hp(golden):
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import PerRow, PerTensor

    for si in range(3):
        w = torch.from_numpy(golden[f"s{si}_w"].view(np.int16)).view(torch.bfloat16)
        for gname, gran in (("PerTensor", PerTensor()), ("PerRow", PerRow())):
            t = PrototypeFloat8Tensor.from_hp(w, torch.float8_e4m3fn, gran)
            assert np.array_equal(t.qdata.view(torch.uint8).numpy(), golden[f"s{si}_{gname}_wq"]), (si, gname)
            assert np.array_equal(t.scale.numpy(), golden[f"s{si}_{gname}_ws"]), (si, gname)


# ---------------------------------------------------------------- ops and C ABI
def test_meta_shapes_and_schemas():
    import ao_b200  # noqa: F401

    op = torch.ops.ao_b200.fp8_quantize_static
    x = torch.empty(130, 256, dtype=torch.bfloat16, device="meta")
    q, s = op(x, torch.empty(1, 1, device="meta"))
    assert (q.shape, q.dtype, s.shape, s.dtype) == ((130, 256), torch.float8_e4m3fn, (130,), torch.float32)
    assert str(op.default._schema).endswith("(Tensor x, Tensor scale) -> (Tensor, Tensor)")
    op2 = torch.ops.ao_b200.fp8_static_linear
    wq = torch.empty(48, 256, dtype=torch.float8_e4m3fn, device="meta")
    for w_scale, out_scale in ((torch.empty(48, device="meta"), None), (torch.empty(1, device="meta"),
                                                                        torch.empty(130, 1, device="meta"))):
        y = op2(q, s, wq, w_scale, None, out_scale)
        assert (y.shape, y.dtype, y.device.type) == ((130, 48), torch.bfloat16, "meta")
    assert str(op2.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale, Tensor? bias, Tensor? out_scale) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    dummy = ctypes.c_void_p(4096)   # never dereferenced: every call below fails its checks or returns before a launch

    def err():
        return lib.ao_b200_last_error()

    def quant(ldx=4096, M=4, K=4096, scale=dummy, x=dummy, q=dummy, xs=dummy):
        return lib.ao_fp8_quantize_static(x, ldx, M, K, scale, 0, q, xs, None)

    assert quant(K=4100) == -1 and b"bad sizes" in err()
    assert quant(K=0) == -1 and b"bad sizes" in err()
    assert quant(M=-1) == -1 and b"bad sizes" in err()
    assert quant(scale=None) == -1 and b"null pointer" in err()
    assert quant(q=None) == -1 and b"null pointer" in err()
    assert quant(xs=None) == -1 and b"null pointer" in err()
    assert quant(ldx=4100) == -1 and b"multiple of 8" in err()
    assert quant(ldx=4088) == -1 and b"ldx" in err()
    assert quant(x=ctypes.c_void_p(4104)) == -1 and b"16-byte aligned" in err()
    assert quant(M=0, x=None, scale=None, q=None, xs=None) == 0   # M == 0: nothing to do, no CUDA call

    def lin(M=4, K=4096, N=4096, xq=dummy, ws=dummy, y=dummy):
        return lib.ao_fp8_static_linear(xq, dummy, M, K, dummy, ws, 1, N, None, None, 0, y, dummy,
                                        ctypes.c_size_t(1 << 20), None)

    assert lin(K=4104) == -1 and b"K=4104" in err()
    assert lin(N=4104) == -1 and b"N=4104" in err()
    assert lin(N=0) == -1 and b"bad sizes" in err()
    assert lin(ws=None) == -1 and b"null pointer" in err()
    assert lin(y=None) == -1 and b"null pointer" in err()
    assert lin(xq=ctypes.c_void_p(4104)) == -1 and b"16-byte aligned" in err()
    assert lin(M=0, xq=None, ws=None, y=None) == 0


# ---------------------------------------------------------------- the calibrated scales travel with the weight
def _static_weight(e=None, n=64, k=128):
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import PerRow, QuantizeTensorToFloat8Kwargs

    torch.manual_seed(0)
    shape = (n, k) if e is None else (e, n, k)
    kw = QuantizeTensorToFloat8Kwargs(granularity=PerRow())
    return PrototypeFloat8Tensor.from_hp(torch.randn(*shape).to(torch.bfloat16), torch.float8_e4m3fn, PerRow(),
                                         act_quant_kwargs=kw, act_quant_scale=torch.rand(4, 1) + 0.01,
                                         output_act_quant_scale=torch.rand(4, 1) + 0.5, output_act_quant_kwargs=kw)


def _same_act_attrs(a, b):
    return all(getattr(a, n) is getattr(b, n) for n in ("act_quant_scale", "output_act_quant_scale", "act_quant_kwargs",
                                                       "output_act_quant_kwargs", "mm_config", "kernel_preference"))


def test_select_slice_and_transpose_keep_the_calibrated_scales():
    w3 = _static_weight(e=3)
    for e in range(3):
        we = w3[e]
        assert _same_act_attrs(we, w3) and torch.equal(we.qdata.view(torch.uint8), w3.qdata[e].view(torch.uint8)) and torch.equal(we.scale, w3.scale[e])
        assert list(we.block_size) == list(w3.block_size[1:]) and we.dtype == torch.bfloat16
    w = _static_weight()
    for sl, rows in ((w[:32], 32), (w[:, :64], 64), (w.narrow(0, 16, 16), 16)):
        assert _same_act_attrs(sl, w)
    assert torch.equal(w[:32].scale, w.scale[:32]) and torch.equal(w[:, :64].scale, w.scale)
    assert torch.equal(w.narrow(0, 16, 16).qdata.view(torch.uint8), w.qdata[16:32].view(torch.uint8))
    for t in (w.t(), w.transpose(0, 1)):
        assert _same_act_attrs(t, w) and t.shape == (128, 64) and list(t.block_size) == [128, 1]
    for c in (w.detach(), w.clone(), w.to("cpu")):
        assert torch.equal(c.act_quant_scale, w.act_quant_scale) and c.output_act_quant_kwargs == w.output_act_quant_kwargs


def test_torch_save_round_trip(tmp_path):
    w = _static_weight()
    torch.save({"weight": w}, tmp_path / "w.pt")
    r = torch.load(tmp_path / "w.pt", weights_only=True)["weight"]
    assert type(r) is type(w)
    assert all(torch.equal(getattr(r, n).view(torch.uint8) if n == "qdata" else getattr(r, n),
                           getattr(w, n).view(torch.uint8) if n == "qdata" else getattr(w, n))
               for n in ("qdata", "scale", "act_quant_scale", "output_act_quant_scale"))
    assert r.act_quant_kwargs == w.act_quant_kwargs and list(r.block_size) == list(w.block_size)


def test_linear_rejects_a_scale_of_another_batch():
    import torch.nn.functional as F

    w = _static_weight()   # [4, 1] scales
    with pytest.raises(ValueError, match="act_quant_scale has shape"):
        F.linear(torch.randn(5, 128).to(torch.bfloat16), w)
    w.act_quant_scale = torch.rand(5, 1)
    with pytest.raises(ValueError, match="output_act_quant_scale has shape"):
        F.linear(torch.randn(5, 128).to(torch.bfloat16), w)
