"""CPU tests: the C-ABI library loads and exports every declared symbol; host-side logic
(configs, registry, module walk, dispatch tables, (de)serialisation) behaves like the reference's."""
import ctypes
import os
import re
from collections import OrderedDict

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_c_abi_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "ao_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = re.findall(r"\b(ao_[a-z0-9_]+)\s*\(", hdr)
    assert len(names) >= 18
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    for n in names:
        assert hasattr(lib, n), f"libao_b200.so does not export {n}"
    lib.ao_b200_version.restype = ctypes.c_int
    assert lib.ao_b200_version() >= 100
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    assert lib.ao_b200_workspace_bytes(32, 4096) >= 16 * 1024 * 1024


def test_c_abi_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call (error code + message, no crash)."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    rc = lib.ao_int4_tilepacked_linear(None, 4, 1000, None, None, 32, 128, None, None, 128, None, ctypes.c_size_t(0), 0, None)
    assert rc == -1 and b"multiple of 1024" in lib.ao_b200_last_error()
    rc = lib.ao_int4_tilepacked_linear(None, 4, 1024, None, None, 48, 128, None, None, 128, None, ctypes.c_size_t(0), 0, None)
    assert rc == -1 and b"group_size" in lib.ao_b200_last_error()
    rc = lib.ao_int4_pack_tile4d(None, None, 12, 128, 8, None)
    assert rc == -1
    rc = lib.ao_int4_hqq_quantize(None, 8, 1024, 48, None, None, None, None, ctypes.c_size_t(0), None)
    assert rc == -1 and b"group_size" in lib.ao_b200_last_error()
    lib.ao_int4_hqq_workspace_bytes.restype = ctypes.c_size_t
    assert lib.ao_int4_hqq_workspace_bytes(4096, 4096, 32) >= 2 * 4 * 4096 * 128
    rc = lib.ao_fp8_rowwise_linear(None, None, 4, 4096, None, None, 100, None, None, None, ctypes.c_size_t(0), None)
    assert rc == -1 and b"multiple of 16" in lib.ao_b200_last_error()
    # M == 0 is a no-op success (reference: empty-input short circuit, int4_tile_packed_to_4d_tensor.py:284-285)
    assert lib.ao_int4_tilepacked_linear(None, 0, 1024, None, None, 32, 128, None, None, 128, None, ctypes.c_size_t(0), 0, None) == 0


# Every dense linear's C entry point as fn(x, M, p): x the activation, M the rows, p every other pointer.  K = 4096 and
# N = 256 pass every format's K and N rules.
_K, _N = 4096, 256
_WS = ctypes.c_size_t(1 << 20)
_DENSE = {
    "ao_int8_dyn_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_int8_mm_i32": ("xq", lambda x, M, p: (x, M, _K, p, _N, p, p, _WS, None)),
    "ao_int8_weight_linear": ("x", lambda x, M, p: (x, _K, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_fp8_weight_linear": ("x", lambda x, M, p: (x, _K, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_fp8_rowwise_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_fp8_static_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, 1, _N, p, p, 0, p, p, _WS, None)),
    "ao_fp8_blockwise_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_fp8_sparse_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, p, _N, p, p, p, _WS, None)),
    "ao_mxfp8_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_mxfp4_linear": ("xq", lambda x, M, p: (x, p, M, _K, p, p, _N, p, p, p, _WS, None)),
    "ao_nvfp4_linear": ("xq", lambda x, M, p: (x, p, p, M, _K, p, p, p, _N, p, p, p, _WS, None)),
    "ao_nvfp4_weight_linear_ex": ("x", lambda x, M, p: (x, _K, p, M, _K, p, p, p, 0, _N, p, p, p, _WS, None)),
    "ao_int4_tilepacked_linear_strided": ("x", lambda x, M, p: (x, _K, M, _K, p, p, 32, _N, p, p, _N, p, _WS, 0, None)),
}


@pytest.mark.parametrize("name", sorted(_DENSE))
def test_dense_entry_points_check_the_activation_before_any_cuda_call(name):
    """Every dense linear rejects an activation that does not start on 16 bytes with a message (the kernels read it by
    TMA or by 16-byte vector loads) and returns 0 at M == 0 without looking at a pointer.  No GPU: a CUDA call would
    fail with a different error."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    x_name, args = _DENSE[name]
    fn = getattr(lib, name)
    one = ctypes.c_void_p(4096)
    assert fn(*args(ctypes.c_void_p(4104), 4, one)) == -1
    assert f"{x_name} must be 16-byte aligned".encode() in lib.ao_b200_last_error(), lib.ao_b200_last_error()
    assert fn(*args(None, 4, one)) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert fn(*args(None, 0, None)) == 0


def test_pdl_fence_on_the_null_stream():
    """ao_b200_pdl_fence(NULL) launches its empty kernel on the legacy default stream; without a device it reports the
    failed launch instead of crashing.  torch.ops.ao_b200.pdl_fence is its registration."""
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_pdl_fence.argtypes = [ctypes.c_void_p]
    rc = lib.ao_b200_pdl_fence(None)
    if torch.cuda.is_available():
        assert rc == 0, lib.ao_b200_last_error()
        torch.cuda.synchronize()
    else:
        assert rc == -2 and b"pdl_fence_kernel" in lib.ao_b200_last_error()
    assert torch.ops.ao_b200.pdl_fence.default._schema.returns == []


def test_torch_ops_registered_with_meta_kernels():
    import ao_b200  # noqa: F401

    x = torch.empty(3, 1024, dtype=torch.bfloat16, device="meta")
    qd = torch.empty(16, 8, 32, 4, dtype=torch.int32, device="meta")
    sz = torch.empty(32, 128, 2, dtype=torch.bfloat16, device="meta")
    assert torch.ops.ao_b200.int4_tilepacked_linear(x, qd, 32, sz, None).shape == (3, 128)
    assert torch.ops.ao_b200.int4_tilepacked_linear(x, qd, 32, sz, None, 100).shape == (3, 100)
    q, s = torch.ops.ao_b200.int8_quantize_rowwise(x)
    assert q.dtype == torch.int8 and s.shape == (3, 1)
    q4, s4, z4 = torch.ops.ao_b200.int4_hqq_quantize(x, 64)
    assert q4.shape == (3, 1024) and q4.dtype == torch.uint8 and s4.shape == z4.shape == (3, 16) and s4.dtype == torch.bfloat16
    q, s = torch.ops.ao_b200.mxfp8_quantize(x, True)
    assert s.shape == (32, 16 * 8)
    q, s = torch.ops.ao_b200.nvfp4_quantize(x, None, True)
    assert q.shape == (3, 512) and s.shape == (32, 16 * 16)
    with pytest.raises(Exception):
        torch.ops.ao_b200.int4_tilepacked_linear(torch.empty(3, 1024, dtype=torch.bfloat16), qd.to("cpu") if False else torch.empty(16, 8, 32, 4, dtype=torch.int32), 32, torch.empty(32, 128, 2, dtype=torch.bfloat16), None)


def test_config_defaults_match_reference():
    from ao_b200.prototype.mx_formats import (MXDynamicActivationMXWeightConfig, NVFP4DynamicActivationNVFP4WeightConfig,
                                              NVFP4WeightOnlyConfig, ScaleCalculationMode)
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Int4PackingFormat, Int4WeightOnlyConfig,
                                      Int8DynamicActivationInt8WeightConfig, KernelPreference, MappingType, PerRow, PerTensor)

    c = Int4WeightOnlyConfig()
    assert (c.group_size, c.int4_packing_format, c.int4_tile_packed_ntile, c.version) == (128, Int4PackingFormat.PLAIN, 8, 2)
    c = Int8DynamicActivationInt8WeightConfig()
    assert c.act_mapping_type == MappingType.SYMMETRIC and c.granularity == PerRow() and c.version == 2 and c.weight_only_decode is False
    with pytest.raises(ValueError):
        Int8DynamicActivationInt8WeightConfig(version=1)
    c = Float8DynamicActivationFloat8WeightConfig()
    assert c.granularity == [PerTensor(), PerTensor()] and c.mm_config.use_fast_accum is True
    assert Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()).granularity == [PerRow(), PerRow()]
    with pytest.raises(ValueError):
        Float8DynamicActivationFloat8WeightConfig(granularity=[PerRow(), PerTensor()])
    c = MXDynamicActivationMXWeightConfig()
    assert c.block_size == 32 and c.scaling_mode == ScaleCalculationMode.RCEIL and c.kernel_preference == KernelPreference.AUTO
    assert NVFP4DynamicActivationNVFP4WeightConfig().use_dynamic_per_tensor_scale is True
    assert NVFP4WeightOnlyConfig().use_dynamic_per_tensor_scale is True
    with pytest.raises(AssertionError):
        Int4WeightOnlyConfig(int4_tile_packed_ntile=4)


def test_config_json_roundtrip():
    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig, NVFP4WeightOnlyConfig
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, FqnToConfig, Int4WeightOnlyConfig,
                                      Int8DynamicActivationInt8WeightConfig, PerRow)

    cfgs = [Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d"),
            Int8DynamicActivationInt8WeightConfig(), Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()),
            MXDynamicActivationMXWeightConfig(), NVFP4WeightOnlyConfig(use_dynamic_per_tensor_scale=False)]
    for c in cfgs:
        d = config_to_dict(c)
        assert d["_type"] == type(c).__name__ and "_version" in d and "_data" in d
        assert config_from_dict(d) == c
    f = FqnToConfig(OrderedDict([("re:.*q_proj", cfgs[0]), ("lm_head", None), ("_default", cfgs[1])]))
    g = config_from_dict(config_to_dict(f))
    assert list(g.fqn_to_config.keys()) == ["re:.*q_proj", "lm_head", "_default"] and g.fqn_to_config["lm_head"] is None
    with pytest.raises(ValueError):
        config_from_dict({"_type": "os", "_data": {}})
    with pytest.raises(ValueError):
        config_from_dict({"_type": "Path", "_version": 1, "_data": {}})   # not in the allow-listed modules
    d = config_to_dict(cfgs[0])
    d["_version"] = 99
    with pytest.raises(ValueError):
        config_from_dict(d)


def test_config_json_is_the_reference_wire_format():
    """config_to_dict output == what torchao 0.19 writes for the same configs (fixture made by
    tests/golden/make_golden_configs.py; this is what HF `TorchAoConfig` stores in config.json), and the reference's
    dicts load into equal configs."""
    import json

    from ao_b200.core.config import config_from_dict, config_to_dict
    from ao_b200.prototype.mx_formats import (MXDynamicActivationMXWeightConfig, NVFP4DynamicActivationNVFP4WeightConfig,
                                              NVFP4WeightOnlyConfig)
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, FqnToConfig, Int4WeightOnlyConfig,
                                      Int8DynamicActivationInt8WeightConfig, PerRow)

    with open(os.path.join(ROOT, "tests", "golden", "config_json.json")) as f:
        gold = json.load(f)
    cfgs = OrderedDict()
    cfgs["int4_tile_g32"] = Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d")
    cfgs["int4_tile_g128_hqq"] = Int4WeightOnlyConfig(group_size=128, int4_packing_format="tile_packed_to_4d",
                                                      int4_choose_qparams_algorithm="hqq")
    cfgs["int8_dyn"] = Int8DynamicActivationInt8WeightConfig()
    cfgs["fp8_rowwise"] = Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())
    cfgs["fp8_default"] = Float8DynamicActivationFloat8WeightConfig()
    cfgs["mxfp8"] = MXDynamicActivationMXWeightConfig()
    cfgs["nvfp4_dyn"] = NVFP4DynamicActivationNVFP4WeightConfig()
    cfgs["nvfp4_wo"] = NVFP4WeightOnlyConfig(use_dynamic_per_tensor_scale=False)
    cfgs["fqn"] = FqnToConfig(OrderedDict([("re:.*q_proj", cfgs["int4_tile_g32"]), ("lm_head", None),
                                           ("_default", cfgs["int8_dyn"])]))
    assert set(gold) == set(cfgs)
    for name, c in cfgs.items():
        assert config_to_dict(c) == gold[name], name
        assert config_from_dict(gold[name]) == c, name


def test_handler_registry_and_module_walk():
    from ao_b200.core.config import AOBaseConfig
    from ao_b200.quantization import quantize_, register_quantize_module_handler
    from ao_b200.quantization.quant_api import _is_linear
    from dataclasses import dataclass

    @dataclass
    class DoubleConfig(AOBaseConfig):
        factor: float = 2.0

    seen = []

    @register_quantize_module_handler(DoubleConfig)
    def _h(module, config, *, parameter_name="weight"):
        seen.append(module)
        with torch.no_grad():
            getattr(module, parameter_name).mul_(config.factor)
        return module

    m = torch.nn.Sequential(torch.nn.Linear(8, 8), torch.nn.ReLU(), torch.nn.Sequential(torch.nn.Linear(8, 4)), torch.nn.LayerNorm(4))
    w0 = m[0].weight.detach().clone()
    assert quantize_(m, DoubleConfig()) is None
    assert len(seen) == 2 and torch.equal(m[0].weight, w0 * 2)
    seen.clear()
    quantize_(m, DoubleConfig(), filter_fn=lambda mod, fqn: _is_linear(mod) and fqn == "2.0")
    assert len(seen) == 1 and seen[0] is m[2][0]
    with pytest.raises(AssertionError):
        quantize_(m, lambda x: x)
    assert not _is_linear(torch.nn.modules.linear.NonDynamicallyQuantizableLinear(4, 4))


def test_fqn_to_config_precedence():
    from ao_b200.core.config import AOBaseConfig
    from ao_b200.quantization import FqnToConfig, quantize_, register_quantize_module_handler
    from dataclasses import dataclass

    @dataclass
    class TagConfig(AOBaseConfig):
        tag: str = ""

    @register_quantize_module_handler(TagConfig)
    def _h(module, config, *, parameter_name="weight"):
        module._tag = config.tag
        return module

    class Blk(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj = torch.nn.Linear(4, 4)
            self.k_proj = torch.nn.Linear(4, 4)
            self.norm = torch.nn.LayerNorm(4)

    m = torch.nn.ModuleDict({"l0": Blk(), "l1": Blk()})
    cfg = FqnToConfig(OrderedDict([("l0.q_proj", TagConfig("exact")), ("re:.*\\.q_proj", TagConfig("regex")),
                                   ("l1.k_proj", None), ("_default", TagConfig("default"))]))
    quantize_(m, cfg, filter_fn=None)
    assert m["l0"].q_proj._tag == "exact" and m["l1"].q_proj._tag == "regex"
    assert m["l0"].k_proj._tag == "default" and not hasattr(m["l1"].k_proj, "_tag") and not hasattr(m["l0"].norm, "_tag")
    with pytest.raises(ValueError):
        quantize_(m, cfg, filter_fn=lambda *_: True)


def test_int4_skip_rule_and_unsupported_formats():
    """K % group_size != 0 -> layer silently left unquantized (quant_api.py:549-553); PLAIN needs mslk in the
    reference and raises here."""
    from ao_b200.quantization import Int4WeightOnlyConfig, quantize_

    lin = torch.nn.Linear(100, 16, bias=False, dtype=torch.bfloat16)
    quantize_(lin, Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d"))
    assert type(lin.weight.data) is torch.Tensor
    lin = torch.nn.Linear(128, 16, bias=False, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        quantize_(lin, Int4WeightOnlyConfig(group_size=32))
    with pytest.raises(NotImplementedError):  # CPU tensor: no CPU packing kernel; same exception type as the reference
        quantize_(lin, Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d"))
    lin32 = torch.nn.Linear(128, 16, bias=False, dtype=torch.float32)
    with pytest.raises(AssertionError):
        quantize_(lin32, Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d"))


def test_granularity_block_sizes_and_primitives_vs_oracle():
    import numpy as np

    from ao_b200.quantization import PerRow, PerTensor
    from ao_b200.quantization.quant_primitives import (choose_qparams_affine_int8, choose_qparams_affine_tinygemm,
                                                       choose_scale_float8, quantize_affine_float8, quantize_affine_int8,
                                                       quantize_affine_tinygemm)
    from ao_b200.quantization.utils import get_block_size, pack_tinygemm_scales_and_zeros
    from oracle import oracle as o

    assert get_block_size((4, 8), PerRow()) == (1, 8) and get_block_size((4, 8), PerTensor()) == (4, 8)
    assert get_block_size((2, 4, 8), PerRow()) == (1, 1, 8)
    torch.manual_seed(0)
    w = (torch.randn(24, 256) * 0.02).to(torch.bfloat16)
    w[3, :32] = 0
    s, z = choose_qparams_affine_tinygemm(w, 32)
    q = quantize_affine_tinygemm(w, 32, s, z)
    so, zo = o.int4_choose_qparams(o.bf16_bits(w), 32)
    assert np.array_equal(o.bf16_bits(s), so) and np.array_equal(o.bf16_bits(z), zo)
    assert np.array_equal(q.numpy().astype(np.uint8), o.int4_quantize(o.bf16_bits(w), 32, so, zo))
    assert np.array_equal(o.bf16_bits(pack_tinygemm_scales_and_zeros(s, z)), o.pack_scales_and_zeros(so, zo))
    x = torch.randn(5, 192).to(torch.bfloat16)
    x[2] = 0
    sc, zp = choose_qparams_affine_int8(x, [1, 192])
    qi = quantize_affine_int8(x, [1, 192], sc, zp)
    qo, so = o.int8_quantize_rowwise(o.bf16_bits(x))
    assert np.array_equal(sc.reshape(-1).numpy(), so) and np.array_equal(qi.numpy(), qo)
    x = (torch.randn(6, 128) * 3).to(torch.bfloat16)
    sc = choose_scale_float8(x, [1, 128])
    qf = quantize_affine_float8(x, sc)
    qo, so = o.fp8_quantize_rowwise(o.bf16_bits(x))
    assert np.array_equal(sc.reshape(-1).numpy(), so) and np.array_equal(qf.view(torch.uint8).numpy(), qo)


def test_tensor_subclass_plumbing_on_cpu():
    """Construction, flatten/unflatten, detach/clone, state_dict round trip, copy_, slice -- no kernels needed."""
    from ao_b200.quantization import Float8Tensor, Int4TilePackedTo4dTensor, Int8Tensor, PerRow
    from ao_b200.quantization.quantize_.workflows import QuantizeTensorToInt8Kwargs

    w = torch.randn(16, 64).to(torch.bfloat16)
    t = Int8Tensor.from_hp(w, PerRow(), act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow()))
    assert t.shape == (16, 64) and t.dtype == torch.bfloat16 and t.qdata.dtype == torch.int8 and t.scale.shape == (16, 1)
    names, attrs = t.__tensor_flatten__()
    assert names == ["qdata", "scale", "zero_point"] and attrs["block_size"] == [1, 64]
    t2 = Int8Tensor.__tensor_unflatten__({n: getattr(t, n) for n in names}, attrs, None, None)
    assert torch.equal(t2.qdata, t.qdata) and t2.act_quant_kwargs == t.act_quant_kwargs
    assert torch.equal(t.detach().qdata, t.qdata) and torch.equal(t.clone().scale, t.scale)
    err = (t.dequantize().float() - w.float()).abs().max()
    assert err < 0.05
    lin = torch.nn.Linear(64, 16, bias=False)
    lin.weight = torch.nn.Parameter(t, requires_grad=False)
    import io

    buf = io.BytesIO()
    torch.save(lin.state_dict(), buf)
    buf.seek(0)
    sd = torch.load(buf, weights_only=True)
    assert isinstance(sd["weight"], Int8Tensor) and torch.equal(sd["weight"].qdata, t.qdata)
    s = t[4:8]
    assert s.shape == (4, 64) and torch.equal(s.qdata, t.qdata[4:8]) and s.scale.shape == (4, 1)
    dst = Int8Tensor.from_hp(torch.zeros(16, 64, dtype=torch.bfloat16), PerRow(),
                             act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow()))
    dst.copy_(t)
    assert torch.equal(dst.qdata, t.qdata)
    with pytest.raises(ValueError):
        dst.copy_(t[0:8])
    f = Float8Tensor.from_hp(w, granularity=PerRow())
    assert f.qdata.dtype == torch.float8_e4m3fn and f.scale.shape == (16, 1) and f.block_size == [1, 64]
    with pytest.raises(NotImplementedError):
        torch.nn.functional.linear(torch.randn(2, 64).to(torch.bfloat16), f)  # weight-only fp8: out of scope
    with pytest.raises(NotImplementedError):
        torch.relu(t)  # unhandled op raises (reference utils.py:678-697)
    qd = torch.zeros(2, 8, 32, 4, dtype=torch.int32)
    sz = torch.zeros(32, 16, 2, dtype=torch.bfloat16)
    i4 = Int4TilePackedTo4dTensor(qd, sz, [1, 32], torch.Size([16, 1024]))
    assert i4.shape == (16, 1024) and i4[8:16].qdata.shape == (1, 8, 32, 4) and i4[8:16].scale_and_zero.shape == (32, 8, 2)


def test_missing_native_library_fails_loudly(monkeypatch, tmp_path):
    from ao_b200 import _native

    monkeypatch.setattr(_native, "_LIB_DIR", tmp_path)
    monkeypatch.setattr(_native, "_LOADED", False)
    with pytest.raises(ImportError, match="native library not built"):
        _native.load_native()


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under ao_b200/ may import, link or call it."""
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "ao_b200")):
        if os.path.basename(dirpath) in ("lib", "obj", "__pycache__"):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".inc")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|ao_oracle|libao_oracle", txt, flags=re.M):
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_clean_checkout_can_build_itself(tmp_path):
    """A fresh checkout has no ao_b200/lib (git-ignored): every build entry point must work without importing the
    package's native side first, and a plain `import ao_b200` must still fail loudly."""
    import shutil
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dst = tmp_path / "repo"
    shutil.copytree(root, dst, ignore=shutil.ignore_patterns("lib", "_build", "_ref", ".git", "gpurun_out", "__pycache__",
                                                             "profiles", "golden", "*.so", "*.o", ".pytest_cache"))
    env = dict(os.environ, PYTHONPATH=str(dst))
    env.pop("AO_B200_BUILDING", None)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=dst, env=env, capture_output=True, text=True, timeout=120)
    r = run("-m", "ao_b200._build", "--dry-run")
    assert r.returncode == 0 and "int4_linear.cu" in r.stdout, r.stderr[-2000:]
    r = run("-c", "import __graft_entry__ as e; m = e.load_build_module(); print(sorted(p.name for p in m.CSRC.glob('*.cu')))")
    assert r.returncode == 0 and "lowp_linear.cu" in r.stdout, r.stderr[-2000:]
    r = run("-c", "import ao_b200")
    assert r.returncode != 0 and "native library not built" in r.stderr
