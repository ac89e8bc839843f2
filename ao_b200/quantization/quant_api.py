"""User API: ``quantize_`` + the stable configs + their module handlers.

Same names, dataclass fields and defaults as torchao/quantization/quant_api.py
(quantize_ :249-321, Int4WeightOnlyConfig :502-535, Int8WeightOnlyConfig :703-780,
Int8DynamicActivationInt8WeightConfig :808-862, Int8StaticActivationInt8WeightConfig :918-978,
Float8WeightOnlyConfig :1031-1109, Float8DynamicActivationFloat8WeightConfig :1112-1172, FqnToConfig :1514-1600;
handlers :597-627,
:885-915, :981-1028, :1299-1336).  Differences, all deliberate:
  * handlers do NOT touch global inductor flags (the reference calls
    recommended_inductor_config_setter(); this engine has no compiler in the hot path) --
    ``set_inductor_config`` is kept as an accepted, ignored field;
  * int4 packing formats other than TILE_PACKED_TO_4D raise (they need ``mslk`` in the reference too).
"""
from __future__ import annotations

import logging
import re
import types
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Any, Callable, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from ao_b200._native import require_sm90
from ao_b200.core.config import AOBaseConfig
from ao_b200.float8.inference import (FP8Granularity, Float8MMConfig, _granularity_is_a_1_128_w_128_128,
                                      _normalize_granularity)
from ao_b200.quantization.granularity import Granularity, PerGroup, PerRow, PerTensor
from ao_b200.quantization.quant_primitives import MappingType
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.workflows import (
    Float8PackingFormat, Float8Sparse2x4_2DData2DMetadataTensor, Float8Tensor, Int4ChooseQParamsAlgorithm,
    Int4PackingFormat, Int4TilePackedTo4dTensor, Int8Tensor, QuantizeTensorToFloat8Kwargs, QuantizeTensorToInt8Kwargs)
from ao_b200.quantization.transform_module import _QUANTIZE_CONFIG_HANDLER, register_quantize_module_handler

logger = logging.getLogger(__name__)

__all__ = [
    "quantize_", "Int4WeightOnlyConfig", "Int8DynamicActivationInt8WeightConfig", "Int8StaticActivationInt8WeightConfig",
    "Int8WeightOnlyConfig",
    "Float8DynamicActivationFloat8WeightConfig", "Float8WeightOnlyConfig", "FqnToConfig", "ModuleFqnToConfig",
    "fqn_matches_fqn_config", "_is_linear", "_replace_with_custom_fn_if_matches_filter",
]


# ---------------------------------------------------------------------------------------------
# module walk
# ---------------------------------------------------------------------------------------------
def _replace_with_custom_fn_if_matches_filter(model, replacement_fn, filter_fn, cur_fqn="", device=None,
                                              extra_args: Optional[Tuple[Any, ...]] = ()):
    """Depth-first: replace every child for which filter_fn(child, fqn) holds (reference :120-163)."""
    if filter_fn(model, cur_fqn[:-1]):
        if device is not None:
            model.to(device=device)
        return replacement_fn(model, *extra_args)
    for name, child in list(model.named_children()):
        new_child = _replace_with_custom_fn_if_matches_filter(child, replacement_fn, filter_fn, f"{cur_fqn}{name}.",
                                                              device, extra_args)
        if new_child is not child and new_child is not None:
            setattr(model, name, new_child)
    if device is not None:
        model.to(device=device)
    return model


def _is_linear(mod, *args):
    return (isinstance(mod, torch.nn.Linear) and hasattr(mod, "weight")
            and not isinstance(mod, nn.modules.linear.NonDynamicallyQuantizableLinear))


def _linear_extra_repr(self):
    from ao_b200.utils import TorchAOBaseTensor

    w = self.weight
    desc = f"{type(w).__name__}({w._quantization_type()})" if isinstance(w, TorchAOBaseTensor) and hasattr(w, "_quantization_type") else "not quantized"
    return f"in_features={w.shape[1]}, out_features={w.shape[0]}, weight={desc}"


def _set_quantized_param(module, parameter_name, new_tensor):
    setattr(module, parameter_name, torch.nn.Parameter(new_tensor, requires_grad=False))
    module.extra_repr = types.MethodType(_linear_extra_repr, module)
    return module


def quantize_(model: torch.nn.Module, config: AOBaseConfig,
              filter_fn: Optional[Callable[[torch.nn.Module, str], bool]] = _is_linear,
              device: Optional[torch.types.Device] = None):
    """Convert the weight of linear modules in ``model`` according to ``config``, in place; returns None."""
    if isinstance(config, FqnToConfig):
        if filter_fn is not None:   # the default `_is_linear` included, exactly like the reference (quant_api.py:286-290)
            raise ValueError("Custom filter_fn and FqnToConfig were both specified. Only filter_fn=None is supported "
                             "when FqnToConfig is specified.")
        named_modules = dict(model.named_modules())
        for module_fqn, module in named_modules.items():
            if (fqn_matches_fqn_config(module_fqn, config) or _module_param_matches_fqn_config(module, module_fqn, config)
                    or ("_default" in config.fqn_to_config and _is_linear(module))):
                replacement = _fqn_to_config_handler(module, module_fqn, config)
                if device is not None:
                    replacement = replacement.to(device=device)
                if replacement is not module and module_fqn != "":
                    child = module_fqn.split(".")[-1]
                    parent = named_modules[module_fqn.removesuffix(child).removesuffix(".")]
                    setattr(parent, child, replacement)
        _fence_quantized_weights(model)
        return
    if not isinstance(config, AOBaseConfig):
        raise AssertionError("quantize_ expects an AOBaseConfig workflow configuration object")
    filter_fn = _is_linear if filter_fn is None else filter_fn
    if type(config) not in _QUANTIZE_CONFIG_HANDLER:
        raise KeyError(f"no quantize handler registered for {type(config).__name__}")
    handler = _QUANTIZE_CONFIG_HANDLER[type(config)]
    _replace_with_custom_fn_if_matches_filter(model, handler, filter_fn, device=device, extra_args=(config,))
    _fence_quantized_weights(model)


def _fence_quantized_weights(model: torch.nn.Module):
    """The GEMM behind a quantized linear starts loading its weights before it waits for the kernel ahead of it
    (programmatic dependent launch), and the weight quantizers let the next kernels start early.  One
    torch.ops.ao_b200.pdl_fence per device that holds CUDA parameters, on its current stream, makes the weights just
    written complete before the first linear (or the activation quantizer ahead of it) starts."""
    for d in {p.device for p in model.parameters() if p.is_cuda}:
        with torch.cuda.device(d):
            torch.ops.ao_b200.pdl_fence()


# ---------------------------------------------------------------------------------------------
# int4 weight only
# ---------------------------------------------------------------------------------------------
@dataclass
class Int4WeightOnlyConfig(AOBaseConfig):
    """int4 group-wise weight-only quantization.  ``group_size`` in {256,128,64,32}.
    BASELINE uses ``int4_packing_format="tile_packed_to_4d"`` and ``group_size=32``."""

    group_size: int = 128
    set_inductor_config: bool = True
    int4_packing_format: Int4PackingFormat = Int4PackingFormat.PLAIN
    int4_choose_qparams_algorithm: Int4ChooseQParamsAlgorithm = Int4ChooseQParamsAlgorithm.TINYGEMM
    int4_tile_packed_ntile: int = 8
    version: int = 2

    def __post_init__(self):
        assert self.int4_tile_packed_ntile in [8, 16], "int4_tile_packed_ntile must be either 8 or 16"
        # like the reference, the two format fields keep what the caller passed (a plain string stays a string in
        # the config JSON); both are str-Enums, so comparisons with the enum members work either way
        Int4PackingFormat(self.int4_packing_format)                      # validates
        Int4ChooseQParamsAlgorithm(self.int4_choose_qparams_algorithm)   # validates


def _int4_weight_only_quantize_tensor(weight, config: Int4WeightOnlyConfig):
    group_size = config.group_size
    if weight.shape[-1] % group_size != 0:
        # reference :549-553: the layer is left unquantized
        logger.info(f"Skipping quantizing weight with int4 weight only quantization, because the shape of weight "
                    f"{weight.shape} is not compatible with group_size {group_size}")
        return weight
    block_size = list([1 for _ in range(weight.ndim - 1)] + [group_size])
    fmt = Int4PackingFormat(config.int4_packing_format)
    if fmt == Int4PackingFormat.TILE_PACKED_TO_4D:
        assert config.int4_tile_packed_ntile == 8, "ntile 16 is the ROCm variant; CUDA uses 8"
        return Int4TilePackedTo4dTensor.from_hp(weight, block_size,
                                                int4_choose_qparams_algorithm=Int4ChooseQParamsAlgorithm(
                                                    config.int4_choose_qparams_algorithm),
                                                ntile_size=config.int4_tile_packed_ntile)
    raise NotImplementedError(
        f"int4_packing_format={fmt.value!r}: only 'tile_packed_to_4d' has sm_90a kernels in this engine "
        f"(plain/preshuffled need the external mslk library in the reference as well)")


@register_quantize_module_handler(Int4WeightOnlyConfig)
def _int4_weight_only_transform(module: torch.nn.Module, config: Int4WeightOnlyConfig, *,
                                parameter_name: str = "weight") -> torch.nn.Module:
    assert hasattr(module, parameter_name), f"Expected module to have {parameter_name!r}"
    new_weight = _int4_weight_only_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# int8 dynamic activation x int8 weight
# ---------------------------------------------------------------------------------------------
def _validate_granularity_int8(act_granularity, weight_granularity):
    for g in (act_granularity, weight_granularity):
        if not isinstance(g, (PerRow, PerTensor)):
            raise ValueError(f"Unsupported granularity {g}: only PerTensor and PerRow are supported for int8")
        if isinstance(g, PerRow) and g.dim != -1:
            raise ValueError(f"Only PerRow(dim=-1) is supported, got {g}")


@dataclass
class Int8DynamicActivationInt8WeightConfig(AOBaseConfig):
    act_mapping_type: Optional[MappingType] = MappingType.SYMMETRIC
    weight_only_decode: bool = False
    granularity: Optional[Union[Granularity, List[Granularity]]] = PerRow()
    set_inductor_config: bool = True
    version: int = 2
    reduce_range: Optional[bool] = False

    def __post_init__(self):
        if self.version == 1:
            raise ValueError("version 1 of Int8DynamicActivationInt8WeightConfig has been removed, please use version 2")
        a, w = Int8Tensor._normalize_granularity(self.granularity)
        _validate_granularity_int8(a, w)
        assert self.act_mapping_type in (MappingType.SYMMETRIC, MappingType.ASYMMETRIC), (
            "Int8DynamicActivationInt8WeightConfig requires `act_mapping_type` in (MappingType.SYMMETRIC, "
            "MappingType.ASYMMETRIC).")


def _int8_dynamic_activation_int8_weight_quantize_tensor(weight, config):
    a, w = Int8Tensor._normalize_granularity(config.granularity)
    if weight.shape[-1] % 16 != 0 or weight.shape[-2] % 8 != 0:
        # the reference's cuBLAS path needs K % 8 == 0 and N % 8 == 0 and otherwise falls back to a CPU matmul
        # (int8/kernels.py:48-58); this engine has no fallback and its TMA row pitch needs K % 16 == 0: leave the
        # layer unquantized, with a log line, like the int4 / float8 flows do for incompatible shapes
        logger.info(f"Skipping int8 dynamic quantization: weight shape {tuple(weight.shape)} needs in_features % 16 == 0 "
                    f"and out_features % 8 == 0 for the sm_90a kernel")
        return weight
    return Int8Tensor.from_hp(
        weight, granularity=w, mapping_type=MappingType.SYMMETRIC,
        act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=a, mapping_type=config.act_mapping_type,
                                                    reduce_range=bool(config.reduce_range)),
        reduce_range=config.reduce_range)


@register_quantize_module_handler(Int8DynamicActivationInt8WeightConfig)
def _int8_dynamic_activation_int8_weight_transform(module, config, *, parameter_name="weight"):
    assert hasattr(module, parameter_name), f"Expected module to have {parameter_name!r}"
    new_weight = _int8_dynamic_activation_int8_weight_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# int8 static activation x int8 weight
# ---------------------------------------------------------------------------------------------
@dataclass
class Int8StaticActivationInt8WeightConfig(AOBaseConfig):
    """int8 weights with int8 activations quantized by a calibrated (static) scale, e.g. from SmoothQuant (reference
    :918-978).  ``act_quant_scale`` is f32 ``[1, 1]`` (PerTensor) or ``[M, 1]`` (PerRow, one calibration batch);
    ``act_quant_zero_point`` is int8 of the same shape, for ASYMMETRIC activations.  The linear quantizes the
    activations with one kernel (``torch.ops.ao_b200.int8_quantize_static``), fusing the weight's ``act_pre_scale``."""

    act_quant_scale: Optional[torch.Tensor] = None
    act_quant_zero_point: Optional[torch.Tensor] = None
    granularity: Optional[Union[Granularity, List[Granularity]]] = PerRow()
    act_mapping_type: Optional[MappingType] = MappingType.SYMMETRIC
    set_inductor_config: bool = True
    version: int = 1
    reduce_range: Optional[bool] = False

    def __post_init__(self):
        a, w = Int8Tensor._normalize_granularity(self.granularity)
        _validate_granularity_int8(a, w)
        assert self.act_mapping_type in (MappingType.SYMMETRIC, MappingType.ASYMMETRIC), (
            "Int8StaticActivationInt8WeightConfig requires `act_mapping_type` in (MappingType.SYMMETRIC, "
            "MappingType.ASYMMETRIC).")

    def get_act_quant_kwargs(self) -> QuantizeTensorToInt8Kwargs:
        """The activation quantization kwargs the quantized weight carries (reference :964-978)."""
        a, _ = Int8Tensor._normalize_granularity(self.granularity)
        return QuantizeTensorToInt8Kwargs(granularity=a, mapping_type=self.act_mapping_type,
                                          reduce_range=self.reduce_range)


def _int8_static_activation_int8_weight_quantize_tensor(weight, config):
    if config.act_quant_scale is None:
        # the reference fails on `None.detach()` (:1010)
        raise ValueError("Int8StaticActivationInt8WeightConfig needs act_quant_scale (a calibrated activation scale)")
    _, w = Int8Tensor._normalize_granularity(config.granularity)
    if weight.shape[-1] % 16 != 0 or weight.shape[-2] % 8 != 0:
        logger.info(f"Skipping int8 static quantization: weight shape {tuple(weight.shape)} needs in_features % 16 == 0 "
                    f"and out_features % 8 == 0 for the sm_90a kernel")
        return weight
    # the calibrated tensors move to the weight's device here, so the forward (and a CUDA graph capturing it) never
    # copies them from the host
    zp = config.act_quant_zero_point
    return Int8Tensor.from_hp(
        weight, granularity=w, act_quant_kwargs=config.get_act_quant_kwargs(),
        act_quant_scale=config.act_quant_scale.detach().to(weight.device),
        act_quant_zero_point=None if zp is None else zp.detach().to(weight.device),
        reduce_range=config.reduce_range)


@register_quantize_module_handler(Int8StaticActivationInt8WeightConfig)
def _int8_static_activation_int8_weight_transform(module, config, *, parameter_name="weight"):
    assert hasattr(module, parameter_name), f"Expected module to have attribute `{parameter_name}` but not found"
    new_weight = _int8_static_activation_int8_weight_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# int8 weight only
# ---------------------------------------------------------------------------------------------
@dataclass
class Int8WeightOnlyConfig(AOBaseConfig):
    """int8 symmetric weight-only quantization, bf16 activations (reference :703-740).  ``PerRow()`` and
    ``PerTensor()`` run on the sm_90a kernel; ``PerGroup`` is accepted here, as in the reference, and rejected by the
    quantize handler."""

    group_size: Optional[int] = None
    granularity: Optional[Granularity] = PerRow()
    set_inductor_config: bool = True
    version: int = 2

    def __post_init__(self):
        if self.version == 1:
            raise ValueError("version 1 of Int8WeightOnlyConfig has been removed, please use version 2")
        assert self.group_size is None, (
            f"Only support version 2 with group_size=None, got {self.group_size}. "
            f"Use granularity=PerGroup({self.group_size}) instead.")
        assert isinstance(self.granularity, (PerTensor, PerRow, PerGroup)), (
            f"granularity must be PerTensor, PerRow, or PerGroup, but got {self.granularity}")


def _int8_weight_only_quantize_tensor(weight, config):
    if isinstance(config.granularity, PerGroup):
        # the reference serves PerGroup by dequantize-then-mm (int8_tensor.py:338-345): another arithmetic, no kernel here
        raise NotImplementedError(
            f"Int8WeightOnlyConfig(granularity={config.granularity}): PerGroup int8 weights have no sm_90a kernel in "
            f"this engine; use PerRow() or PerTensor()")
    if weight.shape[-1] % 16 != 0:
        # no fallback: the TMA row pitch of the int8 weights needs K % 16 == 0; leave the layer unquantized, with a log
        # line, like the int8 dynamic flow does for its shape rule
        logger.info(f"Skipping int8 weight only quantization: weight shape {tuple(weight.shape)} needs "
                    f"in_features % 16 == 0 for the sm_90a kernel")
        return weight
    return Int8Tensor.from_hp(weight, granularity=config.granularity)


@register_quantize_module_handler(Int8WeightOnlyConfig)
def _int8_weight_only_transform(module, config, *, parameter_name="weight"):
    assert hasattr(module, parameter_name), f"Expected module to have {parameter_name!r}"
    new_weight = _int8_weight_only_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# float8 dynamic activation x float8 weight
# ---------------------------------------------------------------------------------------------
e4m3_dtype = torch.float8_e4m3fn


@dataclass
class Float8DynamicActivationFloat8WeightConfig(AOBaseConfig):
    activation_dtype: torch.dtype = e4m3_dtype
    weight_dtype: torch.dtype = e4m3_dtype
    granularity: Optional[Union[FP8Granularity, List[FP8Granularity]]] = None
    packing_format: Optional[Float8PackingFormat] = Float8PackingFormat.PLAIN
    mm_config: Optional[Float8MMConfig] = None
    activation_value_lb: Optional[float] = None
    activation_value_ub: Optional[float] = None
    kernel_preference: KernelPreference = KernelPreference.AUTO
    set_inductor_config: bool = True
    version: int = 2
    alg_id: int = 0

    def __post_init__(self):
        a, w = _normalize_granularity(self.granularity)
        self.granularity = [a, w]
        default_use_fast_accum = True
        if _granularity_is_a_1_128_w_128_128(self.granularity):
            # reference quant_api.py:1160-1166
            assert self.kernel_preference in (KernelPreference.AUTO, KernelPreference.TORCH), "unimplemented"
            assert self.version >= 2, "unimplemented"
            default_use_fast_accum = False
        if self.mm_config is None:
            self.mm_config = Float8MMConfig(use_fast_accum=default_use_fast_accum)


def _fp8_mm_compat(weight: torch.Tensor) -> bool:
    """Both dims must be multiples of 16, else the layer is skipped (reference quantization/utils.py:663-687)."""
    assert weight.dim() in (2, 3), f"float8 quantization only works for 2/3-D tensors, got {weight.dim()}D"
    out_dim, in_dim = weight.shape[-2:]
    if in_dim % 16 != 0 or out_dim % 16 != 0:
        logger.info(f"Skipping float8 quantization: weight shape {weight.shape} is not compatible with _scaled_mm "
                    f"(both dims must be multiples of 16).")
        return False
    return True


def _fp8_sparse_kernel_compat(weight) -> bool:
    """The 2:4-sparse kernel reads 16-byte rows of compressed codes, K / 2 bytes each: K % 32.  The reference would
    quantize such a layer and fail at its first forward; here it stays unquantized, with a log line, as the other
    float8 flows skip incompatible shapes (_fp8_mm_compat)."""
    if weight.shape[-1] % 32 != 0:
        logger.info(f"Skipping 2:4-sparse float8 quantization: in_features={weight.shape[-1]} is not a multiple of 32; "
                    f"weight shape {tuple(weight.shape)} stays {weight.dtype}")
        return False
    return True


def _float8_dynamic_activation_float8_weight_quantize_tensor(weight, config):
    if config.packing_format == Float8PackingFormat.SPARSE_1D_DATA_1D_METADATA:
        raise NotImplementedError("float8 packing_format SPARSE_1D_DATA_1D_METADATA is the reference's hipSPARSELt "
                                  "(ROCm) format; on sm_90a use SPARSE_2D_DATA_2D_METADATA")
    if config.packing_format not in (Float8PackingFormat.PLAIN, Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA):
        raise NotImplementedError(f"float8 packing_format={config.packing_format}: only PLAIN and "
                                  f"SPARSE_2D_DATA_2D_METADATA are implemented")
    a_gran, w_gran = config.granularity
    if not _fp8_mm_compat(weight):
        return weight
    if config.packing_format == Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA:
        # reference quant_api.py:1233-1245 and the tensor's from_hp assertions
        assert isinstance(w_gran, PerRow), "Sparse packing format only supports per-row quantization"
        assert config.weight_dtype == torch.float8_e4m3fn, "CUTLASS sparse kernel only supports float8_e4m3fn dtype"
        if weight.dtype != torch.bfloat16:
            raise NotImplementedError(f"2:4-sparse float8: bf16 weights only, got {weight.dtype}")
        if not _fp8_sparse_kernel_compat(weight):
            return weight
        act_quant_kwargs = QuantizeTensorToFloat8Kwargs(config.activation_dtype, a_gran,
                                                        hp_value_lb=config.activation_value_lb,
                                                        hp_value_ub=config.activation_value_ub,
                                                        kernel_preference=config.kernel_preference)
        return Float8Sparse2x4_2DData2DMetadataTensor.from_hp(weight, float8_dtype=config.weight_dtype,
                                                              granularity=w_gran, act_quant_kwargs=act_quant_kwargs)
    if isinstance(w_gran, PerRow):
        assert weight.dtype == torch.bfloat16, "PerRow quantization only works for bfloat16 precision input weight"
    act_quant_kwargs = QuantizeTensorToFloat8Kwargs(config.activation_dtype, a_gran, hp_value_lb=config.activation_value_lb,
                                                    hp_value_ub=config.activation_value_ub,
                                                    kernel_preference=config.kernel_preference)
    return Float8Tensor.from_hp(weight, float8_dtype=config.weight_dtype, granularity=w_gran, mm_config=config.mm_config,
                                kernel_preference=config.kernel_preference, act_quant_kwargs=act_quant_kwargs)


@register_quantize_module_handler(Float8DynamicActivationFloat8WeightConfig)
def _float8_dynamic_activation_float8_weight_transform(module, config, *, parameter_name="weight"):
    if torch.cuda.is_available():
        require_sm90()
    assert hasattr(module, parameter_name), f"Expected module to have {parameter_name!r}"
    new_weight = _float8_dynamic_activation_float8_weight_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# float8 weight only
# ---------------------------------------------------------------------------------------------
@dataclass
class Float8WeightOnlyConfig(AOBaseConfig):
    """float8 symmetric weight-only quantization, bf16 activations (reference :1031-1060).  e4m3 weights with
    ``PerRow()`` (the default) or ``PerTensor()`` scales run on the sm_90a kernel; ``PerGroup`` is accepted here, as in
    the reference, and rejected by the quantize handler, as is ``weight_dtype=torch.float8_e5m2``.  Weights that are
    not bf16 are left unquantized: the reference computes their linear in their own dtype."""

    weight_dtype: torch.dtype = e4m3_dtype
    set_inductor_config: bool = True
    version: int = 2
    granularity: Granularity = None  # type: ignore[assignment]

    def __post_init__(self):
        if self.granularity is None:
            self.granularity = PerRow()
        assert isinstance(self.granularity, (PerTensor, PerRow, PerGroup)), (
            f"granularity must be PerTensor, PerRow, or PerGroup, got {type(self.granularity)}")


def _float8_weight_only_quantize_tensor(weight, config):
    assert config.version == 2, f"Unexpected version: {config.version}"
    if isinstance(config.granularity, PerGroup):
        # [N, K / g] scales: the per-row box of one 128-k chunk is under TMA's 16-byte minimum for g = 64 and 128
        raise NotImplementedError(
            f"Float8WeightOnlyConfig(granularity={config.granularity}): PerGroup float8 weights have no sm_90a kernel "
            f"in this engine; use PerRow() or PerTensor()")
    if config.weight_dtype != e4m3_dtype:
        raise NotImplementedError(
            f"Float8WeightOnlyConfig(weight_dtype={config.weight_dtype}): only torch.float8_e4m3fn weights have an "
            f"sm_90a kernel in this engine")
    if weight.shape[-1] % 16 != 0:
        # no fallback: the TMA row pitch of the e4m3 weights needs K % 16 == 0; leave the layer unquantized, with a log
        # line, like the int8 weight-only flow does
        logger.info(f"Skipping float8 weight only quantization: weight shape {tuple(weight.shape)} needs "
                    f"in_features % 16 == 0 for the sm_90a kernel")
        return weight
    if weight.dtype != torch.bfloat16:
        # the reference dequantizes into the weight's dtype and multiplies in it; the kernel computes in bf16 only
        logger.info(f"Skipping float8 weight only quantization: weight dtype {weight.dtype} needs to be "
                    f"torch.bfloat16 for the sm_90a kernel")
        return weight
    return Float8Tensor.from_hp(weight, float8_dtype=config.weight_dtype, granularity=config.granularity)


@register_quantize_module_handler(Float8WeightOnlyConfig)
def _float8_weight_only_transform(module, config, *, parameter_name="weight"):
    assert hasattr(module, parameter_name), f"Expected module to have {parameter_name!r}"
    new_weight = _float8_weight_only_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)


# ---------------------------------------------------------------------------------------------
# FqnToConfig (per-module / per-parameter configs; used by HF TorchAoConfig)
# ---------------------------------------------------------------------------------------------
@dataclass
class FqnToConfig(AOBaseConfig):
    """Ordered map key -> config (or None). Key: exact fqn of a module/parameter, ``re:<regex>``, or ``_default``."""

    fqn_to_config: "OrderedDict[str, Optional[AOBaseConfig]]" = field(default_factory=OrderedDict)
    module_fqn_to_config: "OrderedDict[str, Optional[AOBaseConfig]]" = field(default_factory=OrderedDict)
    version: int = 1

    def __post_init__(self):
        if len(self.module_fqn_to_config) > 0 and len(self.fqn_to_config) > 0 and \
                dict(self.module_fqn_to_config) != dict(self.fqn_to_config):
            raise ValueError("`fqn_to_config` and `module_fqn_to_config` are both specified and are not equal!")
        if len(self.module_fqn_to_config) > 0:
            self.fqn_to_config = self.module_fqn_to_config
        if len(self.fqn_to_config) > 0:
            self.module_fqn_to_config = self.fqn_to_config
        if any(k.startswith("re:") for k in self.fqn_to_config) and "_default" in self.fqn_to_config:
            logger.warning("`_default` with regex keys: regexes are tried first, `_default` is the fallback")


ModuleFqnToConfig = FqnToConfig


def fqn_matches_fqn_config(fqn: str, config: FqnToConfig) -> bool:
    if fqn in config.fqn_to_config:
        assert not fqn.startswith("re:"), f"Error: Exact match but regex {fqn} specified."
        return True
    return any(p.startswith("re:") and re.fullmatch(p[3:], fqn) for p in config.fqn_to_config)


def _top_level_params(module, fqn):
    for name, param in module.named_parameters():
        if name in dir(module):
            yield name, param, (f"{fqn}.{name}" if fqn else name)


def _module_param_matches_fqn_config(module, fqn, config) -> bool:
    return any(fqn_matches_fqn_config(pfqn, config) for _, _, pfqn in _top_level_params(module, fqn))


def _apply(module, c, parameter_name=None):
    if c is None:
        return module
    handler = _QUANTIZE_CONFIG_HANDLER[type(c)]
    return handler(module, c) if parameter_name is None else handler(module, c, parameter_name=parameter_name)


def _fqn_to_config_handler(module: torch.nn.Module, fqn: str, config: FqnToConfig):
    """Same order as the reference (quant_api.py:1638-1701): exact parameter fqns first (several may match; a `None`
    config takes the parameter out of the regex pass), then -- only when no parameter matched -- the exact module
    fqn; then EVERY regex that fully matches a remaining top-level parameter, in dict order; then -- only when still
    nothing matched -- the first module-fqn regex, and finally `_default`."""
    found = False
    remaining = []
    for name, _, pfqn in _top_level_params(module, fqn):
        if pfqn in config.fqn_to_config:
            found = True
            c = config.fqn_to_config[pfqn]
            if c is not None:
                module = _apply(module, c, parameter_name=name)
        else:
            remaining.append((name, pfqn))
    if not found and fqn in config.fqn_to_config:
        return _apply(module, config.fqn_to_config[fqn])
    for name, pfqn in remaining:
        for pat, c in config.fqn_to_config.items():
            if pat.startswith("re:") and re.fullmatch(pat[3:], pfqn):
                found = True
                module = _apply(module, c, parameter_name=name)
    if found:
        return module
    for pat, c in config.fqn_to_config.items():
        if pat.startswith("re:") and re.fullmatch(pat[3:], fqn):
            return _apply(module, c)
    if "_default" in config.fqn_to_config and _is_linear(module):
        return _apply(module, config.fqn_to_config["_default"])
    return module
