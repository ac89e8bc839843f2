"""MX / NVFP4 inference configs + handlers (reference: torchao/prototype/mx_formats/inference_workflow.py:
MXDynamicActivationMXWeightConfig :102-112, NVFP4DynamicActivationNVFP4WeightConfig :221-223,
NVFP4WeightOnlyConfig :370, handlers :119-163, :230-353, :373-400)."""
from __future__ import annotations

import types
from dataclasses import dataclass
from enum import Enum
from typing import Optional

import logging

import torch

from ao_b200._native import require_sm90
from ao_b200.core.config import AOBaseConfig
from ao_b200.quantization.quant_api import _set_quantized_param
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.transform_module import register_quantize_module_handler

from .mx_tensor import MXTensor, QuantizeTensorToMXKwargs, ScaleCalculationMode
from .nvfp4_tensor import (NVFP4Tensor, QuantizeTensorToFloat8ActKwargs, QuantizeTensorToNVFP4Kwargs,
                           per_tensor_amax_to_scale)


class QuantizationStep(str, Enum):
    PREPARE = "prepare"
    CONVERT = "convert"


logger = logging.getLogger(__name__)


@dataclass
class MXDynamicActivationMXWeightConfig(AOBaseConfig):
    block_size: int = 32
    activation_dtype: torch.dtype = torch.float8_e4m3fn
    weight_dtype: torch.dtype = torch.float8_e4m3fn
    kernel_preference: KernelPreference = KernelPreference.AUTO
    scaling_mode: ScaleCalculationMode = ScaleCalculationMode.RCEIL

    def __post_init__(self):
        assert self.activation_dtype == self.weight_dtype, "For now - we only support matching input/weight dtypes."


@register_quantize_module_handler(MXDynamicActivationMXWeightConfig)
def _mx_inference_linear_transform(module, config: MXDynamicActivationMXWeightConfig, *, parameter_name="weight"):
    weight = getattr(module, parameter_name)
    assert weight.dtype == torch.bfloat16, f"Only supporting bf16 out dtype for now, got {weight.dtype}"
    act = QuantizeTensorToMXKwargs(elem_dtype=config.activation_dtype, block_size=config.block_size,
                                   kernel_preference=config.kernel_preference, is_swizzled_scales=True,
                                   scaling_mode=config.scaling_mode)
    qw = MXTensor.to_mx(weight.contiguous(), config.weight_dtype, block_size=config.block_size,
                        kernel_preference=config.kernel_preference, act_quant_kwargs=act, is_swizzled_scales=True,
                        scaling_mode=config.scaling_mode)
    return _set_quantized_param(module, parameter_name, qw)


def _check_nvfp4_shape(weight):
    if weight.shape[-2] % 16 != 0 or weight.shape[-1] % 16 != 0:
        raise RuntimeError(f"NVFP4 only supports weight shape with last 2 dims divisible by 16, got {weight.shape}")


def _nvfp4_kernel_compat(weight, k_multiple: int) -> bool:
    """The sm_90a kernels stream K in chunks whose block-scale tiles must exist in full: K % 256 for nvfp4 x nvfp4
    (lowp_linear.cu), K % 128 for the weight-only / fp8-activation kernel (ts_gemm.cuh).  The reference accepts any
    K % 16 (inference_workflow.py:248-251); such a layer is left unquantized here, with a log line, the way the int4
    and float8 flows skip incompatible shapes (quant_api.py:549-553, quantization/utils.py:663-687) -- never
    quantized into something whose first forward raises."""
    if weight.shape[-1] % k_multiple != 0:
        logger.info(f"Skipping NVFP4 quantization: in_features={weight.shape[-1]} is not a multiple of {k_multiple} "
                    f"(kernel K-chunk); weight shape {tuple(weight.shape)} stays {weight.dtype}")
        return False
    return True


def _nvfp4_expert_rows_compat(weight) -> bool:
    """The grouped expert GEMM reads each expert's weights and blocked scales as whole 128-row blocks of the stacked
    [E * N, ..] tensors (ts_gemm.cuh, Grouped<Nvfp4Fmt>), so it needs out_features % 128 == 0; the reference's 3-D
    blocked scale layout has the same requirement (to_blocked over E * N rows).  Other layers stay unquantized."""
    if weight.shape[-2] % 128 != 0:
        logger.info(f"Skipping NVFP4 quantization: expert out_features={weight.shape[-2]} is not a multiple of 128; "
                    f"weight shape {tuple(weight.shape)} stays {weight.dtype}")
        return False
    return True


@dataclass
class NVFP4DynamicActivationNVFP4WeightConfig(AOBaseConfig):
    use_triton_kernel: bool = True   # accepted for compatibility; the CUDA quantizer is always used
    use_dynamic_per_tensor_scale: bool = True
    step: Optional[QuantizationStep] = None

    def __post_init__(self):
        if isinstance(self.step, str):
            self.step = QuantizationStep(self.step)
        if self.step is not None:
            raise NotImplementedError("observer-based static calibration (step=prepare/convert) is out of scope (SURVEY §2.1)")


@register_quantize_module_handler(NVFP4DynamicActivationNVFP4WeightConfig)
def _nvfp4_inference_linear_transform(module, config, *, parameter_name="weight"):
    weight = getattr(module, parameter_name)
    _check_nvfp4_shape(weight)
    if torch.cuda.is_available():
        require_sm90()
    if weight.dim() == 3:
        # MoE expert weights [E, N, K] for torch._grouped_mm: one per-tensor scale per expert [E, 1, 1] (reference
        # :307-319).  The grouped kernel quantizes each expert's routed tokens with their own dynamic scale, so the
        # static form has nothing to run on (the reference's handler would fail at the first forward)
        if not config.use_dynamic_per_tensor_scale:
            raise NotImplementedError("NVFP4DynamicActivationNVFP4WeightConfig on 3-D (MoE) weights needs "
                                      "use_dynamic_per_tensor_scale=True")
        if not _nvfp4_kernel_compat(weight, 128) or not _nvfp4_expert_rows_compat(weight):
            return module
        pts = per_tensor_amax_to_scale(torch.amax(torch.abs(weight), dim=(1, 2))).view(-1, 1, 1)
    else:
        assert weight.dim() == 2, f"NVFP4: 2-D or 3-D weights only, got {weight.dim()}-D"
        if not _nvfp4_kernel_compat(weight, 256):
            return module
        pts = per_tensor_amax_to_scale(torch.max(torch.abs(weight))) if config.use_dynamic_per_tensor_scale else None
    act = QuantizeTensorToNVFP4Kwargs(use_dynamic_per_tensor_scale=config.use_dynamic_per_tensor_scale,
                                      use_triton_kernel=config.use_triton_kernel, is_swizzled_scales=True)
    qw = NVFP4Tensor.to_nvfp4(weight.contiguous(), per_tensor_scale=pts, is_swizzled_scales=True,
                              use_triton_kernel=False, act_quant_kwargs=act)
    qw.use_triton_kernel = config.use_triton_kernel
    return _set_quantized_param(module, parameter_name, qw)


@dataclass
class NVFP4WeightOnlyConfig(AOBaseConfig):
    use_dynamic_per_tensor_scale: bool = True


@register_quantize_module_handler(NVFP4WeightOnlyConfig)
def _nvfp4_weight_only_linear_transform(module, config, *, parameter_name="weight"):
    weight = getattr(module, parameter_name)
    assert weight.dim() == 2, "3D weights not yet supported in this workflow"
    _check_nvfp4_shape(weight)
    if not _nvfp4_kernel_compat(weight, 128):
        return module
    pts = per_tensor_amax_to_scale(torch.max(torch.abs(weight))) if config.use_dynamic_per_tensor_scale else None
    qw = NVFP4Tensor.to_nvfp4(weight.contiguous(), per_tensor_scale=pts, is_swizzled_scales=True, act_quant_kwargs=None)
    return _set_quantized_param(module, parameter_name, qw)


@dataclass
class NVFP4WeightFloat8ActivationConfig(AOBaseConfig):
    """NVFP4 weights x dynamic e4m3 per-token activations (BASELINE config 5).  The reference has no
    such config (SURVEY §0-5); semantics are defined as
    ``F.linear(dequant(Float8Tensor.from_hp(x, PerRow())), NVFP4Tensor.dequantize())``."""

    use_dynamic_per_tensor_scale: bool = True


@register_quantize_module_handler(NVFP4WeightFloat8ActivationConfig)
def _nvfp4_weight_fp8_act_transform(module, config, *, parameter_name="weight"):
    weight = getattr(module, parameter_name)
    assert weight.dim() == 2
    _check_nvfp4_shape(weight)
    if not _nvfp4_kernel_compat(weight, 128):
        return module
    pts = per_tensor_amax_to_scale(torch.max(torch.abs(weight))) if config.use_dynamic_per_tensor_scale else None
    qw = NVFP4Tensor.to_nvfp4(weight.contiguous(), per_tensor_scale=pts, is_swizzled_scales=True,
                              act_quant_kwargs=QuantizeTensorToFloat8ActKwargs())
    return _set_quantized_param(module, parameter_name, qw)
