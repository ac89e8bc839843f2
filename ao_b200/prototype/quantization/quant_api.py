"""Float8StaticActivationFloat8WeightConfig: e4m3 weights with calibrated (static) per-tensor or per-row e4m3
activation scales, and an optional calibrated output fake-quant.

Same name, dataclass fields, defaults, ``__post_init__`` and ``get_act_quant_kwargs()`` as
torchao/prototype/quantization/quant_api.py:222-324; handler :481-679.  Differences, all deliberate:
  * only the direct path (``step=None`` with ``act_quant_scale``) is served.  ``step="prepare"`` / ``"convert"``
    (the observer flow, ``Float8ObservedLinear``) and the ``Softmax`` fake-quant modules raise NotImplementedError;
  * the calibrated scales move to the weight's device at quantize time, so the forward (and a CUDA graph of it) never
    copies them from the host;
  * a weight that fails the ``_scaled_mm`` shape rule (both dims multiples of 16) stays unquantized with a log line,
    as for Float8DynamicActivationFloat8WeightConfig;
  * global inductor flags are not touched (``set_inductor_config`` is accepted and ignored).
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Optional

import torch

from ao_b200._native import require_sm90
from ao_b200.core.config import AOBaseConfig
from ao_b200.float8.inference import Float8MMConfig
from ao_b200.prototype.mx_formats.inference_workflow import QuantizationStep
from ao_b200.prototype.quantization.float8_static_quant.prototype_float8_tensor import PrototypeFloat8Tensor
from ao_b200.quantization.granularity import Granularity, PerRow, PerTensor
from ao_b200.quantization.quant_api import _fp8_mm_compat, _set_quantized_param
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.common.quantize_tensor_kwargs import QuantizeTensorKwargs
from ao_b200.quantization.quantize_.workflows import QuantizeTensorToFloat8Kwargs
from ao_b200.quantization.transform_module import register_quantize_module_handler

__all__ = ["Float8StaticActivationFloat8WeightConfig"]
logger = logging.getLogger(__name__)
e4m3_dtype = torch.float8_e4m3fn


@dataclass
class Float8StaticActivationFloat8WeightConfig(AOBaseConfig):
    """e4m3 weights and e4m3 activations quantized with a calibrated scale ``act_quant_scale``: f32 ``[1, 1]``
    (PerTensor, the default granularity) or ``[M, 1]`` (PerRow, one calibration batch).  ``output_act_quant_scale``
    (same shapes) adds the output fake-quant: the linear's bf16 output is quantized to e4m3 with it and dequantized.
    The linear is two kernels: ``torch.ops.ao_b200.fp8_quantize_static`` and the e4m3 GEMM, which applies the output
    fake-quant in its epilogue."""

    step: Optional[QuantizationStep] = None
    act_quant_scale: Optional[torch.Tensor] = None
    activation_dtype: torch.dtype = e4m3_dtype
    weight_dtype: torch.dtype = e4m3_dtype
    granularity: Optional[Granularity] = None
    mm_config: Optional[Float8MMConfig] = None
    kernel_preference: KernelPreference = KernelPreference.AUTO
    set_inductor_config: bool = True
    quantize_and_dequantize_output: bool = False
    output_act_quant_scale: Optional[torch.Tensor] = None

    def __post_init__(self):
        if self.mm_config is None:
            self.mm_config = Float8MMConfig(use_fast_accum=True)
        # string step values are allowed for convenience (reference :292-300)
        if self.step is not None:
            if isinstance(self.step, str):
                self.step = self.step.lower()
            all_step_values = [s.value for s in QuantizationStep]
            if self.step not in all_step_values and self.step not in list(QuantizationStep):
                raise ValueError(f"{self.step} is not one of {all_step_values}")

    def get_act_quant_kwargs(self) -> QuantizeTensorKwargs:
        """The activation quantization kwargs the quantized weight carries (reference :310-324)."""
        granularity = self.granularity if self.granularity is not None else PerTensor()
        return QuantizeTensorToFloat8Kwargs(float8_dtype=self.activation_dtype, granularity=granularity,
                                            mm_config=self.mm_config, kernel_preference=self.kernel_preference)


def _float8_static_activation_float8_weight_quantize_tensor(weight, config):
    if config.act_quant_scale is None:
        raise ValueError("When step is None, act_quant_scale must be provided for direct quantization. "
                         "Alternatively, use step='prepare' followed by step='convert' for observer-based flow.")
    granularity = config.granularity if config.granularity is not None else PerTensor()
    if not isinstance(granularity, (PerTensor, PerRow)) or config.activation_dtype != e4m3_dtype \
            or config.weight_dtype != e4m3_dtype:
        raise NotImplementedError(f"Float8StaticActivationFloat8WeightConfig: PerTensor or PerRow granularity with "
                                  f"e4m3 activations and weights only, got {granularity}, {config.activation_dtype} "
                                  f"activations and {config.weight_dtype} weights")
    if not _fp8_mm_compat(weight):
        return weight
    act_quant_kwargs = config.get_act_quant_kwargs()
    out_scale = config.output_act_quant_scale
    # the calibrated tensors move to the weight's device here, so the forward (and a CUDA graph capturing it) never
    # copies them from the host
    return PrototypeFloat8Tensor.from_hp(
        weight, float8_dtype=config.weight_dtype, granularity=granularity, mm_config=config.mm_config,
        kernel_preference=config.kernel_preference, act_quant_kwargs=act_quant_kwargs,
        act_quant_scale=config.act_quant_scale.detach().to(weight.device),
        output_act_quant_scale=None if out_scale is None else out_scale.detach().to(weight.device),
        output_act_quant_kwargs=None if out_scale is None else config.get_act_quant_kwargs())


@register_quantize_module_handler(Float8StaticActivationFloat8WeightConfig)
def _float8_static_activation_float8_weight_transform(module, config, *, parameter_name="weight"):
    if config.step is not None:
        raise NotImplementedError(f"Float8StaticActivationFloat8WeightConfig(step={config.step!r}): the observer flow "
                                  f"is not implemented; pass a calibrated act_quant_scale with step=None")
    if torch.cuda.is_available():
        require_sm90()
    assert hasattr(module, parameter_name), f"Expected module to have attribute `{parameter_name}` but not found"
    new_weight = _float8_static_activation_float8_weight_quantize_tensor(getattr(module, parameter_name), config)
    return _set_quantized_param(module, parameter_name, new_weight)
