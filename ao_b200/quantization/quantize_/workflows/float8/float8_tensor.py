"""e4m3 rowwise-scaled weight, dynamic rowwise activation quant, wgmma e4m3 GEMM.

Attribute names / order match torchao's Float8Tensor
(torchao/quantization/quantize_/workflows/float8/float8_tensor.py:105-113).  The linear replaces
``_float8_addmm_impl -> addmm_float8_unwrapped_inference -> torch._scaled_mm``
(:338-469, float8/inference.py:86-123) with two launches: the per-token quantizer and the GEMM with
a fused ``acc * s_x[m] * s_w[n] + bias -> bf16`` epilogue.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.float8.inference import FP8Granularity, Float8MMConfig, _is_rowwise_scaled, _is_tensorwise_scaled
from ao_b200.quantization.granularity import PerRow, PerTensor
from ao_b200.quantization.quant_primitives import (
    choose_scale_float8, dequantize_affine_float8, quantize_affine_float8)
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.common.quantize_tensor_kwargs import QuantizeTensorKwargs
from ao_b200.quantization.utils import get_block_size
from ao_b200.utils import TorchAOBaseTensor, fill_defaults, rows_for_kernel

__all__ = ["Float8Tensor", "QuantizeTensorToFloat8Kwargs"]
aten = torch.ops.aten


@dataclass
class QuantizeTensorToFloat8Kwargs(QuantizeTensorKwargs):
    float8_dtype: torch.dtype = torch.float8_e4m3fn
    granularity: FP8Granularity = PerRow()
    mm_config: Optional[Float8MMConfig] = None
    hp_value_lb: Optional[float] = None
    hp_value_ub: Optional[float] = None
    kernel_preference: KernelPreference = KernelPreference.AUTO


class Float8Tensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale"]
    tensor_attribute_names = []
    optional_tensor_attribute_names = ["block_size", "mm_config", "act_quant_kwargs", "kernel_preference", "dtype"]

    def __new__(cls, qdata, scale, block_size: Optional[List[int]] = None, mm_config: Optional[Float8MMConfig] = None,
                act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None,
                kernel_preference: KernelPreference = KernelPreference.AUTO, dtype: Optional[torch.dtype] = None):
        return torch.Tensor._make_wrapper_subclass(cls, qdata.shape, device=qdata.device, dtype=dtype, requires_grad=False)

    def __init__(self, qdata, scale, block_size=None, mm_config=None, act_quant_kwargs=None,
                 kernel_preference=KernelPreference.AUTO, dtype=None):
        super().__init__()
        self.qdata = qdata
        self.scale = scale
        self.block_size = block_size
        self.mm_config = mm_config
        self.act_quant_kwargs = act_quant_kwargs
        self.kernel_preference = kernel_preference

    def _quantization_type(self):
        return (f"{self.act_quant_kwargs=}, {self.block_size=}, {self.mm_config=}, {self.scale.shape=}, "
                f"{self.kernel_preference=}")

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        return dequantize_affine_float8(self.qdata, self.scale, output_dtype or self.dtype)

    @classmethod
    def from_hp(cls, hp_tensor: torch.Tensor, float8_dtype: torch.dtype = torch.float8_e4m3fn,
                granularity: FP8Granularity = PerRow(), mm_config: Optional[Float8MMConfig] = None,
                hp_value_lb: Optional[float] = None, hp_value_ub: Optional[float] = None,
                kernel_preference: KernelPreference = KernelPreference.AUTO,
                act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None):
        block_size = list(get_block_size(hp_tensor.shape, granularity))
        fast = (hp_tensor.is_cuda and hp_tensor.dtype == torch.bfloat16 and float8_dtype == torch.float8_e4m3fn
                and isinstance(granularity, PerRow) and granularity.dim in (-1, hp_tensor.dim() - 1)
                and hp_value_lb is None and hp_value_ub is None and hp_tensor.shape[-1] % 8 == 0
                and kernel_preference in (KernelPreference.AUTO, KernelPreference.B200))
        if fast:
            x2 = rows_for_kernel(hp_tensor.reshape(-1, hp_tensor.shape[-1]))
            data, scale = torch.ops.ao_b200.fp8_quantize_rowwise(x2)
            data = data.reshape(hp_tensor.shape)
            scale = scale.reshape(*hp_tensor.shape[:-1], 1)
        else:
            scale = choose_scale_float8(hp_tensor, block_size, float8_dtype, hp_value_lb, hp_value_ub)
            data = quantize_affine_float8(hp_tensor, scale, float8_dtype)
        return cls(data, scale, block_size=block_size, mm_config=mm_config, act_quant_kwargs=act_quant_kwargs,
                   kernel_preference=kernel_preference, dtype=hp_tensor.dtype)


implements = Float8Tensor.implements
implements_torch_function = Float8Tensor.implements_torch_function


def _float8_linear_impl(input_tensor, weight_tensor: Float8Tensor, bias):
    """weight_tensor: [N, K] e4m3 with scale [N, 1] (rowwise) or [1,1] (tensorwise)."""
    act_quant_kwargs = weight_tensor.act_quant_kwargs
    N, K = weight_tensor.shape[-2], weight_tensor.shape[-1]
    out_shape = (*input_tensor.shape[:-1], N)
    if act_quant_kwargs is None:
        # weight-only float8: outside the north-star path; semantics = matmul with dequantized weight
        assert not isinstance(input_tensor, TorchAOBaseTensor), "Expecting input_tensor to be unquantized"
        raise NotImplementedError(
            "Float8 weight-only linear is outside this engine's scope (SURVEY §8); use "
            "Float8DynamicActivationFloat8WeightConfig")
    assert not isinstance(input_tensor, TorchAOBaseTensor), "input tensor was already quantized"
    gran = act_quant_kwargs.granularity
    w_rowwise = _is_rowwise_scaled(weight_tensor.block_size, weight_tensor.shape)
    w_tensorwise = _is_tensorwise_scaled(weight_tensor.block_size, weight_tensor.shape) and not w_rowwise
    if w_rowwise:
        assert isinstance(gran, PerRow), "Input tensor must be rowwise block size"
    x2 = input_tensor.reshape(-1, K)
    if x2.shape[0] == 0:
        return input_tensor.new_empty(out_shape)
    xq_t = Float8Tensor.from_hp(x2, act_quant_kwargs.float8_dtype, gran, act_quant_kwargs.mm_config,
                                act_quant_kwargs.hp_value_lb, act_quant_kwargs.hp_value_ub,
                                act_quant_kwargs.kernel_preference)
    M = x2.shape[0]
    x_scale = xq_t.scale.reshape(-1)
    if x_scale.numel() == 1:
        x_scale = x_scale.expand(M)
    w_scale = weight_tensor.scale.reshape(-1)
    if w_tensorwise or w_scale.numel() == 1:
        w_scale = w_scale.reshape(1).expand(N)
    y = torch.ops.ao_b200.fp8_rowwise_linear(xq_t.qdata.contiguous(), x_scale.contiguous().float(),
                                             weight_tensor.qdata.contiguous(), w_scale.contiguous().float(), bias)
    return y.reshape(out_shape).to(input_tensor.dtype)


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    input_tensor, weight_tensor, bias = args[0], args[1], args[2] if len(args) > 2 else None
    return _float8_linear_impl(input_tensor, weight_tensor, bias)


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    assert step == 1 and dim in (0, 1)
    qd = aten.slice.Tensor(self.qdata, dim, start, end, step)
    sc = self.scale
    if sc.numel() > 1 and sc.shape[dim] == self.qdata.shape[dim]:
        sc = aten.slice.Tensor(sc, dim, start, end, step)
    bs = list(self.block_size)
    if bs[dim] > qd.shape[dim]:
        bs[dim] = qd.shape[dim]
    return Float8Tensor(qd, sc, bs, self.mm_config, self.act_quant_kwargs, self.kernel_preference, self.dtype)


@implements(aten.transpose.int)
def _(func, types, args, kwargs):
    """A view with qdata, scale and block_size swapped (float8_tensor.py:842-860): how a 3-D expert weight [E, N, K]
    reaches torch._grouped_mm as mat_b [E, K, N]."""
    self, dim0, dim1 = args
    bs = list(self.block_size)
    bs[dim0], bs[dim1] = bs[dim1], bs[dim0]
    new = Float8Tensor(self.qdata.transpose(dim0, dim1), self.scale.transpose(dim0, dim1), bs, self.mm_config,
                       self.act_quant_kwargs, self.kernel_preference, self.dtype)
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements(aten._grouped_mm.default)
def _(func, types, args, kwargs):
    """torch._grouped_mm(x, W.transpose(-2, -1), offs=offs) with a rowwise Float8Tensor expert weight W [E, N, K]
    (the reference's handler, float8_tensor.py:1085-1122): the routed tokens are quantized per row and the grouped
    GEMM runs on the stored qdata with w_scale[e, n].  Only the 2-D x 3-D form with PerRow activations."""
    mat_a, mat_b = args[0], args[1]
    offs = args[2] if len(args) > 2 else kwargs.get("offs", None)
    assert isinstance(mat_b, Float8Tensor)
    assert offs is not None, "offs is required for _grouped_mm"
    assert mat_b.qdata.stride(-2) < mat_b.qdata.stride(-1), "mat_b must be the transposed [E, N, K] weight"
    act_quant_kwargs = mat_b.act_quant_kwargs
    if act_quant_kwargs is None:
        raise NotImplementedError("Float8 weight-only _grouped_mm is outside this engine's scope; use "
                                  "Float8DynamicActivationFloat8WeightConfig")
    if not isinstance(act_quant_kwargs.granularity, PerRow):
        raise NotImplementedError(f"_grouped_mm only supports PerRow granularity, got {act_quant_kwargs.granularity}")
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"_grouped_mm: only 2-D mat_a x 3-D mat_b, got {mat_a.dim()}-D x {mat_b.dim()}-D")
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    assert bias is None, "_grouped_mm with bias is not supported"
    E, K, N = mat_b.shape
    assert mat_a.shape[-1] == K, f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}"
    xq_t = Float8Tensor.from_hp(mat_a, act_quant_kwargs.float8_dtype, act_quant_kwargs.granularity,
                                act_quant_kwargs.mm_config, act_quant_kwargs.hp_value_lb, act_quant_kwargs.hp_value_ub,
                                act_quant_kwargs.kernel_preference)
    wq = mat_b.qdata.transpose(-2, -1)   # back to the stored [E, N, K]
    y = torch.ops.ao_b200.fp8_rowwise_grouped_mm(xq_t.qdata.contiguous(), xq_t.scale.reshape(-1).float().contiguous(),
                                                 wq.contiguous(), mat_b.scale.reshape(E, N).float().contiguous(),
                                                 offs.to(torch.int32))
    return y.to(mat_a.dtype)


Float8Tensor.__module__ = "ao_b200.quantization"
torch.serialization.add_safe_globals([Float8Tensor, QuantizeTensorToFloat8Kwargs, Float8MMConfig])
