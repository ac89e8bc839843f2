"""NVFP4 (e2m1 data, e4m3 block-16 scales, fp32 per-tensor scale) on Hopper wgmma (bf16, exactly dequantised operands).

Attribute names/order match torchao's NVFP4Tensor (torchao/prototype/mx_formats/nvfp4_tensor.py:69-79):
``qdata, scale | block_size, orig_dtype | per_tensor_scale?, act_per_tensor_scale? |
is_swizzled_scales, use_triton_kernel, act_quant_kwargs``.  ``qdata`` is uint8 [.., K/2] with even k
in the LOW nibble (kernels.py:155-160).  The dynamic linear replaces
``nvfp4_linear -> _addmm_nvfp4_dispatch -> torch._scaled_mm`` + separate per-tensor-scale and bias
kernels (:487-619) with: amax -> fused quantize+swizzle -> one GEMM with (pts_a*pts_b, bias) in the
epilogue.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from ao_b200.quantization.quantize_.common.quantize_tensor_kwargs import QuantizeTensorKwargs
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.utils import TorchAOBaseTensor, fill_defaults, rows_for_kernel

from .utils import from_blocked, slice_qdata_and_scale

aten = torch.ops.aten
F4_E2M1_MAX = 6.0
F8E4M3_MAX = 448.0
__all__ = ["NVFP4Tensor", "QuantizeTensorToNVFP4Kwargs", "per_tensor_amax_to_scale"]

_E2M1 = [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, -0.0, -0.5, -1.0, -1.5, -2.0, -3.0, -4.0, -6.0]


def per_tensor_amax_to_scale(amax: torch.Tensor) -> torch.Tensor:
    """amax / (448 * 6) in fp32 (reference :756-769)."""
    return amax.to(torch.float32) / (F8E4M3_MAX * F4_E2M1_MAX)


@dataclass
class QuantizeTensorToNVFP4Kwargs(QuantizeTensorKwargs):
    block_size: int = 16
    is_swizzled_scales: bool = False
    use_triton_kernel: bool = False
    use_dynamic_per_tensor_scale: bool = False


class NVFP4Tensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale"]
    tensor_attribute_names = ["block_size", "orig_dtype"]
    optional_tensor_data_names = ["per_tensor_scale", "act_per_tensor_scale"]
    optional_tensor_attribute_names = ["is_swizzled_scales", "use_triton_kernel", "act_quant_kwargs"]

    def __new__(cls, qdata, scale, block_size, orig_dtype, per_tensor_scale=None, act_per_tensor_scale=None,
                is_swizzled_scales=False, use_triton_kernel=False, act_quant_kwargs=None):
        size = list(qdata.shape)
        size[-1] *= 2
        return torch.Tensor._make_wrapper_subclass(cls, size, dtype=orig_dtype, device=qdata.device, requires_grad=False)

    def __init__(self, qdata, scale, block_size, orig_dtype, per_tensor_scale=None, act_per_tensor_scale=None,
                 is_swizzled_scales=False, use_triton_kernel=False, act_quant_kwargs=None):
        super().__init__()
        if per_tensor_scale is not None:
            # a scalar, like the reference (nvfp4_tensor.py:69-79); or one value per out-feature [N], which only
            # ao_b200.fusion produces: a fused q|k|v / gate|up group keeps every member's own per-tensor scale
            assert per_tensor_scale.dim() == 0 or (per_tensor_scale.dim() == 1 and per_tensor_scale.shape[0] == qdata.shape[-2]), (
                "per_tensor_scale must be a scalar (or one value per out-feature for a fused group)")
        self.qdata = qdata
        self.scale = scale
        self.block_size = block_size
        self.orig_dtype = orig_dtype
        self.per_tensor_scale = per_tensor_scale
        self.act_per_tensor_scale = act_per_tensor_scale
        self.is_swizzled_scales = is_swizzled_scales
        self.use_triton_kernel = use_triton_kernel
        self.act_quant_kwargs = act_quant_kwargs

    def _quantization_type(self):
        return f"{self.is_swizzled_scales=}, {self.use_triton_kernel=}, {self.act_quant_kwargs=}"

    @staticmethod
    def to_nvfp4(data_hp: torch.Tensor, block_size: int = 16, per_tensor_scale: Optional[torch.Tensor] = None,
                 act_per_tensor_scale: Optional[torch.Tensor] = None, is_swizzled_scales: bool = False,
                 use_triton_kernel: bool = False, act_quant_kwargs: Optional[QuantizeTensorToNVFP4Kwargs] = None):
        assert block_size == 16, "NVFP4 requires block_size=16"
        assert data_hp.dim() == 2, "2-D tensors only"
        assert data_hp.dtype == torch.bfloat16, f"NVFP4Tensor.to_nvfp4: bf16 input only in this engine, got {data_hp.dtype}"
        assert data_hp.shape[-1] % block_size == 0, "K dim must be divisible by block_size"
        assert data_hp.is_contiguous() or rows_for_kernel(data_hp) is data_hp, "Only support contiguous data (or a 2-D column slice)"
        pts = per_tensor_scale.reshape(()) if per_tensor_scale is not None else None
        q, s = torch.ops.ao_b200.nvfp4_quantize(data_hp, pts.reshape(1) if pts is not None else None, is_swizzled_scales)
        s = s.view(torch.float8_e4m3fn)
        return NVFP4Tensor(q, s, block_size, data_hp.dtype, pts, act_per_tensor_scale, is_swizzled_scales,
                           use_triton_kernel, act_quant_kwargs)

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """e2m1 * f32(e4m3 scale) * per_tensor_scale, computed in fp32 then cast (reference :199-231)."""
        out = output_dtype or self.orig_dtype
        rows, K = self.shape[-2], self.shape[-1]
        lut = torch.tensor(_E2M1, dtype=torch.float32, device=self.qdata.device)
        q = self.qdata.reshape(rows, K // 2)
        v = torch.stack([lut[(q & 15).long()], lut[(q >> 4).long()]], dim=-1).reshape(rows, K)
        s = self.scale.view(torch.uint8)
        if self.is_swizzled_scales:
            s = from_blocked(s.reshape(-1), rows, K // self.block_size)
        s = s.reshape(rows, K // self.block_size).contiguous().view(torch.float8_e4m3fn).to(torch.float32)
        if self.per_tensor_scale is not None:
            s = s * (self.per_tensor_scale.reshape(-1, 1) if self.per_tensor_scale.dim() == 1 else self.per_tensor_scale)
        return (v * s.repeat_interleave(self.block_size, dim=1)).to(out)


implements = NVFP4Tensor.implements
implements_torch_function = NVFP4Tensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x, w, bias = args[0], args[1], args[2] if len(args) > 2 else None
    if not isinstance(w, NVFP4Tensor):
        raise NotImplementedError("NVFP4Tensor: weight must be NVFP4Tensor")
    assert w.is_swizzled_scales, "the kernels consume pre-swizzled (blocked) weight scales"
    N, K = w.shape[-2], w.shape[-1]
    orig_shape = x.shape
    x2 = x.reshape(-1, K)
    if x2.shape[0] == 0:
        return x.new_empty(*orig_shape[:-1], N)
    k = w.act_quant_kwargs
    b_pts = w.per_tensor_scale.reshape(-1) if w.per_tensor_scale is not None else None
    if k is None:
        # weight-only: y = x_bf16 @ dequant(W)^T, weights dequantised inside the wgmma kernel; a column slice of a
        # wider buffer goes in as is (the TMA descriptor carries the row pitch)
        xb = rows_for_kernel(x2.to(torch.bfloat16))
        y = torch.ops.ao_b200.nvfp4_weight_linear(xb, None, w.qdata, w.scale.view(torch.uint8), b_pts, bias)
        return y.reshape(*orig_shape[:-1], N).to(x.dtype)
    assert w.per_tensor_scale is None or w.per_tensor_scale.dim() == 0 or isinstance(k, QuantizeTensorToFloat8ActKwargs), (
        "a per-out-feature weight scale (fused group) is only supported by the weight-only / fp8-activation kernels")
    if isinstance(k, QuantizeTensorToFloat8ActKwargs):
        # NVFP4 weight x e4m3 rowwise activation (BASELINE config 5; defined in SURVEY §0-5 as
        # dequant(W_nvfp4) @ dequant(X_fp8 PerRow)): both dequants are exact in bf16.
        xq, xs = torch.ops.ao_b200.fp8_fakequant_rowwise(rows_for_kernel(x2.to(torch.bfloat16)))
        y = torch.ops.ao_b200.nvfp4_weight_linear(xq, xs.reshape(-1), w.qdata, w.scale.view(torch.uint8), b_pts, bias)
        return y.reshape(*orig_shape[:-1], N).to(x.dtype)
    xb = rows_for_kernel(x2.to(torch.bfloat16))
    if k.use_dynamic_per_tensor_scale:
        a_pts = per_tensor_amax_to_scale(torch.max(torch.abs(xb))).reshape(1)
    else:
        a_pts = w.act_per_tensor_scale.reshape(1) if w.act_per_tensor_scale is not None else None
    xq, xs = torch.ops.ao_b200.nvfp4_quantize(xb, a_pts, True)
    y = torch.ops.ao_b200.nvfp4_linear(xq, xs, a_pts, w.qdata, w.scale.view(torch.uint8), b_pts, bias)
    return y.reshape(*orig_shape[:-1], N).to(x.dtype)


@dataclass
class QuantizeTensorToFloat8ActKwargs(QuantizeTensorKwargs):
    """Activation recipe for the nvfp4-weight x fp8-activation linear: e4m3, per-token scale."""

    float8_dtype: torch.dtype = torch.float8_e4m3fn


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    """Row / column slices (`narrow`-style tensor-parallel loaders); reference `nvfp4_slice`."""
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    if step != 1:
        raise ValueError("Only support aten.slice with step=1")
    qd, sc = slice_qdata_and_scale(self, dim, start, end)
    pts = self.per_tensor_scale
    if pts is not None and pts.dim() == 1 and dim == 0:
        pts = aten.slice.Tensor(pts, 0, start, end, 1)   # per-out-feature scale of a fused group: follows the rows
    return return_and_correct_aliasing(func, args, kwargs, NVFP4Tensor(qd, sc, self.block_size, self.orig_dtype, pts, self.act_per_tensor_scale, self.is_swizzled_scales, self.use_triton_kernel, self.act_quant_kwargs))


@implements(aten.select.int)
def _(func, types, args, kwargs):
    self, dim, index = args
    assert dim == 0, f"NVFP4Tensor aten.select.int with {dim=} is not yet supported"
    assert self.qdata.dim() == self.scale.dim(), "unsupported"
    assert not self.is_swizzled_scales, "unsupported"
    qd, sc = self.qdata[index], self.scale[index]
    return return_and_correct_aliasing(func, args, kwargs, NVFP4Tensor(qd, sc, self.block_size, self.orig_dtype, self.per_tensor_scale, self.act_per_tensor_scale, self.is_swizzled_scales, self.use_triton_kernel, self.act_quant_kwargs))


NVFP4Tensor.__module__ = "ao_b200.prototype.mx_formats"
torch.serialization.add_safe_globals([NVFP4Tensor, QuantizeTensorToNVFP4Kwargs, QuantizeTensorToFloat8ActKwargs])
