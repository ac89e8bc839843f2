"""MXFP8 / MXFP4 weight/activation tensor on Hopper wgmma (bf16, exactly dequantised operands).

Attribute names/order match torchao's MXTensor (torchao/prototype/mx_formats/mx_tensor.py:509-517):
``qdata, scale | elem_dtype, block_size, orig_dtype, kernel_preference, act_quant_kwargs,
is_swizzled_scales``.  ``to_mx`` (e4m3, block 32, RCEIL) runs the fused CUDA quantizer
(bit-exact with the reference's torch ops, tests/test_oracle_golden.py + test_lowp_gpu.py);
the linear replaces ``mx_linear -> _addmm_mx_dispatch -> torch._scaled_mm`` (:759-882).

With ``elem_dtype=torch.float4_e2m1fn_x2`` (mxfp4) ``qdata`` is uint8 ``[..., K/2]``, two e2m1 codes per byte with
the even k in the low nibble, and the tensor's shape is the high-precision one (``K = 2 * qdata.shape[-1]``), as in
the reference (:530-540).  ``to_mx`` runs ``mxfp4_quantize`` and the linear ``mxfp4_linear``.
"""
from __future__ import annotations

from dataclasses import dataclass
from enum import Enum, auto
from typing import Optional

import torch

from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.common.quantize_tensor_kwargs import QuantizeTensorKwargs
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.utils import TorchAOBaseTensor, fill_defaults, rows_for_kernel

from .utils import from_blocked, hp_data_dims_to_swizzled_scale_dims_mx, slice_qdata_and_scale

aten = torch.ops.aten
__all__ = ["MXTensor", "ScaleCalculationMode", "QuantizeTensorToMXKwargs"]


class ScaleCalculationMode(Enum):
    """How the e8m0 block scale is derived (reference :55-97).  Only RCEIL (the inference default,
    cuBLAS-documented) is implemented by the CUDA quantizer."""

    FLOOR = "floor"
    CEIL = "ceil"
    EVEN = "even"
    RCEIL = "rceil"


@dataclass
class QuantizeTensorToMXKwargs(QuantizeTensorKwargs):
    elem_dtype: torch.dtype = torch.float8_e4m3fn
    block_size: int = 32
    scaling_mode: ScaleCalculationMode = ScaleCalculationMode.RCEIL
    kernel_preference: KernelPreference = KernelPreference.AUTO
    is_swizzled_scales: bool = False


class MXTensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale"]
    tensor_attribute_names = ["elem_dtype", "block_size", "orig_dtype", "kernel_preference", "act_quant_kwargs",
                              "is_swizzled_scales"]

    def __new__(cls, qdata, scale, elem_dtype, block_size, orig_dtype, kernel_preference, act_quant_kwargs,
                is_swizzled_scales):
        shape = qdata.shape
        if elem_dtype == torch.float4_e2m1fn_x2:
            shape = (*shape[:-1], shape[-1] * 2)   # two codes per byte: the high-precision shape
        return torch.Tensor._make_wrapper_subclass(cls, shape, dtype=orig_dtype, device=qdata.device,
                                                   requires_grad=False)

    def __init__(self, qdata, scale, elem_dtype, block_size, orig_dtype, kernel_preference, act_quant_kwargs,
                 is_swizzled_scales):
        super().__init__()
        assert scale.dtype in (torch.float8_e8m0fnu, torch.uint8), f"scale must be e8m0 bytes, got {scale.dtype}"
        self.qdata = qdata
        self.scale = scale
        self.elem_dtype = elem_dtype
        self.block_size = block_size
        self.orig_dtype = orig_dtype
        self.kernel_preference = kernel_preference
        self.act_quant_kwargs = act_quant_kwargs
        self.is_swizzled_scales = is_swizzled_scales

    def _quantization_type(self):
        return f"{self.elem_dtype=}, {self.block_size=}, {self.orig_dtype=}, {self.kernel_preference=}, {self.act_quant_kwargs=}"

    @staticmethod
    def to_mx(data_hp: torch.Tensor, elem_dtype=torch.float8_e4m3fn, block_size: int = 32,
              scaling_mode: ScaleCalculationMode = ScaleCalculationMode.RCEIL,
              kernel_preference: KernelPreference = KernelPreference.AUTO,
              act_quant_kwargs: Optional[QuantizeTensorToMXKwargs] = None, is_swizzled_scales: bool = False):
        assert data_hp.dtype == torch.bfloat16, f"MXTensor.to_mx: bf16 input only in this engine, got {data_hp.dtype}"
        assert data_hp.shape[-1] % block_size == 0, (
            f"the last dimension of shape {data_hp.shape} must be divisible by block_size {block_size}")
        # contiguous like the reference requires (mx_tensor.py:247), or a 2-D column slice (rows with a pitch): the
        # quantizer kernel takes the pitch, no copy
        assert data_hp.is_contiguous() or rows_for_kernel(data_hp) is data_hp, "unsupported"
        if elem_dtype not in (torch.float8_e4m3fn, torch.float4_e2m1fn_x2) or block_size != 32:
            raise NotImplementedError(f"only mxfp8 and mxfp4 (float8_e4m3fn / float4_e2m1fn_x2, block 32) are "
                                      f"implemented, got {elem_dtype} with block {block_size}")
        if scaling_mode != ScaleCalculationMode.RCEIL:
            raise NotImplementedError("only ScaleCalculationMode.RCEIL (the inference default) is implemented")
        lead, K = data_hp.shape[:-1], data_hp.shape[-1]
        x2 = data_hp.reshape(-1, K)
        if elem_dtype == torch.float4_e2m1fn_x2:
            q, s = torch.ops.ao_b200.mxfp4_quantize(x2, is_swizzled_scales)
            q = q.reshape(*lead, K // 2)
        else:
            q, s = torch.ops.ao_b200.mxfp8_quantize(x2, is_swizzled_scales)
            q = q.reshape(*lead, K)
        s = s.view(torch.float8_e8m0fnu)
        if not is_swizzled_scales:
            s = s.reshape(*lead, K // block_size)
        return MXTensor(q, s, elem_dtype, block_size, data_hp.dtype, kernel_preference, act_quant_kwargs,
                        is_swizzled_scales)

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        out = output_dtype or self.orig_dtype
        K = self.shape[-1]
        rows = self.qdata.numel() // self.qdata.shape[-1]
        s = self.scale.view(torch.uint8)
        if self.is_swizzled_scales:
            s = from_blocked(s.reshape(-1), rows, K // self.block_size)
        s = s.reshape(rows, K // self.block_size)
        e = torch.pow(2.0, s.to(torch.float32) - 127.0)
        e = torch.where(s == 255, torch.full_like(e, float("nan")), e)
        if self.elem_dtype == torch.float4_e2m1fn_x2:
            q = self.qdata.view(torch.uint8).reshape(rows, K // 2)
            c = torch.stack([q & 15, q >> 4], dim=-1).reshape(rows, K).to(torch.int32)   # even k in the low nibble
            ce, cm = (c >> 1) & 3, (c & 1).to(torch.float32)
            # e2m1 (s e1 e0 m): m / 2 for e = 0, else 2^(e-1) * (1 + m / 2); no host table, so it can be graph-captured
            p2 = torch.bitwise_left_shift(torch.ones_like(ce), (ce - 1).clamp(min=0)).to(torch.float32)
            v = torch.where(ce == 0, 0.5 * cm, p2 * (1.0 + 0.5 * cm))
            v = torch.where((c & 8) != 0, -v, v)
        else:
            v = self.qdata.reshape(rows, K).to(torch.float32)
        v = v * e.repeat_interleave(self.block_size, dim=1)
        return v.reshape(self.shape).to(out)


implements = MXTensor.implements
implements_torch_function = MXTensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x, w, bias = args[0], args[1], args[2] if len(args) > 2 else None
    assert isinstance(w, MXTensor), "MXTensor: weight must be MXTensor"
    k = w.act_quant_kwargs
    if k is None:
        raise NotImplementedError("MX weight-only linear is outside this engine's scope (SURVEY §8)")
    assert w.is_swizzled_scales and k.is_swizzled_scales, "the kernel consumes pre-swizzled (blocked) scales"
    N, K = w.shape[-2], w.shape[-1]
    orig_shape = x.shape
    x2 = x.reshape(-1, K)
    if x2.shape[0] == 0:
        return x.new_empty(*orig_shape[:-1], N)
    xq = MXTensor.to_mx(rows_for_kernel(x2.to(torch.bfloat16)), k.elem_dtype, k.block_size, k.scaling_mode,
                        k.kernel_preference, None, True)
    mm = torch.ops.ao_b200.mxfp4_linear if w.elem_dtype == torch.float4_e2m1fn_x2 else torch.ops.ao_b200.mxfp8_linear
    y = mm(xq.qdata, xq.scale.view(torch.uint8), w.qdata, w.scale.view(torch.uint8), bias)
    return y.reshape(*orig_shape[:-1], N).to(x.dtype)


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    """Row / column slices (`narrow`-style tensor-parallel loaders); reference `mx_slice`."""
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    if step != 1:
        raise ValueError("Only support aten.slice with step=1")
    qd, sc = slice_qdata_and_scale(self, dim, start, end)
    return return_and_correct_aliasing(func, args, kwargs, MXTensor(qd, sc, self.elem_dtype, self.block_size, self.orig_dtype, self.kernel_preference, self.act_quant_kwargs, self.is_swizzled_scales))


@implements(aten.select.int)
def _(func, types, args, kwargs):
    self, dim, index = args
    assert dim == 0, f"MXTensor aten.select.int with {dim=} is not yet supported"
    assert self.qdata.dim() == self.scale.dim(), "unsupported"
    assert not self.is_swizzled_scales, "unsupported"
    qd, sc = self.qdata[index], self.scale[index]
    return return_and_correct_aliasing(func, args, kwargs, MXTensor(qd, sc, self.elem_dtype, self.block_size, self.orig_dtype, self.kernel_preference, self.act_quant_kwargs, self.is_swizzled_scales))


MXTensor.__module__ = "ao_b200.prototype.mx_formats"
torch.serialization.add_safe_globals([MXTensor, QuantizeTensorToMXKwargs, ScaleCalculationMode])
