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
        shape = list(qdata.shape)
        if elem_dtype == torch.float4_e2m1fn_x2:
            # two codes per byte: the high-precision shape.  A transposed 3-D expert weight (qdata [E, K/2, N], how
            # torch._grouped_mm receives it) packs dim -2
            shape[-2 if _is_transposed_3d(qdata) else -1] *= 2
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
        quantize = torch.ops.ao_b200.mxfp4_quantize if elem_dtype == torch.float4_e2m1fn_x2 else torch.ops.ao_b200.mxfp8_quantize
        if data_hp.dim() == 3 and is_swizzled_scales:
            # a 3-D expert weight [E, N, K]: expert by expert (setup time only), each expert's blocked scales one after
            # the other, [E, 32 * ceil(N/128), 16 * ceil(K/128)].  For N % 128 == 0 that is the reference's to_blocked of
            # the [E*N, K/32] scales (mx_tensor.py:401-407); otherwise every expert starts on its own 128-row block
            qs, ss = zip(*(quantize(data_hp[e], True) for e in range(data_hp.shape[0])))
            q, s = torch.stack(qs), torch.stack(ss)
        else:
            q, s = quantize(data_hp.reshape(-1, K), is_swizzled_scales)
            q = q.reshape(*lead, q.shape[-1])
        s = s.view(torch.float8_e8m0fnu)
        if not is_swizzled_scales:
            s = s.reshape(*lead, K // block_size)
        return MXTensor(q, s, elem_dtype, block_size, data_hp.dtype, kernel_preference, act_quant_kwargs,
                        is_swizzled_scales)

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """code x 2^(e - 127) in fp32, then cast.  A 3-D expert weight is dequantized expert by expert, its transposed
        view as the transpose of that."""
        out = output_dtype or self.orig_dtype
        if self.qdata.dim() == 3:
            q, s = self.qdata, self.scale
            transposed = _is_transposed_3d(q)
            if transposed:
                q, s = q.transpose(-2, -1), s.transpose(-2, -1)
            y = torch.stack([_dequant_2d(q[e], s[e], self.elem_dtype, self.block_size, self.is_swizzled_scales, out)
                             for e in range(q.shape[0])])
            return y.transpose(-2, -1) if transposed else y
        y = _dequant_2d(self.qdata, self.scale, self.elem_dtype, self.block_size, self.is_swizzled_scales, out)
        return y.reshape(self.shape)


def _is_transposed_3d(qdata):
    return qdata.dim() == 3 and qdata.stride(-2) < qdata.stride(-1)


def _dequant_2d(qdata, scale, elem_dtype, block_size, swizzled, out):
    """[rows, K] codes ([rows, K/2] bytes for mxfp4, or any leading dims) with their scales (plain or blocked) -> [rows, K]."""
    fp4 = elem_dtype == torch.float4_e2m1fn_x2
    K = qdata.shape[-1] * (2 if fp4 else 1)
    rows = qdata.numel() // qdata.shape[-1]
    s = scale.view(torch.uint8)
    if swizzled:
        s = from_blocked(s.reshape(-1), rows, K // block_size)
    s = s.reshape(rows, K // block_size)
    e = torch.pow(2.0, s.to(torch.float32) - 127.0)
    e = torch.where(s == 255, torch.full_like(e, float("nan")), e)
    if fp4:
        q = qdata.view(torch.uint8).reshape(rows, K // 2)
        c = torch.stack([q & 15, q >> 4], dim=-1).reshape(rows, K).to(torch.int32)   # even k in the low nibble
        ce, cm = (c >> 1) & 3, (c & 1).to(torch.float32)
        # e2m1 (s e1 e0 m): m / 2 for e = 0, else 2^(e-1) * (1 + m / 2); no host table, so it can be graph-captured
        p2 = torch.bitwise_left_shift(torch.ones_like(ce), (ce - 1).clamp(min=0)).to(torch.float32)
        v = torch.where(ce == 0, 0.5 * cm, p2 * (1.0 + 0.5 * cm))
        v = torch.where((c & 8) != 0, -v, v)
    else:
        v = qdata.reshape(rows, K).to(torch.float32)
    return (v * e.repeat_interleave(block_size, dim=1)).to(out)


implements = MXTensor.implements
implements_torch_function = MXTensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x, w, bias = args[0], args[1], args[2] if len(args) > 2 else None
    assert isinstance(w, MXTensor), "MXTensor: weight must be MXTensor"
    if w.qdata.dim() != 2:
        raise NotImplementedError("MXTensor linear: 2-D weights only; a 3-D expert weight runs through "
                                  "torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)")
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
    # expert e of a 3-D weight [E, N, K] with N % 128 == 0: its blocked scales are the contiguous
    # [32 * N/128, 16 * ceil(K/128)] slice e of the stacked ones (to_mx), what F.linear(x, w[e]) runs on
    expert = self.qdata.dim() == 3 and not _is_transposed_3d(self.qdata) and self.shape[-2] % 128 == 0
    assert not self.is_swizzled_scales or expert, "unsupported"
    qd, sc = self.qdata[index], self.scale[index]
    return return_and_correct_aliasing(func, args, kwargs, MXTensor(qd, sc, self.elem_dtype, self.block_size, self.orig_dtype, self.kernel_preference, self.act_quant_kwargs, self.is_swizzled_scales))


@implements(aten.transpose.int)
def _(func, types, args, kwargs):
    """A view of a 3-D expert weight with qdata and scale transposed: how W [E, N, K] reaches torch._grouped_mm as
    mat_b [E, K, N]."""
    self, dim0, dim1 = args
    assert self.qdata.dim() == 3, f"MXTensor transpose: 3-D tensors only, got rank {self.qdata.dim()}"
    assert (dim0, dim1) in ((1, 2), (2, 1), (-1, -2), (-2, -1)), f"transpose unsupported for {dim0=} {dim1=}"
    new = MXTensor(self.qdata.transpose(dim0, dim1), self.scale.transpose(dim0, dim1), self.elem_dtype, self.block_size,
                   self.orig_dtype, self.kernel_preference, self.act_quant_kwargs, self.is_swizzled_scales)
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements(aten._grouped_mm.default)
def _(func, types, args, kwargs):
    """torch._grouped_mm(x, W.transpose(-2, -1), offs=offs) with an MXTensor expert weight W [E, N, K]
    (MXDynamicActivationMXWeightConfig, mxfp8 or mxfp4): expert e's rows of the output are the dense MX linear of its
    rows of x against W[e].  The activations are quantized to the weight's format and dequantized exactly as bf16
    (mx*_fakequant: MX scales belong to one block of one row, so no expert bookkeeping), then multiplied by each
    expert's weights, dequantized exactly inside the grouped GEMM.  Only the 2-D x 3-D form, with offs and without
    bias."""
    mat_a, mat_b = args[0], args[1]
    offs = args[2] if len(args) > 2 else kwargs.get("offs", None)
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    if not isinstance(mat_b, MXTensor) or isinstance(mat_a, MXTensor):
        raise NotImplementedError("MXTensor _grouped_mm: only a bf16 mat_a times an MXTensor mat_b")
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"MXTensor _grouped_mm: only 2-D mat_a x 3-D mat_b, got {mat_a.dim()}-D x {mat_b.dim()}-D")
    if offs is None:
        raise NotImplementedError("MXTensor _grouped_mm: offs is required")
    if bias is not None:
        raise NotImplementedError("MXTensor _grouped_mm: bias is not supported")
    if not _is_transposed_3d(mat_b.qdata):
        raise NotImplementedError("MXTensor _grouped_mm: mat_b must be the transposed [E, N, K] weight")
    if not mat_b.is_swizzled_scales:
        raise NotImplementedError("MXTensor _grouped_mm: the kernel consumes blocked (swizzled) weight scales")
    k = mat_b.act_quant_kwargs
    if k is None:
        raise NotImplementedError("MXTensor _grouped_mm: MX weight-only is outside this engine's scope; only "
                                  "MXDynamicActivationMXWeightConfig (act_quant_kwargs set)")
    if k.elem_dtype != mat_b.elem_dtype:
        raise NotImplementedError(f"MXTensor _grouped_mm: activation element dtype {k.elem_dtype} differs from the "
                                  f"weight's {mat_b.elem_dtype}")
    E, K, N = mat_b.shape
    if mat_a.shape[-1] != K:
        raise ValueError(f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}")
    ops = torch.ops.ao_b200
    fp4 = mat_b.elem_dtype == torch.float4_e2m1fn_x2
    xhat = (ops.mxfp4_fakequant if fp4 else ops.mxfp8_fakequant)(rows_for_kernel(mat_a.to(torch.bfloat16)))
    wq = mat_b.qdata.transpose(-2, -1)   # back to the stored [E, N, K] / [E, N, K/2]
    ws = mat_b.scale.transpose(-2, -1)
    mm = ops.mxfp4_grouped_mm if fp4 else ops.mxfp8_grouped_mm
    y = mm(xhat, wq.contiguous(), ws.contiguous().view(torch.uint8), offs.to(torch.int32))
    return y.to(mat_a.dtype)


MXTensor.__module__ = "ao_b200.prototype.mx_formats"
torch.serialization.add_safe_globals([MXTensor, QuantizeTensorToMXKwargs, ScaleCalculationMode])
