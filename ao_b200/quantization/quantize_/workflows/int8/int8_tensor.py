"""int8 per-row weight with dynamic per-token int8 activations on wgmma s8.

Attribute names / order match torchao's Int8Tensor
(torchao/quantization/quantize_/workflows/int8/int8_tensor.py:74-85).  The linear replaces
``Int8Tensor.from_hp(x) -> _int_scaled_matmul -> aten._int_mm -> pointwise epilogue``
(:266-359, int8/kernels.py:114-144) with two launches: a fused per-token quantizer and an int8 GEMM
whose epilogue reproduces the reference's rounding order bf16(bf16(acc*s_x)*s_w + bias).
Without ``act_quant_kwargs`` (Int8WeightOnlyConfig) the linear is one launch: bf16 activations on the int8 weights.
With a calibrated ``act_quant_scale`` (Int8StaticActivationInt8WeightConfig) one kernel applies ``act_pre_scale`` and the
static scale and zero point, then the same GEMM runs.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.quantization.granularity import Granularity, PerRow, PerTensor
from ao_b200.quantization.quant_primitives import (
    MappingType, choose_qparams_affine_int8, dequantize_affine_int8, quantize_affine_int8)
from ao_b200.quantization.quantize_.common.quantize_tensor_kwargs import QuantizeTensorKwargs
from ao_b200.quantization.utils import get_block_size
from ao_b200.utils import TorchAOBaseTensor, fill_defaults, rows_for_kernel

__all__ = ["Int8Tensor", "QuantizeTensorToInt8Kwargs"]
aten = torch.ops.aten


@dataclass
class QuantizeTensorToInt8Kwargs(QuantizeTensorKwargs):
    granularity: Granularity
    mapping_type: MappingType = MappingType.SYMMETRIC
    reduce_range: bool = False


class Int8Tensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale"]
    optional_tensor_data_names = ["zero_point", "act_quant_scale", "act_quant_zero_point", "act_pre_scale"]
    tensor_attribute_names = ["block_size", "dtype"]
    optional_tensor_attribute_names = ["act_quant_kwargs", "reduce_range"]

    def __new__(cls, qdata, scale, block_size: List[int], dtype: torch.dtype, zero_point=None, act_quant_scale=None,
                act_quant_zero_point=None, act_pre_scale=None, act_quant_kwargs=None, reduce_range=False):
        return torch.Tensor._make_wrapper_subclass(cls, qdata.shape, device=qdata.device, dtype=dtype, requires_grad=False)

    def __init__(self, qdata, scale, block_size, dtype, zero_point=None, act_quant_scale=None,
                 act_quant_zero_point=None, act_pre_scale=None, act_quant_kwargs=None, reduce_range=False):
        super().__init__()
        self.qdata = qdata
        self.scale = scale
        self.block_size = block_size
        self.zero_point = zero_point
        self.act_quant_scale = act_quant_scale
        self.act_quant_zero_point = act_quant_zero_point
        self.act_pre_scale = act_pre_scale
        self.act_quant_kwargs = act_quant_kwargs
        self.reduce_range = reduce_range

    def _quantization_type(self):
        return f"{self.act_quant_kwargs=}, {self.block_size=}, {self.scale.shape=}"

    @staticmethod
    def _normalize_granularity(granularity):
        if granularity is None:
            return PerRow(), PerRow()
        if isinstance(granularity, (list, tuple)):
            assert len(granularity) == 2, "granularity list must be [activation, weight]"
            return granularity[0], granularity[1]
        return granularity, granularity

    @classmethod
    def from_hp(cls, hp_tensor: torch.Tensor, granularity: Granularity, mapping_type=MappingType.SYMMETRIC,
                scale=None, zero_point=None, act_quant_kwargs=None, act_quant_scale=None,
                act_quant_zero_point=None, act_pre_scale=None, reduce_range: Optional[bool] = False):
        block_size = list(get_block_size(hp_tensor.shape, granularity))
        qmin, qmax = (-64, 63) if reduce_range else (-128, 127)
        fast = (scale is None and hp_tensor.is_cuda and hp_tensor.dtype == torch.bfloat16
                and mapping_type == MappingType.SYMMETRIC and isinstance(granularity, PerRow)
                and granularity.dim in (-1, hp_tensor.dim() - 1) and not reduce_range and hp_tensor.shape[-1] % 8 == 0)
        if fast:
            x2 = rows_for_kernel(hp_tensor.reshape(-1, hp_tensor.shape[-1]))
            q, s = torch.ops.ao_b200.int8_quantize_rowwise(x2)
            int_data = q.reshape(hp_tensor.shape)
            scale = s.reshape(*hp_tensor.shape[:-1], 1)
            zero_point = torch.zeros_like(scale, dtype=torch.int8)
        else:
            if scale is None:
                scale, zero_point = choose_qparams_affine_int8(hp_tensor, block_size, mapping_type, qmin, qmax)
            else:
                assert scale.ndim == hp_tensor.ndim
                if zero_point is None:
                    zero_point = torch.zeros_like(scale, dtype=torch.int8)
            int_data = quantize_affine_int8(hp_tensor, block_size, scale, zero_point, qmin, qmax)
        return cls(int_data, scale, block_size, hp_tensor.dtype, zero_point=zero_point, act_quant_scale=act_quant_scale,
                   act_quant_zero_point=act_quant_zero_point, act_pre_scale=act_pre_scale,
                   act_quant_kwargs=act_quant_kwargs, reduce_range=reduce_range)

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        return dequantize_affine_int8(self.qdata, self.block_size, self.scale, self.zero_point,
                                      output_dtype if output_dtype is not None else self.dtype)


implements = Int8Tensor.implements
implements_torch_function = Int8Tensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x, w, bias = args[0], args[1], args[2] if len(args) > 2 else None
    assert isinstance(w, Int8Tensor), f"Expected weight to be Int8Tensor, got {type(w)}"
    out_dtype = x.dtype
    N, K = w.qdata.shape[-2], w.qdata.shape[-1]
    if w.act_quant_kwargs is not None and _static_quantizer_serves(x, w):
        return _static_linear(x, w, bias, out_dtype)
    if w.act_pre_scale is not None:
        x = x * w.act_pre_scale
    if w.act_quant_kwargs is None:
        return _weight_only_linear(x, w, bias, out_dtype)
    x2 = x.reshape(-1, K)
    out_shape = (*x.shape[:-1], N)
    if x2.shape[0] == 0:
        return x.new_empty(out_shape)
    kw = w.act_quant_kwargs
    xt = Int8Tensor.from_hp(x2, kw.granularity, mapping_type=kw.mapping_type, scale=w.act_quant_scale,
                            zero_point=w.act_quant_zero_point, reduce_range=kw.reduce_range)
    M = x2.shape[0]
    xs = xt.scale.reshape(-1).float()
    if xs.numel() == 1:
        xs = xs.expand(M)
    return _int8_activation_linear(xt.qdata, xs.contiguous(), xt.zero_point, w, bias, out_shape, out_dtype)


def _static_quantizer_serves(x, w):
    """The calibrated-scale path: bf16 activations and an fp32 ``act_quant_scale`` on x's device, the dtypes
    calibration produces.  A bf16 scale would make torch take the reciprocal and the product in bf16, and other
    activation dtypes promote differently: those keep the torch route below."""
    s, zp, p = w.act_quant_scale, w.act_quant_zero_point, w.act_pre_scale
    return (s is not None and x.dtype == torch.bfloat16 and x.is_cuda and s.dtype == torch.float32
            and s.device == x.device and (zp is None or (zp.dtype == torch.int8 and zp.device == x.device))
            and (p is None or (p.dtype in (torch.bfloat16, torch.float32) and p.numel() == x.shape[-1]
                               and p.device == x.device)))


def _static_linear(x, w, bias, out_dtype):
    """Two launches for a symmetric mapping: int8_quantize_static (the pre-scale product, the calibrated scale and zero
    point, the clamp) and int8_dyn_linear.  The scales are read on the device, so a CUDA graph replays whatever
    ``act_quant_scale`` holds.  Unlike the reference, a ``[1, 1]`` scale also serves a 3-D input: x is flattened to
    [M, K] first."""
    N, K = w.qdata.shape[-2], w.qdata.shape[-1]
    out_shape = (*x.shape[:-1], N)
    x2 = x.reshape(-1, K)
    if x2.shape[0] == 0:
        return x.new_empty(out_shape, dtype=out_dtype)
    qmin, qmax = (-64, 63) if w.act_quant_kwargs.reduce_range else (-128, 127)
    xq, xs, xzp = torch.ops.ao_b200.int8_quantize_static(rows_for_kernel(x2), w.act_quant_scale, w.act_quant_zero_point,
                                                         w.act_pre_scale, qmin, qmax)
    return _int8_activation_linear(xq, xs, xzp, w, bias, out_shape, out_dtype)


def _int8_activation_linear(xq, xs, xzp, w, bias, out_shape, out_dtype):
    """int8 activations xq [M, K] with f32 scales xs [M] (zero points xzp for an asymmetric mapping) on the weight."""
    N = w.qdata.shape[-2]
    ws = w.scale.reshape(-1).float()
    if ws.numel() == 1:
        ws = ws.expand(N)
    wq = w.qdata.contiguous()
    if w.act_quant_kwargs.mapping_type == MappingType.SYMMETRIC:
        y = torch.ops.ao_b200.int8_dyn_linear(xq.contiguous(), xs, wq, ws.contiguous(), bias)
        return y.reshape(out_shape).to(out_dtype)
    # asymmetric activations (int8_tensor.py:322-330): Y = (Xq Wq^T) s_x s_w - zp_x s_x rowsum(Wq) s_w
    acc = torch.ops.ao_b200.int8_mm_i32(xq.contiguous(), wq)
    y = (acc * xs.reshape(-1, 1)).to(out_dtype)
    zp = xzp.reshape(-1, 1).float()
    corr = (zp * xs.reshape(-1, 1)) * w.qdata.sum(dim=-1).float()
    y = (y - corr.to(out_dtype)) * ws
    if bias is not None:
        y = y + bias
    return y.reshape(out_shape).to(out_dtype)


def _weight_only_linear(x, w, bias, out_dtype):
    """bf16 activations on per-row / per-tensor int8 weights (reference :336-359): one launch whose epilogue keeps the
    reference's roundings bf16(bf16(bf16(acc) * bf16(s_w)) + bias).  Other activation dtypes are cast to bf16."""
    N, K = w.qdata.shape[-2], w.qdata.shape[-1]
    if w.qdata.dim() != 2 or list(w.block_size) not in ([1, K], [N, K]):
        raise NotImplementedError(
            f"int8 weight-only linear: block_size {list(w.block_size)} of a {tuple(w.qdata.shape)} weight is neither "
            f"per-row nor per-tensor (PerGroup has no sm_90a kernel in this engine)")
    out_shape = (*x.shape[:-1], N)
    if x.numel() == 0:
        return x.new_empty(out_shape)
    x2 = rows_for_kernel(x.to(torch.bfloat16).reshape(-1, K))
    ws = w.scale.reshape(-1).float()
    if ws.numel() == 1:
        ws = ws.expand(N)
    y = torch.ops.ao_b200.int8_weight_linear(x2, w.qdata.contiguous(), ws.contiguous(), bias)
    return y.reshape(out_shape).to(out_dtype)


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    assert step == 1 and dim in (0, 1, 2)
    qd = aten.slice.Tensor(self.qdata, dim, start, end, step)
    sc, zp = self.scale, self.zero_point
    if sc.numel() > 1 and sc.dim() == self.qdata.dim() and sc.shape[dim] == self.qdata.shape[dim]:
        sc = aten.slice.Tensor(sc, dim, start, end, step)
        if zp is not None:
            zp = aten.slice.Tensor(zp, dim, start, end, step)
    bs = list(self.block_size)
    if bs[dim] > qd.shape[dim]:
        bs[dim] = qd.shape[dim]
    return Int8Tensor(qd, sc, bs, self.dtype, zero_point=zp, act_quant_scale=self.act_quant_scale,
                      act_quant_zero_point=self.act_quant_zero_point, act_pre_scale=self.act_pre_scale,
                      act_quant_kwargs=self.act_quant_kwargs, reduce_range=self.reduce_range)


@implements(aten.select.int)
def _(func, types, args, kwargs):
    self, dim, index = args
    assert dim == 0
    sc = self.scale[index] if self.scale.dim() == self.qdata.dim() and self.scale.shape[0] == self.qdata.shape[0] else self.scale
    zp = self.zero_point
    if zp is not None and zp.dim() == self.qdata.dim() and zp.shape[0] == self.qdata.shape[0]:
        zp = zp[index]
    return Int8Tensor(self.qdata[index], sc, list(self.block_size[1:]), self.dtype, zero_point=zp,
                      act_quant_scale=self.act_quant_scale, act_quant_zero_point=self.act_quant_zero_point,
                      act_pre_scale=self.act_pre_scale, act_quant_kwargs=self.act_quant_kwargs,
                      reduce_range=self.reduce_range)


@implements(aten.transpose.int)
def _(func, types, args, kwargs):
    """A view with qdata, scale, zero_point and block_size swapped: how a 3-D expert weight [E, N, K] reaches
    torch._grouped_mm as mat_b [E, K, N].  Transposing twice gives back the stored form."""
    self, dim0, dim1 = args
    bs = list(self.block_size)
    bs[dim0], bs[dim1] = bs[dim1], bs[dim0]

    def swap(t):
        return t.transpose(dim0, dim1) if t is not None and t.dim() == self.qdata.dim() else t

    new = Int8Tensor(self.qdata.transpose(dim0, dim1), swap(self.scale), bs, self.dtype,
                     zero_point=swap(self.zero_point), act_quant_scale=self.act_quant_scale,
                     act_quant_zero_point=self.act_quant_zero_point, act_pre_scale=self.act_pre_scale,
                     act_quant_kwargs=self.act_quant_kwargs, reduce_range=self.reduce_range)
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements(aten._grouped_mm.default)
def _(func, types, args, kwargs):
    """torch._grouped_mm(x, W.transpose(-2, -1), offs=offs) with an Int8Tensor expert weight W [E, N, K], 2-D x 3-D:
    expert e's rows [offs[e-1], offs[e]) of x times W[e] in one launch, computing what the per-expert recipe
    F.linear(x[rows_e], W[e]) (select, then the dense linear) computes:

    * weight-only (no ``act_quant_kwargs``): bf16(bf16(bf16(x W[e]^T) * bf16(s_w[e]))), on bf16 x (after
      ``act_pre_scale``), ``int8_weight_grouped_mm``;
    * dynamic, symmetric PerRow activations: every routed row quantized as the dense linear quantizes it (a row's
      scale depends on that row only, so all M rows at once equal each expert's rows), then ``int8_dyn_grouped_mm``;
    * static, symmetric PerTensor activations with a [1, 1] ``act_quant_scale``: one scale for every row, the fused
      ``int8_quantize_static`` (``act_pre_scale`` included), then ``int8_dyn_grouped_mm``.

    Rows from offs[-1] on are left unwritten, as torch leaves them.  Other forms raise NotImplementedError."""
    mat_a, mat_b = args[0], args[1]
    offs = args[2] if len(args) > 2 else kwargs.get("offs", None)
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    out_dtype = args[4] if len(args) > 4 else kwargs.get("out_dtype", None)
    assert isinstance(mat_b, Int8Tensor)
    assert offs is not None, "offs is required for _grouped_mm"
    what = "Int8Tensor _grouped_mm"
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"{what}: only 2-D mat_a x 3-D mat_b, got {mat_a.dim()}-D x {mat_b.dim()}-D")
    if mat_b.qdata.stride(-2) >= mat_b.qdata.stride(-1):
        raise NotImplementedError(f"{what}: mat_b must be the transposed [E, N, K] expert weight, "
                                  f"W.transpose(-2, -1)")
    if bias is not None:
        raise NotImplementedError(f"{what}: bias is not supported")
    if isinstance(mat_a, TorchAOBaseTensor) or mat_a.dtype != torch.bfloat16 or out_dtype not in (None, torch.bfloat16):
        raise NotImplementedError(f"{what}: bf16 mat_a and output only, got {mat_a.dtype} -> {out_dtype}")
    E, K, N = mat_b.shape
    if list(mat_b.block_size) not in ([1, K, 1], [E, K, N]):
        raise NotImplementedError(
            f"{what}: block_size {list(mat_b.block_size)} of a {tuple(mat_b.shape)} weight is neither per-row nor "
            f"per-tensor (PerGroup has no sm_90a kernel in this engine)")
    if mat_a.shape[-1] != K:
        raise ValueError(f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}")
    if mat_a.shape[0] == 0:
        return mat_a.new_empty((0, N))
    wq = mat_b.qdata.transpose(-2, -1).contiguous()   # back to the stored [E, N, K]
    ws = mat_b.scale.float()
    # a per-tensor scale is expanded to one value per (expert, feature), a torch copy
    ws = (ws.reshape(E, N) if ws.numel() == E * N else ws.reshape(1, 1).expand(E, N)).contiguous()
    offs = offs.to(torch.int32)
    kw = mat_b.act_quant_kwargs
    x = mat_a
    if kw is None:
        if mat_b.act_pre_scale is not None:
            x = x * mat_b.act_pre_scale
        return torch.ops.ao_b200.int8_weight_grouped_mm(x.to(torch.bfloat16), wq, ws, offs)
    if kw.mapping_type != MappingType.SYMMETRIC or mat_b.act_quant_zero_point is not None:
        raise NotImplementedError(
            f"{what}: asymmetric int8 activations (or a static act_quant_zero_point) need each expert's rowsum(Wq) "
            f"correction, which the grouped kernel does not apply")
    if N % 8 != 0:
        raise NotImplementedError(f"{what}: N={N} output features per expert; the int8 x int8 kernel needs N % 8 == 0 "
                                  f"(the dense int8 rule)")
    s = mat_b.act_quant_scale
    if s is None:
        if not isinstance(kw.granularity, PerRow):
            raise NotImplementedError(
                f"{what}: dynamic {kw.granularity} activations; the per-expert recipe computes one scale over each "
                f"expert's own rows, not over all M, so only PerRow activations are served")
        if mat_b.act_pre_scale is not None:
            x = x * mat_b.act_pre_scale
        xt = Int8Tensor.from_hp(x, kw.granularity, mapping_type=kw.mapping_type, reduce_range=kw.reduce_range)
        xq, xs = xt.qdata, xt.scale.reshape(-1).float()
    else:
        if not isinstance(kw.granularity, PerTensor) or s.numel() != 1:
            raise NotImplementedError(
                f"{what}: a static {kw.granularity} act_quant_scale of shape {tuple(s.shape)}; it is tied to the rows "
                f"of one calibration batch and does not fit an expert's rows.  Only PerTensor with a [1, 1] scale")
        if _static_quantizer_serves(x, mat_b):
            qmin, qmax = (-64, 63) if kw.reduce_range else (-128, 127)
            xq, xs, _ = torch.ops.ao_b200.int8_quantize_static(rows_for_kernel(x), s, None, mat_b.act_pre_scale,
                                                               qmin, qmax)
        else:
            if mat_b.act_pre_scale is not None:
                x = x * mat_b.act_pre_scale
            xt = Int8Tensor.from_hp(x, kw.granularity, mapping_type=kw.mapping_type, scale=s,
                                    reduce_range=kw.reduce_range)
            xq, xs = xt.qdata, xt.scale.reshape(-1).float().expand(x.shape[0])
    return torch.ops.ao_b200.int8_dyn_grouped_mm(xq.contiguous(), xs.contiguous(), wq, ws, offs)


Int8Tensor.__module__ = "ao_b200.quantization"
torch.serialization.add_safe_globals([Int8Tensor, QuantizeTensorToInt8Kwargs, MappingType])
