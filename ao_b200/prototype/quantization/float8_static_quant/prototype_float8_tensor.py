"""e4m3 weight with a calibrated (static) e4m3 activation scale and an optional output fake-quant.

Attribute names, order and defaults match torchao's PrototypeFloat8Tensor
(torchao/prototype/quantization/float8_static_quant/prototype_float8_tensor.py:58-144).  The linear replaces
``_float8_addmm_impl`` (:329-474): ``from_hp(x, scale=act_quant_scale)`` -> ``torch._scaled_mm`` -> (with
``output_act_quant_scale``) ``from_hp(y, scale=output_act_quant_scale).dequantize()`` with two launches: the static
quantizer (``fp8_quantize_static``) and the e4m3 GEMM (``fp8_static_linear``: the epilogue of the dynamic linear, and
the output fake-quant after it).  The scales are read on the device, so a CUDA graph of the linear replays
whatever the scale tensors hold.  Deliberate difference: x is flattened to [M, K] first, so a ``[1, 1]`` scale also
serves 3-D inputs, which the reference rejects (``scale.ndim == x.ndim``).  A ``[M', 1]`` scale with M' != M raises
ValueError instead of broadcasting.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.float8.inference import FP8Granularity, Float8MMConfig
from ao_b200.quantization.granularity import PerRow
from ao_b200.quantization.quant_primitives import dequantize_affine_float8, quantize_affine_float8
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.workflows.float8.float8_tensor import (
    Float8Tensor, QuantizeTensorToFloat8Kwargs, _float8_linear_impl, _weight_only_linear)
from ao_b200.quantization.utils import get_block_size
from ao_b200.utils import TorchAOBaseTensor, fill_defaults, rows_for_kernel

__all__ = ["PrototypeFloat8Tensor"]
aten = torch.ops.aten


class PrototypeFloat8Tensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale"]
    optional_tensor_data_names = ["act_quant_scale", "output_act_quant_scale"]
    tensor_attribute_names = []
    optional_tensor_attribute_names = ["block_size", "mm_config", "act_quant_kwargs", "kernel_preference", "dtype",
                                       "output_act_quant_kwargs"]

    def __new__(cls, qdata, scale, act_quant_scale=None, output_act_quant_scale=None,
                block_size: Optional[List[int]] = None, mm_config: Optional[Float8MMConfig] = None,
                act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None,
                kernel_preference: KernelPreference = KernelPreference.AUTO, dtype: Optional[torch.dtype] = None,
                output_act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None):
        return torch.Tensor._make_wrapper_subclass(cls, qdata.shape, device=qdata.device, dtype=dtype, requires_grad=False)

    def __init__(self, qdata, scale, act_quant_scale=None, output_act_quant_scale=None, block_size=None, mm_config=None,
                 act_quant_kwargs=None, kernel_preference=KernelPreference.AUTO, dtype=None,
                 output_act_quant_kwargs=None):
        super().__init__()
        self.qdata = qdata
        self.scale = scale
        self.act_quant_scale = act_quant_scale
        self.block_size = block_size
        self.mm_config = mm_config
        self.act_quant_kwargs = act_quant_kwargs
        self.kernel_preference = kernel_preference
        self.output_act_quant_scale = output_act_quant_scale
        self.output_act_quant_kwargs = output_act_quant_kwargs

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
                act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None, scale: Optional[torch.Tensor] = None,
                act_quant_scale: Optional[torch.Tensor] = None, output_act_quant_scale: Optional[torch.Tensor] = None,
                output_act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None):
        """Without ``scale``: the scale and codes Float8Tensor.from_hp computes (the reference's
        _choose_scale_float8 / _quantize_affine_float8).  With ``scale`` (static): the codes of that scale, whose
        shape must be the tensor's block grid (reference :182-203)."""
        block_size = list(get_block_size(hp_tensor.shape, granularity))
        if scale is not None:
            assert scale.ndim == hp_tensor.ndim
            assert all(hp_tensor.shape[i] // block_size[i] == scale.shape[i] for i in range(hp_tensor.ndim))
            data = quantize_affine_float8(hp_tensor, scale, float8_dtype)
        else:
            t = Float8Tensor.from_hp(hp_tensor, float8_dtype, granularity, mm_config, hp_value_lb, hp_value_ub,
                                     kernel_preference)
            data, scale = t.qdata, t.scale
        return cls(data, scale, act_quant_scale=act_quant_scale, output_act_quant_scale=output_act_quant_scale,
                   block_size=block_size, mm_config=mm_config, act_quant_kwargs=act_quant_kwargs,
                   kernel_preference=kernel_preference, dtype=hp_tensor.dtype,
                   output_act_quant_kwargs=output_act_quant_kwargs)

    def _like(self, qdata, scale, block_size):
        """A tensor with new codes, scales and block size that keeps every other attribute, the calibrated scales
        included (what slice / select / transpose need)."""
        return PrototypeFloat8Tensor(qdata, scale, act_quant_scale=self.act_quant_scale,
                                     output_act_quant_scale=self.output_act_quant_scale, block_size=list(block_size),
                                     mm_config=self.mm_config, act_quant_kwargs=self.act_quant_kwargs,
                                     kernel_preference=self.kernel_preference, dtype=self.dtype,
                                     output_act_quant_kwargs=self.output_act_quant_kwargs)


implements = PrototypeFloat8Tensor.implements
implements_torch_function = PrototypeFloat8Tensor.implements_torch_function


def _token_scale(s: torch.Tensor, M: int, name: str) -> torch.Tensor:
    """A calibrated scale as the kernels take it: one value, or one per row of the flattened [M, K] input."""
    if s.numel() != 1 and s.numel() != M:
        raise ValueError(f"PrototypeFloat8Tensor: {name} has shape {tuple(s.shape)}; it must hold one scale "
                         f"(PerTensor) or one per row of the input, M={M} (PerRow)")
    return s


def _static_linear(x, w, bias):
    """Two launches: the static quantizer and the e4m3 GEMM (with the output fake-quant in its epilogue when the
    weight has ``output_act_quant_scale``).  bf16 activations with an fp32 scale on their device run
    fp8_quantize_static; other dtypes take the reference's torch ops for the codes and then the same GEMM, whose
    output is bf16 cast to x's dtype, as for the dynamic Float8Tensor."""
    N, K = w.qdata.shape[-2], w.qdata.shape[-1]
    out_shape = (*x.shape[:-1], N)
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    s = _token_scale(w.act_quant_scale, M, "act_quant_scale")
    so = w.output_act_quant_scale
    if so is not None:
        so = _token_scale(so, M, "output_act_quant_scale")
    if M == 0:
        return x.new_empty(out_shape)
    if x.dtype == torch.bfloat16 and x.is_cuda and s.dtype == torch.float32 and s.device == x.device:
        xq, xs = torch.ops.ao_b200.fp8_quantize_static(rows_for_kernel(x2), s)
    else:
        s = s.to(x.device).reshape(-1, 1)
        xq = quantize_affine_float8(x2, s, w.act_quant_kwargs.float8_dtype)
        xs = s.float().reshape(-1).expand(M).contiguous()
    # a per-tensor weight scale stays one value (the kernel reads it for every output feature: no [N] copy)
    ws = w.scale.reshape(-1).float().contiguous()
    if so is not None:
        so = so.to(device=x.device, dtype=torch.float32)
    y = torch.ops.ao_b200.fp8_static_linear(xq, xs, w.qdata.contiguous(), ws, bias, so)
    return y.reshape(out_shape).to(x.dtype)


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x, w, bias = args[0], args[1], args[2] if len(args) > 2 else None
    assert isinstance(w, PrototypeFloat8Tensor), f"Expected weight to be PrototypeFloat8Tensor, got {type(w)}"
    assert not isinstance(x, TorchAOBaseTensor), "input tensor was already quantized"
    if w.act_quant_kwargs is None:
        if w.output_act_quant_kwargs is not None:
            raise NotImplementedError("PrototypeFloat8Tensor: the output fake-quant runs with static activations only")
        return _weight_only_linear(x, w, bias)
    if w.act_quant_scale is None:
        # dynamic activations (the reference's from_hp without a scale): the Float8Tensor linear
        if w.output_act_quant_kwargs is not None:
            raise NotImplementedError("PrototypeFloat8Tensor: the output fake-quant runs with static activations only")
        return _float8_linear_impl(x, w, bias)
    return _static_linear(x, w, bias)


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    """Rows or columns of a per-tensor or per-row weight (vLLM's weight loading narrows the parameter); the scale is
    sliced with the rows it describes."""
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    assert step == 1 and 0 <= dim < self.qdata.dim(), f"unsupported slice dim={dim} step={step}"
    qd = aten.slice.Tensor(self.qdata, dim, start, end, step)
    sc = self.scale
    if sc.numel() > 1 and sc.dim() == self.qdata.dim() and sc.shape[dim] == self.qdata.shape[dim]:
        sc = aten.slice.Tensor(sc, dim, start, end, step)
    bs = list(self.block_size)
    bs[dim] = min(bs[dim], qd.shape[dim])
    return self._like(qd, sc, bs)


@implements(aten.select.int)
def _(func, types, args, kwargs):
    """Expert `index` of a 3-D weight (reference :969-993), keeping the calibrated scales: the MoE expert loop's
    ``F.linear(x, w[e])``.  A per-tensor scale [1, 1, 1] is shared by every expert."""
    self, dim, index = args
    assert dim == 0, f"PrototypeFloat8Tensor aten.select.int with {dim=} is not yet supported"
    assert self.qdata.dim() == self.scale.dim() == len(self.block_size), "unsupported"
    sc = self.scale[index] if self.scale.shape[0] == self.qdata.shape[0] else self.scale[0]
    return return_and_correct_aliasing(func, args, kwargs, self._like(self.qdata[index], sc, self.block_size[1:]))


@implements(aten.transpose.int)
def _(func, types, args, kwargs):
    self, dim0, dim1 = args
    bs = list(self.block_size)
    bs[dim0], bs[dim1] = bs[dim1], bs[dim0]
    new = self._like(self.qdata.transpose(dim0, dim1), self.scale.transpose(dim0, dim1), bs)
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements(aten.t.default)
def _(func, types, args, kwargs):
    self = args[0]
    assert len(self.block_size) == 2
    new = self._like(self.qdata.t(), self.scale.t(), [self.block_size[1], self.block_size[0]])
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements_torch_function(torch.Tensor.t)
def _(func, types, args, kwargs):
    self = args[0]
    assert len(self.block_size) == 2
    return self._like(self.qdata.t(), self.scale.t(), [self.block_size[1], self.block_size[0]])


PrototypeFloat8Tensor.__module__ = "ao_b200.prototype.quantization.float8_static_quant"
# Allow a model with PrototypeFloat8Tensor weights to be loaded with `weights_only=True`
torch.serialization.add_safe_globals([PrototypeFloat8Tensor])
