"""NF4 (QLoRA) weights: ``NF4Tensor`` with the reference's constructor, attributes and checkpoint layout
(torchao/quantization/quantize_/workflows/nf4/nf4_tensor.py), served on sm_90a by one kernel launch per linear.

A 2-D weight ``[N, K]`` is stored as 4-bit indices into a 16-entry code table (``nf4``), two per byte with the even
element in the high nibble, one absmax scaler per ``block_size`` consecutive elements of the flattened weight, and the
scalers themselves double-quantized: minus their mean, scaled to int8 by one factor per ``scaler_block_size`` scalers.

The reference's forward is ``F.linear(x, weight.get_original_weight())`` (+ ``bias`` as a separate add), which rebuilds
the whole bf16 weight in eager torch on every call.  Here ``F.linear`` / ``linear_nf4`` run
``torch.ops.ao_b200.nf4_linear``: the scalers are decoded and every weight dequantized inside the GEMM, with the
reference's roundings (``ao_nf4_linear`` in ``include/ao_b200.h``).  Served: bf16 weights, bf16 activations, inference.
The training-side ops of the reference (backward, FSDP all-gather, ``split``, ``new_zeros``, ``as_strided``, ...) raise
``NotImplementedError``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

aten = torch.ops.aten

# the quantizer compares each element against the 16 table values; it runs over this many elements at a time
CHUNK_SIZE = 1024**2

# the NF4 code table of QLoRA (stored with every tensor, in the weight's dtype)
_NF4_VALUES = [-1.0000, -0.6962, -0.5251, -0.3949, -0.2844, -0.1848, -0.0911, 0.0000,
               0.0796, 0.1609, 0.2461, 0.3379, 0.4407, 0.5626, 0.7230, 1.0000]


@dataclass(frozen=True)
class SubclassTensorArgs:
    original_shape: torch.Size
    original_strides: Tuple
    storage_offset: int
    dtype: torch.dtype
    device: torch.device
    requires_grad: bool


def get_block_absmax(input_tensor: torch.Tensor, block_size: int) -> torch.Tensor:
    """The absmax of each block of ``block_size`` consecutive elements of a flat tensor."""
    assert input_tensor.dim() == 1, "Input tensor must be flattened"
    assert input_tensor.numel() % block_size == 0, (
        f"Input tensor must be divisible by block size, got {input_tensor.numel()} and {block_size}")
    return input_tensor.view(-1, block_size).abs().max(dim=1).values


_INNER = ["quantized_data", "scaler_mean", "quantization_factor", "quantized_scalers", "nf4"]


class NF4Tensor(torch.Tensor):
    """A 2-D (or 1-D) weight in the QLoRA NF4 format."""

    @staticmethod
    def __new__(cls, tensor_meta: SubclassTensorArgs, block_size: int, n_blocks: int, scaler_block_size: int,
                quantized_scalers: torch.Tensor, quantization_factor: torch.Tensor, scaler_mean: torch.Tensor,
                quantized_data: torch.Tensor, nf4: torch.Tensor):
        return torch.Tensor._make_wrapper_subclass(
            cls, tensor_meta.original_shape, tensor_meta.original_strides, tensor_meta.storage_offset,
            dtype=tensor_meta.dtype, device=tensor_meta.device, requires_grad=tensor_meta.requires_grad)

    def __init__(self, tensor_meta: SubclassTensorArgs, block_size: int, n_blocks: int, scaler_block_size: int,
                 quantized_scalers: torch.Tensor, quantization_factor: torch.Tensor, scaler_mean: torch.Tensor,
                 quantized_data: torch.Tensor, nf4: torch.Tensor):
        self.block_size = block_size
        self.n_blocks = n_blocks
        self.scaler_block_size = scaler_block_size
        self.quantized_scalers = quantized_scalers
        self.quantization_factor = quantization_factor
        self.scaler_mean = scaler_mean
        self.quantized_data = quantized_data
        self.nf4 = nf4

    # ---------------------------------------------------------------------------------------- quantization
    @classmethod
    @torch.no_grad()
    def from_tensor(cls, input_tensor: torch.Tensor, block_size: int, scaler_block_size: int) -> "NF4Tensor":
        assert input_tensor.dim() <= 2, f"expect input tensor dim <= 2 but got dim = {input_tensor.dim()}"
        assert input_tensor.numel() % block_size == 0, (
            f"Input tensor must be divisible by block size, got {input_tensor.numel()} and {block_size}")
        nf4 = torch.tensor(_NF4_VALUES, device=input_tensor.device, dtype=input_tensor.dtype)
        n_blocks = input_tensor.numel() // block_size
        quantized_scalers, quantization_factor, scaler_mean = cls.double_quantize_scalers(
            input_tensor.flatten(), block_size, scaler_block_size)
        quantized_data = cls.convert_to_norm_float_weight(input_tensor, n_blocks, block_size, nf4)
        meta = SubclassTensorArgs(input_tensor.size(), input_tensor.stride(), input_tensor.storage_offset(),
                                  input_tensor.dtype, input_tensor.device, input_tensor.requires_grad)
        return cls(meta, block_size, n_blocks, scaler_block_size, quantized_scalers, quantization_factor, scaler_mean,
                   quantized_data, nf4)

    @staticmethod
    def double_quantize_scalers(input_tensor: torch.Tensor, block_size: int,
                                scaler_block_size: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Block absmaxes minus their mean, as int8 codes with one factor ``256 / (2 * absmax)`` per
        ``scaler_block_size`` of them.  Returns (int8 scalers [n_blocks], factors [n_scaler_blocks], the mean)."""
        assert input_tensor.dim() == 1, "Input tensor must be flattened"
        assert input_tensor.numel() % scaler_block_size == 0, (
            f"Input tensor must be divisible by block size, got {input_tensor.numel()} and {scaler_block_size}")
        absmax = get_block_absmax(input_tensor, block_size)
        mean = absmax.mean()
        centered = absmax - mean
        assert centered.numel() % scaler_block_size == 0, (
            f"Number of scalers must be divisible by scaler block size, got {centered.numel()} scaler_block_size "
            f"{scaler_block_size} ")
        rows = centered.view(-1, scaler_block_size)
        factor = 256 / (2 * get_block_absmax(centered, scaler_block_size))   # elementwise: one value per row
        codes = (rows * factor.unsqueeze(-1)).round().clamp(-128, 127)
        return codes.flatten().to(torch.int8), factor.contiguous(), mean

    def dequantize_scalers(self, input_tensor: torch.Tensor, quantization_factor: torch.Tensor,
                           scaler_block_size: int) -> torch.Tensor:
        """The block scalers: ``bf16(q / factor) + mean`` in the weight's dtype."""
        assert input_tensor.dim() == 1, "Input tensor must be flattened"
        assert input_tensor.numel() % scaler_block_size == 0, (
            f"Input tensor must be divisible by block size, got {input_tensor.numel()} and {scaler_block_size}")
        rows = input_tensor.view(-1, scaler_block_size)
        return (rows / quantization_factor.unsqueeze(-1)).flatten().to(self.dtype) + self.scaler_mean

    @staticmethod
    def convert_to_norm_float_weight(input_tensor: torch.Tensor, n_blocks: int, block_size: int,
                                     nf4: torch.Tensor) -> torch.Tensor:
        """Each element over its block's absmax, to the nearest table entry; two 4-bit indices per byte, the even
        element in the high nibble."""
        flat = input_tensor.flatten()
        numel = flat.numel()
        assert numel % 2 == 0, "Number of elements must be even just to not have to think about the end"
        absmax = get_block_absmax(flat, block_size)
        scaled = (flat.view(n_blocks, block_size) / absmax.unsqueeze(-1).expand(n_blocks, block_size)).flatten()
        codes = torch.empty(numel, dtype=torch.uint8, device=input_tensor.device)
        for i in range(math.ceil(numel / CHUNK_SIZE)):
            lo, hi = i * CHUNK_SIZE, min((i + 1) * CHUNK_SIZE, numel)
            codes[lo:hi] = NF4Tensor.quantize_tensor_nearest(scaled[lo:hi], nf4).to(torch.uint8)
        return (codes[::2] << 4 | codes[1::2]).to(torch.uint8)

    @staticmethod
    def quantize_tensor_nearest(value: torch.Tensor, nf4: torch.Tensor) -> torch.Tensor:
        """The index of the nearest table entry (the first one on a tie)."""
        return (value.unsqueeze(-1) - nf4).abs().min(dim=-1).indices

    @staticmethod
    def dequantize(value: torch.Tensor, nf4: torch.Tensor) -> torch.Tensor:
        return nf4[value]

    def get_original_weight(self) -> torch.Tensor:
        """The dequantized weight: ``nf4[code] * scaler`` per element, in the weight's dtype."""
        even = self.dequantize((self.quantized_data >> 4).to(torch.long), self.nf4)
        odd = self.dequantize((self.quantized_data & 0b1111).to(torch.long), self.nf4)
        scalers = self.dequantize_scalers(self.quantized_scalers, self.quantization_factor, self.scaler_block_size)
        s = scalers.unsqueeze(-1).expand(scalers.size(0), self.block_size // 2).flatten()
        return torch.stack([even * s, odd * s], dim=-1).reshape(self.shape)

    # ---------------------------------------------------------------------------------------- tensor protocol
    def __repr__(self) -> str:
        return f"Quantized Data: {self.quantized_data}\nScalers: {self.quantized_scalers}\n"

    def __str__(self) -> str:
        return f"NF4Tensor({self.shape}, {self.block_size})"

    def _meta(self, **changes) -> SubclassTensorArgs:
        d = dict(original_shape=self.shape, original_strides=self.stride(), storage_offset=self.storage_offset(),
                 dtype=self.dtype, device=self.device, requires_grad=self.requires_grad)
        d.update(changes)
        return SubclassTensorArgs(**d)

    def __tensor_flatten__(self):
        ctx = {"block_size": self.block_size, "n_blocks": self.n_blocks, "scaler_block_size": self.scaler_block_size,
               "tensor_meta": self._meta()}
        return list(_INNER), ctx

    @staticmethod
    def __tensor_unflatten__(inner_tensors: Dict, metadata, outer_size, outer_stride):
        assert len(inner_tensors) == 5, "Expected 5 inner tensors"
        return NF4Tensor(metadata["tensor_meta"], metadata["block_size"], metadata["n_blocks"],
                         metadata["scaler_block_size"], inner_tensors["quantized_scalers"],
                         inner_tensors["quantization_factor"], inner_tensors["scaler_mean"],
                         inner_tensors["quantized_data"], inner_tensors["nf4"])

    def _with_inner(self, fn, **meta_changes) -> "NF4Tensor":
        t = {name: fn(getattr(self, name)) for name in _INNER}
        meta_changes.setdefault("device", t["quantized_data"].device)
        return NF4Tensor(self._meta(**meta_changes), self.block_size, self.n_blocks, self.scaler_block_size,
                         t["quantized_scalers"], t["quantization_factor"], t["scaler_mean"], t["quantized_data"],
                         t["nf4"])

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func in _NF4_OPS:
            return _NF4_OPS[func](func, args, kwargs)
        raise NotImplementedError(f"NF4Tensor dispatch: attempting to run {func}, this is not supported")

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func in _NF4_FUNCTIONS:
            return _NF4_FUNCTIONS[func](*args, **kwargs)
        with torch._C.DisableTorchFunctionSubclass():
            return func(*args, **kwargs)


def _same_metadata(a: NF4Tensor, b: NF4Tensor) -> bool:
    return (a.shape == b.shape and a.block_size == b.block_size and a.n_blocks == b.n_blocks
            and a.scaler_block_size == b.scaler_block_size
            and all(getattr(a, n).shape == getattr(b, n).shape for n in _INNER))


def _detach(func, args, kwargs):
    return args[0]._with_inner(lambda t: t.detach(), requires_grad=False)


def _clone(func, args, kwargs):
    return args[0]._with_inner(lambda t: t.clone())


def _to_copy(func, args, kwargs):
    t = args[0]
    dtype = kwargs.get("dtype")
    if dtype is not None and dtype != t.dtype:
        raise NotImplementedError("NF4Tensor: a dtype change dequantizes; use .to(dtype) or get_original_weight()")
    device = kwargs.get("device", t.device)
    return t._with_inner(lambda x: x.to(device=device, non_blocking=kwargs.get("non_blocking", False)))


def _copy_(func, args, kwargs):
    dst, src = args[0], args[1]
    if not (isinstance(dst, NF4Tensor) and isinstance(src, NF4Tensor) and _same_metadata(dst, src)):
        raise NotImplementedError("NF4Tensor.copy_ needs an NF4Tensor source with equal shape and block sizes")
    for name in _INNER:
        getattr(dst, name).copy_(getattr(src, name))
    return dst


def _is_pinned(func, args, kwargs):
    return args[0].quantized_data.is_pinned()


_NF4_OPS = {
    aten.detach.default: _detach,
    aten.clone.default: _clone,
    aten._to_copy.default: _to_copy,
    aten.copy_.default: _copy_,
    aten.is_pinned.default: _is_pinned,
}


def linear_nf4(input: torch.Tensor, weight: NF4Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``F.linear(input, weight.get_original_weight())`` (+ ``bias``, a separate bf16 add) in one launch of the
    sm_90a NF4 kernel.  Inference only: bf16 weights and activations, no input that requires grad with grad on."""
    if weight.dtype != torch.bfloat16:
        raise NotImplementedError(f"linear_nf4: NF4Tensor of dtype {weight.dtype}; the sm_90a kernel serves "
                                  f"NF4 weights of bf16 models only")
    if input.dtype != torch.bfloat16:
        raise NotImplementedError(f"linear_nf4: activations of dtype {input.dtype}; the sm_90a kernel takes bf16")
    if bias is not None and bias.dtype != torch.bfloat16:
        raise NotImplementedError(f"linear_nf4: bias of dtype {bias.dtype}; the sm_90a kernel takes bf16")
    if torch.is_grad_enabled() and input.requires_grad:
        raise NotImplementedError("linear_nf4: the backward of NF4 linears (QLoRA training) is not served")
    if weight.dim() != 2:
        raise NotImplementedError(f"linear_nf4: a {weight.dim()}-D NF4Tensor; only 2-D weights are served")
    from ao_b200.utils import rows_for_kernel

    K = input.shape[-1]
    y = torch.ops.ao_b200.nf4_linear(rows_for_kernel(input.reshape(-1, K)), weight.quantized_data,
                                     weight.quantized_scalers, weight.quantization_factor, weight.scaler_mean,
                                     weight.nf4, weight.block_size, weight.scaler_block_size, bias)
    return y.reshape(*input.shape[:-1], y.shape[-1])


def to_nf4(tensor, block_size: int = 64, scaler_block_size: int = 256) -> NF4Tensor:
    """Convert a tensor to NF4."""
    return NF4Tensor.from_tensor(tensor, block_size, scaler_block_size)


def _fn_to(tensor, *args, **kwargs):
    device, dtype, non_blocking, memory_format = torch._C._nn._parse_to(*args, **kwargs)
    if dtype is not None:
        return tensor.get_original_weight().to(device, dtype, non_blocking, memory_format=memory_format)
    if device is None:
        return tensor
    return tensor._with_inner(lambda t: t.to(device, non_blocking=non_blocking))


def _fn_cpu(tensor, *args, **kwargs):
    return _fn_to(tensor, "cpu")


def _fn_cuda(tensor, *args, **kwargs):
    return tensor._with_inner(lambda t: t.cuda(*args, **kwargs))


def _fn_linear(input, weight, bias=None):
    if not isinstance(weight, NF4Tensor):
        raise NotImplementedError("F.linear with an NF4Tensor input and a plain weight is not served")
    return linear_nf4(input, weight, bias)


def _fn_unsupported(name):
    def fn(*args, **kwargs):
        raise NotImplementedError(f"NF4Tensor.{name} is not served (QLoRA training / FSDP ops are out of scope)")
    return fn


_NF4_FUNCTIONS = {
    torch.Tensor.to: _fn_to,
    torch.Tensor.cpu: _fn_cpu,
    torch.Tensor.cuda: _fn_cuda,
    F.linear: _fn_linear,
    torch.Tensor.split: _fn_unsupported("split"),
    torch.Tensor.new_zeros: _fn_unsupported("new_zeros"),
    torch.Tensor.as_strided: _fn_unsupported("as_strided"),
}

torch.serialization.add_safe_globals([NF4Tensor, SubclassTensorArgs])
