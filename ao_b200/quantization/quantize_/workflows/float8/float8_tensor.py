"""e4m3 rowwise-scaled weight, dynamic rowwise activation quant, wgmma e4m3 GEMM.

Attribute names / order match torchao's Float8Tensor
(torchao/quantization/quantize_/workflows/float8/float8_tensor.py:105-113).  The linear replaces
``_float8_addmm_impl -> addmm_float8_unwrapped_inference -> torch._scaled_mm``
(:338-469, float8/inference.py:86-123) with two launches: the per-token quantizer and the GEMM with
a fused ``acc * s_x[m] * s_w[n] + bias -> bf16`` epilogue.
Blockwise weights (``block_size [128, 128]``, ``PerBlock([1, 128])`` activations) replace the reference's Triton GEMM
(:431-447) with two launches: the 1x128 quantizer and the blockwise GEMM (DESIGN §2f).
Without ``act_quant_kwargs`` (Float8WeightOnlyConfig) the linear is one launch: bf16 activations on the e4m3 weights.
``torch.bmm`` on per-row [B, K, N] weights, stored [B, K, N] or as the transposed view of a stored [B, N, K], replaces
the reference's mslk batched GEMM (:472-522) without its transposed weight copy (DESIGN §2a).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.float8.inference import (FP8Granularity, Float8MMConfig, _is_1_128_128_scaled, _is_1_128_scaled,
                                      _is_128_128_scaled, _is_rowwise_scaled, _is_tensorwise_scaled)
from ao_b200.quantization.granularity import PerBlock, PerRow, PerTensor
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
        assert not isinstance(input_tensor, TorchAOBaseTensor), "Expecting input_tensor to be unquantized"
        return _weight_only_linear(input_tensor, weight_tensor, bias)
    assert not isinstance(input_tensor, TorchAOBaseTensor), "input tensor was already quantized"
    gran = act_quant_kwargs.granularity
    if isinstance(gran, PerBlock):
        return _blockwise_linear(input_tensor, weight_tensor, bias)
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


def _blockwise_linear(x, w, bias):
    """1x128 activation blocks on 128x128 weight blocks (reference :431-447, its Triton GEMM then ``res + bias``): two
    launches, the 1x128 quantizer and the GEMM, which scales each 128-k chunk's partial sums by the token's and the
    weight block's scales as it adds them up and rounds the sum and the bias add to bf16.  The weight must come from a
    bf16 model (the blockwise recipe's only dtype here), and the activations are bf16."""
    kw = w.act_quant_kwargs
    N, K = w.qdata.shape
    if not (_is_128_128_scaled(w.block_size) and _is_1_128_scaled(get_block_size(x.shape, kw.granularity))):
        raise AssertionError(f"unsupported: {list(w.block_size)} weight blocks with {kw.granularity} activations "
                             f"(PerBlock activations run with 128x128 weight blocks and 1x128 activation blocks only)")
    if w.dtype != torch.bfloat16 or x.dtype != torch.bfloat16:
        raise NotImplementedError(f"float8 blockwise linear: bf16 activations and a weight quantized from bf16 only, got "
                                  f"{x.dtype} activations and a {w.dtype} weight")
    if w.qdata.dtype != torch.float8_e4m3fn or kw.float8_dtype != torch.float8_e4m3fn:
        raise NotImplementedError("float8 blockwise linear: e4m3 weights and activations only")
    if kw.hp_value_lb is not None or kw.hp_value_ub is not None:
        raise NotImplementedError("float8 blockwise linear: activation_value_lb / activation_value_ub are not supported")
    out_shape = (*x.shape[:-1], N)
    x2 = x.reshape(-1, K)
    if x2.shape[0] == 0:
        return x.new_empty(out_shape)
    xq, xs = torch.ops.ao_b200.fp8_quantize_1x128(rows_for_kernel(x2))
    y = torch.ops.ao_b200.fp8_blockwise_linear(xq, xs, w.qdata.contiguous(), w.scale.contiguous(), bias)
    return y.reshape(out_shape)


def _weight_only_linear(x, w, bias):
    """bf16 activations on per-row / per-tensor e4m3 weights (reference :459-469, torch.matmul on the dequantized
    weight, then + bias): one launch that dequantizes each weight as the reference does, bf16(fp32(q) * s), and rounds
    the sum and the bias add to bf16.  Other activation dtypes are cast to bf16.  The weight must come from a bf16
    model: for an fp16 or fp32 one the reference dequantizes into that dtype and multiplies in it, which this kernel
    does not compute."""
    N, K = w.qdata.shape[-2], w.qdata.shape[-1]
    if w.dtype != torch.bfloat16:
        raise NotImplementedError(
            f"float8 weight-only linear: the weight was quantized from {w.dtype}; the reference dequantizes it into "
            f"{w.dtype} and runs the matmul in {w.dtype}, and the sm_90a kernel of this engine computes in "
            f"torch.bfloat16 only")
    if w.qdata.dim() != 2 or w.qdata.dtype != torch.float8_e4m3fn or list(w.block_size) not in ([1, K], [N, K]):
        raise NotImplementedError(
            f"float8 weight-only linear: a {tuple(w.qdata.shape)} {w.qdata.dtype} weight with block_size "
            f"{list(w.block_size)} has no sm_90a kernel in this engine (2-D e4m3 weights with per-row or per-tensor "
            f"scales only)")
    out_shape = (*x.shape[:-1], N)
    if x.numel() == 0:
        return x.new_empty(out_shape)
    x2 = rows_for_kernel(x.to(torch.bfloat16).reshape(-1, K))
    ws = w.scale.reshape(-1).float()
    if ws.numel() == 1:
        ws = ws.expand(N)
    y = torch.ops.ao_b200.fp8_weight_linear(x2, w.qdata.contiguous(), ws.contiguous(), bias)
    return y.reshape(out_shape).to(x.dtype)


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    input_tensor, weight_tensor, bias = args[0], args[1], args[2] if len(args) > 2 else None
    return _float8_linear_impl(input_tensor, weight_tensor, bias)


@implements(aten.bmm.default)
@implements_torch_function(torch.bmm)
def _(func, types, args, kwargs):
    return _float8_bmm_impl(args[0], args[1])


def _float8_bmm_impl(x, w):
    """torch.bmm(x, w) with a per-row Float8Tensor w of shape [B, K, N] (the reference's handler,
    float8_tensor.py:472-522): x's B*M rows are quantized per row to e4m3, then one batched GEMM computes
    bf16(acc * x_scale[m] * w_scale[b, n]) with no bias term.  w arrives in one of two layouts, told apart by qdata's
    strides, both with block_size [1, K, 1] and a scale of B*N values:
      * the transposed view of a stored [B, N, K] weight (torch.bmm(x, w.transpose(-2, -1))): the grouped e4m3 kernel;
      * a stored [B, K, N] weight quantized with PerRow(1) (Llama-4 expert layers, torch.bmm(x, w)): an N-major kernel
        that transposes each weight tile on chip, so no transposed copy of the weights is made.
    Only bf16 x; the weight-only form, per-tensor or blockwise scales and KernelPreference.TORCH are rejected."""
    assert isinstance(w, Float8Tensor), (
        f"Don't expect to reach here with an override other than weight currently, {type(x)} {type(w)}")
    assert w.kernel_preference != KernelPreference.TORCH, "bmm is not supported for TORCH"
    kw = w.act_quant_kwargs
    if kw is None:
        raise NotImplementedError("bmm only support float8 dynamic activation + float8 weight")
    if x.dim() != 3 or w.dim() != 3:
        raise NotImplementedError(f"Float8Tensor bmm: 3-D x and weight only, got {x.dim()}-D x {w.dim()}-D")
    B, K, N = w.shape
    if isinstance(kw.granularity, PerBlock) or _is_1_128_128_scaled(w.block_size):
        raise NotImplementedError(f"Float8Tensor bmm: 128x128 blockwise weights (block_size {list(w.block_size)}) have "
                                  f"no batched kernel in this engine; quantize the weight with PerRow scales")
    assert list(w.block_size) == [1, K, 1], "bmm only works for per row weight quantization"
    assert isinstance(kw.granularity, PerRow), "bmm only works for per row activation quantization"
    if isinstance(x, TorchAOBaseTensor) or x.dtype != torch.bfloat16:
        raise NotImplementedError(f"Float8Tensor bmm: bf16 x only, got {type(x).__name__} {x.dtype}")
    if w.qdata.dtype != torch.float8_e4m3fn or kw.float8_dtype != torch.float8_e4m3fn:
        raise NotImplementedError("Float8Tensor bmm: e4m3 weights and activations only")
    if x.shape[0] != B or x.shape[-1] != K:
        raise ValueError(f"bmm: x {tuple(x.shape)} does not match the weight {tuple(w.shape)}")
    M = x.shape[1]
    if M == 0:
        return x.new_empty(B, 0, N)
    qd = w.qdata
    if qd.stride(-2) < qd.stride(-1):      # the transposed view of a stored [B, N, K] weight
        wq = qd.transpose(-2, -1).contiguous().transpose(-2, -1)
    elif qd.stride(-1) == 1:               # a stored [B, K, N] weight
        wq = qd.contiguous()
    else:
        raise NotImplementedError(f"Float8Tensor bmm: weight qdata strides {qd.stride()} are neither a stored "
                                  f"[B, K, N] nor the transposed view of a stored [B, N, K]")
    xq_t = Float8Tensor.from_hp(x.reshape(-1, K), kw.float8_dtype, kw.granularity, kw.mm_config, kw.hp_value_lb,
                                kw.hp_value_ub, kw.kernel_preference)
    return torch.ops.ao_b200.fp8_rowwise_bmm(xq_t.qdata.reshape(B, M, K), xq_t.scale.reshape(-1).float().contiguous(),
                                             wq, w.scale.reshape(B, N).float().contiguous())


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    assert step == 1 and dim in (0, 1)
    qd = aten.slice.Tensor(self.qdata, dim, start, end, step)
    sc = self.scale
    if sc.numel() > 1 and sc.shape[dim] == self.qdata.shape[dim]:
        sc = aten.slice.Tensor(sc, dim, start, end, step)
    elif sc.numel() > 1 and sc.dim() == self.qdata.dim() and 1 < sc.shape[dim] < self.qdata.shape[dim]:
        sc = _slice_block_scale(sc, self.qdata.shape[dim], dim, start, end)
    bs = list(self.block_size)
    if bs[dim] > qd.shape[dim]:
        bs[dim] = qd.shape[dim]
    return Float8Tensor(qd, sc, bs, self.mm_config, self.act_quant_kwargs, self.kernel_preference, self.dtype)


def _slice_block_scale(sc, size, dim, start, end):
    """The scales of rows / columns [start, end) of a block-scaled tensor (128x128 weight blocks) along dim: whole
    blocks only (reference _slice_scale_for_dimension, :733-790).  A bound inside a block would leave the sliced tensor
    with a block it only partly holds, whose scale no longer describes it: ValueError."""
    block = size // sc.shape[dim]
    start = 0 if start is None else max(0, start + size if start < 0 else start)
    end = size if end is None else min(size, end + size if end < 0 else end)
    if start % block != 0 or (end % block != 0 and end != size):
        raise ValueError(f"Float8Tensor slice [{start}:{end}] along dim {dim} is not aligned to its scale blocks of "
                         f"{block}")
    return aten.slice.Tensor(sc, dim, start // block, -(-end // block), 1)


@implements(aten.select.int)
def _(func, types, args, kwargs):
    """Expert `index` of a 3-D weight as a 2-D tensor (reference :936-955): qdata[index], scale[index] and
    block_size[1:], which the dense linear serves: the MoE expert loop's `F.linear(x, w[e])`.  A per-tensor scale
    [1, 1, 1] is shared by every expert: each gets scale[0] (the reference's scale[index] fails for index > 0)."""
    self, dim, index = args
    assert dim == 0, f"Float8Tensor aten.select.int with {dim=} is not yet supported"
    assert self.qdata.dim() == self.scale.dim() == len(self.block_size), "unsupported"
    sc = self.scale[index] if self.scale.shape[0] == self.qdata.shape[0] else self.scale[0]
    new = Float8Tensor(self.qdata[index], sc, list(self.block_size[1:]), self.mm_config,
                       self.act_quant_kwargs, self.kernel_preference, self.dtype)
    return return_and_correct_aliasing(func, args, kwargs, new)


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
    """torch._grouped_mm(x, W.transpose(-2, -1), offs=offs) with a Float8Tensor expert weight W [E, N, K] (the
    reference's handler, float8_tensor.py:1085-1122).  Dynamic (rowwise) activations: the routed tokens are quantized
    per row and the grouped GEMM runs on the stored qdata with w_scale[e, n].  Only the 2-D x 3-D form with PerRow
    activations.  Weight-only: _weight_only_grouped_mm.  PerBlock([1, 128]) activations on [1, 128, 128] weight
    blocks: _blockwise_grouped_mm."""
    mat_a, mat_b = args[0], args[1]
    offs = args[2] if len(args) > 2 else kwargs.get("offs", None)
    assert isinstance(mat_b, Float8Tensor)
    assert offs is not None, "offs is required for _grouped_mm"
    assert mat_b.qdata.stride(-2) < mat_b.qdata.stride(-1), "mat_b must be the transposed [E, N, K] weight"
    act_quant_kwargs = mat_b.act_quant_kwargs
    if act_quant_kwargs is None:
        return _weight_only_grouped_mm(mat_a, mat_b, offs, args, kwargs)
    gran = act_quant_kwargs.granularity
    if (isinstance(gran, PerBlock) and _is_1_128_scaled(gran.block_size)
            and _is_1_128_128_scaled(mat_b.block_size)):
        return _blockwise_grouped_mm(mat_a, mat_b, offs, args, kwargs)
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


def _blockwise_grouped_mm(mat_a, mat_b, offs, args, kwargs):
    """1x128 activation blocks on [1, 128, 128] expert weight blocks: the reference's per-expert recipe, select and
    the dense blockwise linear (_blockwise_linear), in two launches.  The 1x128 quantizer runs once over all routed rows
    (it is per row, so this equals quantizing each expert's rows on their own), then one grouped GEMM sums and rounds
    each expert's rows as the dense GEMM does.  Rows from offs[-1] on are left unwritten, as torch leaves them.  Only
    the 2-D x 3-D form of a bf16 model, bf16 mat_a and output, e4m3, no bias and no activation clamp."""
    kw = mat_b.act_quant_kwargs
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    out_dtype = args[4] if len(args) > 4 else kwargs.get("out_dtype", None)
    if mat_b.dtype != torch.bfloat16:
        raise NotImplementedError(f"Float8Tensor blockwise _grouped_mm: the weight was quantized from {mat_b.dtype}; "
                                  f"the sm_90a kernel of this engine serves weights quantized from torch.bfloat16 only")
    if isinstance(mat_a, TorchAOBaseTensor) or mat_a.dtype != torch.bfloat16 or out_dtype not in (None, torch.bfloat16):
        raise NotImplementedError(f"Float8Tensor blockwise _grouped_mm: bf16 mat_a and output only, got "
                                  f"{mat_a.dtype} -> {out_dtype}")
    if mat_b.qdata.dtype != torch.float8_e4m3fn or kw.float8_dtype != torch.float8_e4m3fn:
        raise NotImplementedError(f"Float8Tensor blockwise _grouped_mm: e4m3 weights and activations only, got "
                                  f"{mat_b.qdata.dtype} weights and {kw.float8_dtype} activations")
    if kw.hp_value_lb is not None or kw.hp_value_ub is not None:
        raise NotImplementedError("Float8Tensor blockwise _grouped_mm: activation_value_lb / activation_value_ub are "
                                  "not supported")
    if bias is not None:
        raise NotImplementedError("Float8Tensor blockwise _grouped_mm: bias is not supported")
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"Float8Tensor blockwise _grouped_mm: only 2-D mat_a x 3-D mat_b, got "
                                  f"{mat_a.dim()}-D x {mat_b.dim()}-D")
    E, K, N = mat_b.shape
    if mat_a.shape[-1] != K:
        raise ValueError(f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}")
    xq, xs = torch.ops.ao_b200.fp8_quantize_1x128(rows_for_kernel(mat_a))
    # back to the stored [E, N, K] codes and [E, N/128, K/128] scales
    return torch.ops.ao_b200.fp8_blockwise_grouped_mm(xq, xs, mat_b.qdata.transpose(-2, -1).contiguous(),
                                                      mat_b.scale.transpose(-2, -1).contiguous(), offs.to(torch.int32))


def _weight_only_grouped_mm(mat_a, mat_b, offs, args, kwargs):
    """The weight-only branch (reference :1099-1100, torch._grouped_mm on mat_b.dequantize()): expert e's rows
    [offs[e-1], offs[e]) of the bf16 mat_a times its weights, each dequantized as the reference does,
    bf16(fp32(q) * s), inside one grouped wgmma kernel; the sum is rounded once to bf16.  Rows from offs[-1] on are
    left unwritten, as torch leaves them.  Only the 2-D x 3-D form of a bf16 model, no bias, a bf16 output, and
    N % 8 == 0."""
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    out_dtype = args[4] if len(args) > 4 else kwargs.get("out_dtype", None)
    if mat_b.dtype != torch.bfloat16:
        raise NotImplementedError(
            f"Float8Tensor weight-only _grouped_mm: the weight was quantized from {mat_b.dtype}; the reference "
            f"dequantizes it into {mat_b.dtype} and multiplies in {mat_b.dtype}, and the sm_90a kernel of this engine "
            f"computes in torch.bfloat16 only")
    if isinstance(mat_a, TorchAOBaseTensor) or mat_a.dtype != torch.bfloat16 or out_dtype not in (None, torch.bfloat16):
        raise NotImplementedError(f"Float8Tensor weight-only _grouped_mm: bf16 mat_a and output only, got "
                                  f"{mat_a.dtype} -> {out_dtype}")
    if bias is not None:
        raise NotImplementedError("Float8Tensor weight-only _grouped_mm: bias is not supported")
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"Float8Tensor weight-only _grouped_mm: only 2-D mat_a x 3-D mat_b, got "
                                  f"{mat_a.dim()}-D x {mat_b.dim()}-D")
    E, K, N = mat_b.shape
    if mat_b.qdata.dtype != torch.float8_e4m3fn or list(mat_b.block_size) not in ([1, K, 1], [E, K, N]):
        raise NotImplementedError(
            f"Float8Tensor weight-only _grouped_mm: a {mat_b.qdata.dtype} weight with block_size "
            f"{list(mat_b.block_size)} has no sm_90a kernel in this engine (e4m3 expert weights with per-row or "
            f"per-tensor scales only)")
    if N % 8 != 0:
        raise NotImplementedError(f"Float8Tensor weight-only _grouped_mm: N={N} output features per expert; the sm_90a "
                                  f"kernel of this engine needs N % 8 == 0 (each expert's scales start on 32 bytes)")
    if mat_a.shape[-1] != K:
        raise ValueError(f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}")
    wq = mat_b.qdata.transpose(-2, -1)   # back to the stored [E, N, K]
    ws = mat_b.scale.float()
    ws = ws.reshape(E, N) if ws.numel() == E * N else ws.reshape(1, 1).expand(E, N)
    return torch.ops.ao_b200.fp8_weight_grouped_mm(mat_a, wq.contiguous(), ws.contiguous(), offs.to(torch.int32))


Float8Tensor.__module__ = "ao_b200.quantization"
torch.serialization.add_safe_globals([Float8Tensor, QuantizeTensorToFloat8Kwargs, Float8MMConfig])
