"""int4 weight in the tinygemm tile-packed layout, served by the sm_90a wgmma kernel.

Same class / attribute names and on-disk layout as the reference
(torchao/quantization/quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py): ``qdata`` int32
[N/8, K/128, 32, 4], ``scale_and_zero`` bf16 [K/g, N, 2], ``block_size``, ``shape``,
optional ``act_pre_scale``.  What changes is underneath: packing calls
``torch.ops.ao_b200.int4_pack_tile4d`` (instead of aten._convert_weight_to_int4pack, :202) and
the linear calls ``torch.ops.ao_b200.int4_tilepacked_linear`` (instead of
aten._weight_int4pack_mm + pad/slice/bias kernels, :278-299).

MoE expert weights are 3-D, ``[E, N, K]``: ``qdata`` int32 [E, N/8, K/128, 32, 4] and ``scale_and_zero`` bf16
[E, K/g, N, 2] (reference :206-217).  ``select(0, e)`` gives expert e's 2-D tensor (the eager expert loop's
``F.linear(x, w[e])``), and ``torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)`` runs every expert in one
``torch.ops.ao_b200.int4_tilepacked_grouped_mm``.  The transposed view keeps the packed data as it is and records the
transpose in ``shape`` and ``block_size`` ([E, K, N], [1, g, 1]).
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

from ao_b200.quantization.quant_primitives import choose_qparams_affine_tinygemm, quantize_affine_tinygemm
from ao_b200.quantization.utils import pack_tinygemm_scales_and_zeros
from ao_b200.utils import TorchAOBaseTensor, fill_defaults, find_multiple

from .int4_choose_qparams_algorithm import Int4ChooseQParamsAlgorithm

__all__ = ["Int4TilePackedTo4dTensor"]

aten = torch.ops.aten
INNER_K_TILES = 8  # fixed, as in the reference (:119)


class Int4TilePackedTo4dTensor(TorchAOBaseTensor):
    tensor_data_names = ["qdata", "scale_and_zero"]
    tensor_attribute_names = ["block_size", "shape"]
    optional_tensor_data_names = ["act_pre_scale"]

    def __new__(cls, qdata, scale_and_zero, block_size, shape, act_pre_scale: Optional[torch.Tensor] = None):
        kwargs = {"device": qdata.device, "dtype": torch.bfloat16, "requires_grad": False}
        return torch.Tensor._make_wrapper_subclass(cls, shape, **kwargs)

    def __init__(self, qdata, scale_and_zero, block_size, shape, act_pre_scale: Optional[torch.Tensor] = None):
        super().__init__()
        self.qdata = qdata
        self.scale_and_zero = scale_and_zero
        self.block_size = block_size
        self.act_pre_scale = act_pre_scale

    def _quantization_type(self):
        s = f"shape={self.shape}, block_size={self.block_size}, device={self.device}"
        if self.act_pre_scale is not None:
            s += f", act_pre_scale.shape={self.act_pre_scale.shape}"
        return s

    @classmethod
    def from_hp(cls, hp_tensor: torch.Tensor, block_size: List[int],
                int4_choose_qparams_algorithm: Int4ChooseQParamsAlgorithm = Int4ChooseQParamsAlgorithm.TINYGEMM,
                ntile_size: Optional[int] = 8):
        assert len(block_size) == hp_tensor.ndim, (
            f"Expecting the length of block_size to be equal to the dimension of the weight, got {block_size=} and {hp_tensor.ndim=}")
        assert all(x == 1 for x in block_size[:-1]), f"Only per group quantization is supported, got block_size: {block_size}"
        assert hp_tensor.dtype == torch.bfloat16, f"Only bfloat16 is supported for Int4TilePackedTo4dTensor, got {hp_tensor.dtype}"
        assert hp_tensor.dim() in (2, 3), "Int4TilePackedTo4dTensor: 2-D weights, or 3-D [E, N, K] expert weights"
        if not hp_tensor.is_cuda:
            # same exception type as the reference, where aten::_convert_weight_to_int4pack has no CPU kernel
            # (test_int4_tile_packed_to_4d_tensor.py:194-202)
            raise NotImplementedError("Could not run 'ao_b200::int4_pack_tile4d' with arguments from the 'CPU' backend: "
                                      "Int4TilePackedTo4dTensor.from_hp needs a CUDA tensor (sm_90a packing kernel)")
        original_shape = hp_tensor.shape
        lead = tuple(original_shape[:-2])   # (E,) for expert weights
        N0, K0 = original_shape[-2:]
        g = block_size[-1]
        K = find_multiple(K0, 1024)
        N = find_multiple(N0, ntile_size or 8)
        # every expert is padded on its own; its rows are then rows e*N .. e*N+N-1 of one [E*N, K] weight, whose groups,
        # n8-tiles and qparams never cross an expert
        w = torch.nn.functional.pad(hp_tensor, (0, K - K0, 0, N - N0)).reshape(-1, K)
        if int4_choose_qparams_algorithm == Int4ChooseQParamsAlgorithm.HQQ:
            # reference :149-167 -> _choose_qparams_and_quantize_affine_hqq (quant_primitives.py:1797-2002); here one
            # CUDA solver (ao_b200/csrc/int4_hqq.cu), scale / zero already in the tinygemm convention.  Expert weights
            # get ONE solve over the [E*N, K] view, as the reference makes one call on the 3-D tensor: its early stop
            # uses the error of the whole tensor, so an expert is not what quantizing it alone would give
            q, scale, zero = torch.ops.ao_b200.int4_hqq_quantize(w.contiguous(), g)
            q = q.to(torch.int32)
        else:
            assert int4_choose_qparams_algorithm == Int4ChooseQParamsAlgorithm.TINYGEMM, (
                f"Unsupported Int4ChooseQParamsAlgorithm: {int4_choose_qparams_algorithm}")
            scale, zero = choose_qparams_affine_tinygemm(w, g)
            q = quantize_affine_tinygemm(w, g, scale, zero)
        q_u8 = (q[:, ::2] << 4 | q[:, 1::2]).to(torch.uint8).contiguous()
        qdata = torch.ops.ao_b200.int4_pack_tile4d(q_u8, INNER_K_TILES)
        qdata = qdata.reshape(*lead, N // 8, *qdata.shape[1:]) if lead else qdata
        scale, zero = (scale.reshape(*lead, N, -1), zero.reshape(*lead, N, -1)) if lead else (scale, zero)
        scale_and_zero = pack_tinygemm_scales_and_zeros(scale, zero, scale.dtype)
        return cls(qdata=qdata, scale_and_zero=scale_and_zero, block_size=list(block_size), shape=original_shape,
                   act_pre_scale=None)

    def _is_transposed(self) -> bool:
        """The [E, K, N] view of a 3-D expert weight (block_size [1, g, 1]): how torch._grouped_mm receives it."""
        return self.qdata.dim() == 5 and self.block_size[-1] == 1

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """bf16((q-8)*s+z) for the original (unpadded) shape; a transposed expert view as the transpose of that."""
        if self.qdata.dim() == 5:
            # all experts in one call: their n8-tiles are consecutive, their scale groups go to [K/g, E*N, 2]
            E, N, K = self.qdata.shape[0], self.qdata.shape[1] * 8, self.qdata.shape[2] * 128
            g = max(self.block_size)
            sz = self.scale_and_zero.transpose(0, 1).reshape(K // g, E * N, 2)
            w = torch.ops.ao_b200.int4_dequant_tile4d(self.qdata.reshape(E * N // 8, K // 128, 32, 4), sz, g)
            transposed = self._is_transposed()
            N0, K0 = (self.shape[2], self.shape[1]) if transposed else (self.shape[1], self.shape[2])
            w = w.reshape(E, N, K)[:, :N0, :K0]
            w = w.transpose(-2, -1) if transposed else w
        else:
            w = torch.ops.ao_b200.int4_dequant_tile4d(self.qdata, self.scale_and_zero, self.block_size[-1])
            w = w[: self.shape[0], : self.shape[1]]
        return w if output_dtype in (None, torch.bfloat16) else w.to(output_dtype)


implements = Int4TilePackedTo4dTensor.implements
implements_torch_function = Int4TilePackedTo4dTensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    input_tensor, weight_tensor, bias = args[0], args[1], args[2] if len(args) > 2 else None
    if weight_tensor.qdata.dim() != 4:
        raise NotImplementedError(
            f"Int4TilePackedTo4dTensor linear: 2-D weights only, got shape {tuple(weight_tensor.shape)}; a 3-D expert "
            f"weight runs one expert through select (F.linear(x, w[e])) or all of them through "
            f"torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)")
    assert weight_tensor.qdata.is_contiguous(), "Expected qdata to be contiguous"
    assert weight_tensor.scale_and_zero.is_contiguous(), "Expected scale_and_zero to be contiguous"
    assert weight_tensor.block_size[0] == 1, f"Requires groupwise quantization, got block_size: {weight_tensor.block_size}"
    assert input_tensor.shape[-1] == weight_tensor.shape[1], (
        f"need input_tensor shape: {input_tensor.shape} final dim to match weight_tensor shape: {weight_tensor.shape} second dim ")
    if weight_tensor.act_pre_scale is not None:
        input_tensor = input_tensor * weight_tensor.act_pre_scale
    orig_act_size = input_tensor.size()
    orig_dtype = input_tensor.dtype
    act = input_tensor.reshape(-1, input_tensor.shape[-1]).to(torch.bfloat16)
    k_padded = weight_tensor.qdata.shape[1] * 128
    if act.shape[-1] != k_padded:
        act = torch.nn.functional.pad(act, (0, k_padded - act.shape[-1]))
    # a column slice of a wider buffer (e.g. the q part of a fused q|k|v output) goes to the kernel as is: its TMA
    # descriptor carries the row pitch; anything else is made contiguous like the reference does (:278-282)
    # (alignment from the storage offset, not data_ptr(): the handler must stay traceable with fake tensors)
    if not (act.stride(-1) == 1 and act.stride(0) >= act.shape[-1] and act.stride(0) % 8 == 0 and act.storage_offset() % 8 == 0):
        act = act.contiguous()
    n_out = weight_tensor.shape[-2]
    if act.numel() == 0:
        y = act.new_empty(act.shape[0], n_out)
    else:
        # one fused kernel: GEMM + out-feature slice + bias (the reference runs them separately)
        y = torch.ops.ao_b200.int4_tilepacked_linear(act, weight_tensor.qdata, weight_tensor.block_size[-1],
                                                     weight_tensor.scale_and_zero, bias, n_out, 0)
    y = y.reshape(*orig_act_size[:-1], n_out)
    return y.to(orig_dtype)


@implements(aten.slice.Tensor)
def _(func, types, args, kwargs):
    """Slicing on the packed layout, for TP-style weight loaders (reference :302-360)."""
    self, dim, start, end, step = fill_defaults(args, 5, [0, None, None, 1])
    assert step == 1 and dim in (0, 1), "only unit-step slicing of dim 0/1 is supported"
    N, K = self.shape
    start = 0 if start is None else start
    end = (N if dim == 0 else K) if end is None or end > (N if dim == 0 else K) else end
    g = self.block_size[-1]
    if dim == 0:
        assert start % 8 == 0 and end % 8 == 0, "dim-0 slices must be multiples of 8 rows (n-tile)"
        qd = self.qdata[start // 8: end // 8]
        sz = self.scale_and_zero[:, start:end]
        shape = torch.Size([end - start, K])
    else:
        assert start % 1024 == 0 and end % 1024 == 0, "dim-1 slices must be multiples of 1024 (K padding unit)"
        qd = self.qdata[:, start // 128: end // 128]
        sz = self.scale_and_zero[start // g: end // g]
        shape = torch.Size([N, end - start])
    # views, like the reference (:302-360): `param.data.narrow(...).copy_(loaded.narrow(...))` must write through to the
    # parameter's own storage; callers that run a linear on a slice make it contiguous first (the handler asserts it)
    return return_and_correct_aliasing(
        func, args, kwargs, Int4TilePackedTo4dTensor(qd, sz, self.block_size, shape, self.act_pre_scale))


@implements(aten.select.int)
def _(func, types, args, kwargs):
    """Expert `index` of a 3-D weight as a 2-D tensor (reference :365-385), which the dense linear serves: the MoE
    expert loop's `F.linear(x, w[e])`."""
    self, dim, index = args
    assert dim == 0, f"Int4TilePackedTo4dTensor aten.select.int with {dim=} is not yet supported"
    assert self.qdata.dim() == 5, "Int4TilePackedTo4dTensor aten.select.int: 3-D expert weights only"
    assert not self._is_transposed(), "Int4TilePackedTo4dTensor aten.select.int: select the expert before transposing"
    return return_and_correct_aliasing(
        func, args, kwargs, Int4TilePackedTo4dTensor(self.qdata[index], self.scale_and_zero[index],
                                                     list(self.block_size[1:]), torch.Size(self.shape[1:]),
                                                     self.act_pre_scale))


@implements(aten.transpose.int)
def _(func, types, args, kwargs):
    """The [E, K, N] view of a 3-D expert weight, how torch._grouped_mm receives it: the same qdata and scale_and_zero,
    shape and block_size ([1, g, 1]) transposed.  Transposing again gives back the stored form."""
    self, dim0, dim1 = args
    assert self.qdata.dim() == 5, f"Int4TilePackedTo4dTensor transpose: 3-D expert weights only, got shape {tuple(self.shape)}"
    assert (dim0, dim1) in ((1, 2), (2, 1), (-1, -2), (-2, -1)), f"transpose unsupported for {dim0=} {dim1=}"
    E, a, b = self.shape
    bs = list(self.block_size)
    new = Int4TilePackedTo4dTensor(self.qdata, self.scale_and_zero, [bs[0], bs[2], bs[1]], torch.Size([E, b, a]),
                                   self.act_pre_scale)
    return return_and_correct_aliasing(func, args, kwargs, new)


@implements(aten._grouped_mm.default)
def _(func, types, args, kwargs):
    """torch._grouped_mm(x, W.transpose(-2, -1), offs=offs) with a 3-D expert weight W [E, N, K]: expert e's rows
    [offs[e-1], offs[e]) of the bf16 x times its weights, dequantized inside one grouped wgmma kernel.  x is scaled by
    act_pre_scale and padded to the packed K as the linear does; rows from offs[-1] on are left unwritten, as torch
    leaves them.  Only the 2-D x 3-D form with offs, no bias and a bf16 output."""
    mat_a, mat_b = args[0], args[1]
    offs = args[2] if len(args) > 2 else kwargs.get("offs", None)
    bias = args[3] if len(args) > 3 else kwargs.get("bias", None)
    out_dtype = args[4] if len(args) > 4 else kwargs.get("out_dtype", None)
    if not isinstance(mat_b, Int4TilePackedTo4dTensor) or isinstance(mat_a, Int4TilePackedTo4dTensor):
        raise NotImplementedError("Int4TilePackedTo4dTensor _grouped_mm: only a bf16 mat_a times an int4 mat_b")
    if mat_a.dim() != 2 or mat_b.dim() != 3:
        raise NotImplementedError(f"Int4TilePackedTo4dTensor _grouped_mm: only 2-D mat_a x 3-D mat_b, got "
                                  f"{mat_a.dim()}-D x {mat_b.dim()}-D")
    if offs is None:
        raise NotImplementedError("Int4TilePackedTo4dTensor _grouped_mm: offs is required")
    if bias is not None:
        raise NotImplementedError("Int4TilePackedTo4dTensor _grouped_mm: bias is not supported")
    if out_dtype not in (None, torch.bfloat16) or mat_a.dtype != torch.bfloat16:
        raise NotImplementedError(f"Int4TilePackedTo4dTensor _grouped_mm: bf16 mat_a and output only, got "
                                  f"{mat_a.dtype} -> {out_dtype}")
    if not mat_b._is_transposed():
        raise NotImplementedError("Int4TilePackedTo4dTensor _grouped_mm: mat_b must be the transposed [E, N, K] weight "
                                  "(w.transpose(-2, -1))")
    E, K, N = mat_b.shape
    if mat_a.shape[-1] != K:
        raise ValueError(f"_grouped_mm: mat_a has K={mat_a.shape[-1]}, mat_b K={K}")
    x = mat_a
    if mat_b.act_pre_scale is not None:
        x = x * mat_b.act_pre_scale
    k_padded = mat_b.qdata.shape[2] * 128
    if x.shape[-1] != k_padded:
        x = torch.nn.functional.pad(x, (0, k_padded - x.shape[-1]))
    return torch.ops.ao_b200.int4_tilepacked_grouped_mm(x, mat_b.qdata, max(mat_b.block_size),
                                                        mat_b.scale_and_zero, offs.to(torch.int32), N)


Int4TilePackedTo4dTensor.__module__ = "ao_b200.quantization"
torch.serialization.add_safe_globals([Int4TilePackedTo4dTensor])
