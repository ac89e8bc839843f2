"""int4 weight in the tinygemm tile-packed layout, served by the sm_90a wgmma kernel.

Same class / attribute names and on-disk layout as the reference
(torchao/quantization/quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py): ``qdata`` int32
[N/8, K/128, 32, 4], ``scale_and_zero`` bf16 [K/g, N, 2], ``block_size``, ``shape``,
optional ``act_pre_scale``.  What changes is underneath: packing calls
``torch.ops.ao_b200.int4_pack_tile4d`` (instead of aten._convert_weight_to_int4pack, :202) and
the linear calls ``torch.ops.ao_b200.int4_tilepacked_linear`` (instead of
aten._weight_int4pack_mm + pad/slice/bias kernels, :278-299).
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
        assert hp_tensor.dim() == 2, "Int4TilePackedTo4dTensor: 2-D weights only"
        if not hp_tensor.is_cuda:
            # same exception type as the reference, where aten::_convert_weight_to_int4pack has no CPU kernel
            # (test_int4_tile_packed_to_4d_tensor.py:194-202)
            raise NotImplementedError("Could not run 'ao_b200::int4_pack_tile4d' with arguments from the 'CPU' backend: "
                                      "Int4TilePackedTo4dTensor.from_hp needs a CUDA tensor (sm_90a packing kernel)")
        original_shape = hp_tensor.shape
        N0, K0 = original_shape
        g = block_size[-1]
        K = find_multiple(K0, 1024)
        N = find_multiple(N0, ntile_size or 8)
        w = torch.nn.functional.pad(hp_tensor, (0, K - K0, 0, N - N0))
        if int4_choose_qparams_algorithm == Int4ChooseQParamsAlgorithm.HQQ:
            # reference :149-167 -> _choose_qparams_and_quantize_affine_hqq (quant_primitives.py:1797-2002); here one
            # CUDA solver (ao_b200/csrc/int4_hqq.cu), scale / zero already in the tinygemm convention
            q, scale, zero = torch.ops.ao_b200.int4_hqq_quantize(w.contiguous(), g)
            q = q.to(torch.int32)
        else:
            assert int4_choose_qparams_algorithm == Int4ChooseQParamsAlgorithm.TINYGEMM, (
                f"Unsupported Int4ChooseQParamsAlgorithm: {int4_choose_qparams_algorithm}")
            scale, zero = choose_qparams_affine_tinygemm(w, g)
            q = quantize_affine_tinygemm(w, g, scale, zero)
        q_u8 = (q[:, ::2] << 4 | q[:, 1::2]).to(torch.uint8).contiguous()
        qdata = torch.ops.ao_b200.int4_pack_tile4d(q_u8, INNER_K_TILES)
        scale_and_zero = pack_tinygemm_scales_and_zeros(scale, zero, scale.dtype)
        return cls(qdata=qdata, scale_and_zero=scale_and_zero, block_size=list(block_size), shape=original_shape,
                   act_pre_scale=None)

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """bf16((q-8)*s+z) for the original (unpadded) shape."""
        w = torch.ops.ao_b200.int4_dequant_tile4d(self.qdata, self.scale_and_zero, self.block_size[-1])
        w = w[: self.shape[0], : self.shape[1]]
        return w if output_dtype in (None, torch.bfloat16) else w.to(output_dtype)


implements = Int4TilePackedTo4dTensor.implements
implements_torch_function = Int4TilePackedTo4dTensor.implements_torch_function


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    input_tensor, weight_tensor, bias = args[0], args[1], args[2] if len(args) > 2 else None
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


Int4TilePackedTo4dTensor.__module__ = "ao_b200.quantization"
torch.serialization.add_safe_globals([Int4TilePackedTo4dTensor])
