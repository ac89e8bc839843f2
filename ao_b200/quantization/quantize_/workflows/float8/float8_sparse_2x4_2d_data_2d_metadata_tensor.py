"""2:4-sparse e4m3 weight with per-row scales, dynamic per-token e4m3 activations, sm_90a sparse wgmma GEMM.

Attribute names, order and shape match torchao's Float8Sparse2x4_2DData2DMetadataTensor
(torchao/quantization/quantize_/workflows/float8/float8_sparse_2x4_2d_data_2d_metadata_tensor.py).  The weight codes
and scales are the dense ``PerRow`` ``Float8Tensor``'s; the codes are then compressed into CUTLASS's Sm90 2:4 layout:

* ``qdata`` e4m3 ``[N, K/2]``: the two stored codes of each group of 4 k;
* ``sparse_metadata`` uint8 ``[round_up(N, 64), round_up(K, 128) / 8]``: one nibble per group (the two kept positions,
  first in bits 1:0), two groups per byte (the first in the low nibble), in atoms of 64 rows x 128 k (16 bytes per row,
  rows in order), the atoms along N first and then along K (DESIGN §2g).

The compression is plain tensor arithmetic (it runs once per weight, on any device) and writes what the reference's
``to_sparse_semi_structured_cutlass_sm9x_f8`` writes, byte for byte, for every 2:4-sparse code matrix: a group with one
stored code keeps it with a zero at position 3 (or at 0, when the code is at 3), an all-zero group is ``0b0000`` with
two zero codes, the padding is zero, and e4m3 ``-0.0`` counts as zero.  A group with more than two nonzero codes raises
``ValueError`` (the reference's compressor leaves its output unspecified there).

The linear is two launches: the per-token e4m3 quantizer of the dense rowwise path and ``fp8_sparse_linear``, which
computes the reference's CUTLASS epilogue as its build compiles it, ``bf16(fma(acc * w_scale[n], x_scale[m], bias[n]))``.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from ao_b200.float8.inference import FP8Granularity
from ao_b200.quantization.granularity import PerRow
from ao_b200.utils import TorchAOBaseTensor, rows_for_kernel

from .float8_tensor import Float8Tensor, QuantizeTensorToFloat8Kwargs

__all__ = ["Float8Sparse2x4_2DData2DMetadataTensor"]
aten = torch.ops.aten


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def compress_2x4_e4m3(q: torch.Tensor):
    """e4m3 codes ``[N, K]`` (2:4 sparse along K, K % 4 == 0) -> (``qdata`` e4m3 ``[N, K/2]``, ``sparse_metadata`` uint8
    ``[round_up(N, 64), round_up(K, 128) / 8]``) in CUTLASS's Sm90 layout (module docstring)."""
    if q.dim() != 2 or q.dtype != torch.float8_e4m3fn:
        raise ValueError(f"2:4 compression needs 2-D float8_e4m3fn codes, got {tuple(q.shape)} {q.dtype}")
    N, K = q.shape
    if K % 4 != 0:
        raise ValueError(f"2:4 compression needs K % 4 == 0, got K={K}")
    u = q.contiguous().view(torch.uint8).reshape(N, K // 4, 4)
    nz = (u & 0x7F) != 0
    cnt = nz.sum(-1)
    bad = cnt > 2
    if bool(bad.any()):
        row, grp = (int(v) for v in bad.nonzero()[0])
        raise ValueError(f"weight is not 2:4 sparse: row {row}, group {grp} (k {4 * grp}..{4 * grp + 3}) has "
                         f"{int(cnt[row, grp])} nonzero codes; prune the weight to two nonzeros per four first")
    pos = torch.arange(4, device=u.device, dtype=torch.int64)
    first = torch.where(nz, pos, 4).amin(-1)
    last = torch.where(nz, pos, -1).amax(-1)
    three = torch.full_like(first, 3)
    zero = torch.zeros_like(first)
    # two codes: (first, last); one code at p < 3: (p, 3); one at 3: (0, 3); none: (0, 0)
    i0 = torch.where(cnt == 2, first, torch.where((cnt == 1) & (first < 3), first, zero))
    i1 = torch.where(cnt == 2, last, torch.where(cnt == 1, three, zero))
    ucode = torch.where(nz, u, torch.zeros_like(u))   # -0.0 is never stored
    v0 = ucode.gather(-1, i0.unsqueeze(-1)).squeeze(-1)
    v1 = ucode.gather(-1, i1.unsqueeze(-1)).squeeze(-1)
    qdata = torch.stack([v0, v1], -1).reshape(N, K // 2).view(torch.float8_e4m3fn)
    nib = (i0 | (i1 << 2)).to(torch.uint8)                                   # [N, K/4]
    if (K // 4) % 2:
        nib = torch.cat([nib, torch.zeros_like(nib[:, :1])], 1)
    byte = nib[:, 0::2] | (nib[:, 1::2] << 4)                               # [N, ceil(K/8)]
    Np, Kp = _round_up(N, 64), _round_up(K, 128)
    rows = torch.zeros(Np, Kp // 8, dtype=torch.uint8, device=u.device)
    rows[:N, : byte.shape[1]] = byte
    meta = rows.reshape(Np // 64, 64, Kp // 128, 16).permute(2, 0, 1, 3).contiguous().reshape(Np, Kp // 8)
    return qdata, meta


def metadata_rows(meta: torch.Tensor) -> torch.Tensor:
    """The atom-ordered ``sparse_metadata`` as plain rows: ``[round_up(N, 64), round_up(K, 128) / 8]`` with byte
    ``[n, k / 8]`` the nibbles of groups k/4 and k/4 + 1 of row n."""
    Np, kb = meta.shape
    return meta.reshape(kb // 16, Np // 64, 64, 16).permute(1, 2, 0, 3).reshape(Np, kb)


def decompress_2x4_e4m3(qdata: torch.Tensor, meta: torch.Tensor) -> torch.Tensor:
    """Inverse of :func:`compress_2x4_e4m3`: the e4m3 codes ``[N, K]`` (positions not stored are +0)."""
    N, K = qdata.shape[0], 2 * qdata.shape[1]
    rows = metadata_rows(meta)[:N, : (K + 7) // 8]
    nib = torch.stack([rows & 0xF, rows >> 4], -1).reshape(N, -1)[:, : K // 4].to(torch.int64)
    v = qdata.contiguous().view(torch.uint8).reshape(N, K // 4, 2)
    out = torch.zeros(N, K // 4, 4, dtype=torch.uint8, device=qdata.device)
    # the second code last: an all-zero group names position 0 twice and stores two zeros
    out.scatter_(-1, (nib & 3).unsqueeze(-1), v[..., :1])
    out.scatter_(-1, (nib >> 2).unsqueeze(-1), v[..., 1:])
    return out.reshape(N, K).view(torch.float8_e4m3fn)


class Float8Sparse2x4_2DData2DMetadataTensor(TorchAOBaseTensor):
    """2:4-sparse e4m3 weight in CUTLASS's Sm90 layout with a per-row scale ``[N, 1]``; logical shape ``[N, K]``."""

    tensor_data_names = ["qdata", "sparse_metadata", "scale"]
    tensor_attribute_names = []
    optional_tensor_attribute_names = ["block_size", "act_quant_kwargs", "dtype"]

    def __new__(cls, qdata, sparse_metadata, scale, block_size: Optional[List[int]] = None,
                act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None, dtype: Optional[torch.dtype] = None):
        shape = qdata.shape[0], 2 * qdata.shape[1]
        return torch.Tensor._make_wrapper_subclass(cls, shape, device=qdata.device, dtype=dtype, requires_grad=False)

    def __init__(self, qdata, sparse_metadata, scale, block_size=None, act_quant_kwargs=None, dtype=None):
        super().__init__()
        self.qdata = qdata
        self.sparse_metadata = sparse_metadata
        self.scale = scale
        self.block_size = block_size
        self.act_quant_kwargs = act_quant_kwargs

    def _quantization_type(self):
        return f"{self.act_quant_kwargs=}, {self.block_size=}, {self.scale.shape=}"

    def dequantize(self, output_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """bf16(fp32(q) * scale[n]), then ``output_dtype``: the reference runs its sparse GEMM on an identity matrix
        with a bf16 output, so even a float32 dequantize is bf16-rounded."""
        q = decompress_2x4_e4m3(self.qdata, self.sparse_metadata)
        dense = (q.float() * self.scale.reshape(-1, 1).float()).to(torch.bfloat16)
        return dense.to(output_dtype or self.dtype)

    def to(self, *args, **kwargs):
        """``.to(dtype)`` dequantizes, as the reference's aten.to.dtype / to.dtype_layout do; a device move keeps the
        packed form"""
        kw = self._get_to_kwargs(*args, **kwargs)
        if kw["dtype"] != self.dtype:
            return self.dequantize().to(dtype=kw["dtype"], device=kw["device"])
        return super().to(*args, **kwargs)

    @classmethod
    def from_hp(cls, hp_tensor: torch.Tensor, float8_dtype: torch.dtype = torch.float8_e4m3fn,
                granularity: FP8Granularity = PerRow(), hp_value_lb: Optional[float] = None,
                hp_value_ub: Optional[float] = None, act_quant_kwargs: Optional[QuantizeTensorToFloat8Kwargs] = None):
        # the reference's assertions (float8_sparse_2x4_2d_data_2d_metadata_tensor.py, from_hp)
        assert isinstance(granularity, PerRow), "CUTLASS sparse kernel only supports per-row quantization"
        assert granularity.dim in (-1, len(hp_tensor.shape) - 1), \
            "CUTLASS sparse kernel only supports quantizing along the last dimension"
        assert float8_dtype == torch.float8_e4m3fn, "CUTLASS sparse kernel only supports float8_e4m3fn dtype"
        assert hp_value_lb is None, "CUTLASS sparse kernel does not support hp_value_lb"
        if hp_tensor.dim() != 2:
            raise NotImplementedError(f"2:4-sparse float8 weights are 2-D, got {tuple(hp_tensor.shape)}")
        dense = Float8Tensor.from_hp(hp_tensor, float8_dtype, granularity, hp_value_lb=hp_value_lb,
                                     hp_value_ub=hp_value_ub)
        qdata, meta = compress_2x4_e4m3(dense.qdata)
        return cls(qdata, meta, dense.scale, block_size=list(dense.block_size), act_quant_kwargs=act_quant_kwargs,
                   dtype=hp_tensor.dtype)


implements = Float8Sparse2x4_2DData2DMetadataTensor.implements
implements_torch_function = Float8Sparse2x4_2DData2DMetadataTensor.implements_torch_function


def _sparse_linear(x: torch.Tensor, w: Float8Sparse2x4_2DData2DMetadataTensor, bias: Optional[torch.Tensor]):
    kw = w.act_quant_kwargs
    if kw is None:
        raise NotImplementedError("2:4-sparse float8 linear: the weight has no activation quantization "
                                  "(act_quant_kwargs); the reference has no weight-only sparse path either")
    assert not isinstance(x, TorchAOBaseTensor), "input tensor was already quantized"
    if x.dtype != torch.bfloat16 or w.dtype != torch.bfloat16:
        raise NotImplementedError(f"2:4-sparse float8 linear: bf16 activations and a weight quantized from bf16 only, "
                                  f"got {x.dtype} activations and a {w.dtype} weight")
    N, K = w.shape
    out_shape = (*x.shape[:-1], N)
    x2 = x.reshape(-1, K)
    if x2.shape[0] == 0:
        return x.new_empty(out_shape)
    xq = Float8Tensor.from_hp(rows_for_kernel(x2), kw.float8_dtype, kw.granularity, kw.mm_config, kw.hp_value_lb,
                              kw.hp_value_ub, kw.kernel_preference)
    y = torch.ops.ao_b200.fp8_sparse_linear(xq.qdata.contiguous(), xq.scale.reshape(-1).float().contiguous(), w.qdata,
                                            w.sparse_metadata, w.scale.reshape(-1).float().contiguous(), bias)
    return y.reshape(out_shape)


@implements(aten.linear.default)
@implements_torch_function(torch.nn.functional.linear)
def _(func, types, args, kwargs):
    x = kwargs.get("input", args[0] if len(args) > 0 else None)
    w = kwargs.get("weight", args[1] if len(args) > 1 else None)
    bias = kwargs.get("bias", args[2] if len(args) > 2 else None)
    return _sparse_linear(x, w, bias)


@implements(aten.to.dtype_layout)
def _(func, types, args, kwargs):
    return args[0].dequantize().to(*args[1:], dtype=kwargs.get("dtype", args[0].dtype),
                                   device=kwargs.get("device", args[0].device))


@implements(aten.to.dtype)
def _(func, types, args, kwargs):
    dtype = kwargs.get("dtype", args[1] if len(args) > 1 else None)
    assert dtype is not None, "dtype must not be None"
    return args[0].dequantize().to(dtype=dtype)


torch.serialization.add_safe_globals([Float8Sparse2x4_2DData2DMetadataTensor])
