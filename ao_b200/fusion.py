"""Run quantized linears that share their input as ONE kernel launch.

``q_proj | k_proj | v_proj`` and ``gate_proj | up_proj`` of a transformer layer read the same activations.  At decode
sizes each of them is a few microseconds of weight streaming wrapped in a fixed per-launch cost (dependent-launch
latency, split-tile reduction), so launching them separately pays that cost three and two times over.  All five
weight formats of this engine store the out-feature dimension outermost (``qdata`` rows / ``[N/8]`` tiles, per-row or
per-block scales), so the packed tensors of such a group can be CONCATENATED along the out-feature dimension into one
packed weight of the same class -- the kernels and the checkpoint layout are unchanged, and for the dynamic-activation
formats the activations are also quantized once instead of once per projection.  This is what serving stacks do with
the reference's tensors as well (vLLM quantizes its merged QKV / gate-up parameters as one torchao tensor and loads
shards with ``narrow`` + ``copy_``; reference slicing support: torchao/testing/utils.py:471-519).

``fuse_parallel_linears(model)`` rewires the member ``nn.Linear`` modules in place:

* the group's packed weights (and biases) are concatenated once; every member keeps its own ``weight`` / ``bias``
  parameters, now VIEWS of the fused storage (``narrow`` + ``copy_`` loaders keep working and write through);
* a member's ``forward(x)`` returns its slice of the fused output.  The first member called with a given input runs
  the fused linear; the others recognise the same input (same storage, shape, strides and version counter) and
  reuse that result -- each member at most once per result, so the next forward pass (or CUDA-graph capture) over the
  same buffer runs again.  A member called alone, or with a different input, still returns the right values (the
  fused linear simply runs for it).

The returned slices are strided views ``[..., n_i]`` of the fused ``[..., sum n]`` output; this engine's linears take
a row-strided input directly (the TMA descriptor carries the row pitch), so feeding a slice to the next linear costs
no copy.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ["fuse_parallel_linears", "FusedLinearMember", "cat_out_features", "DEFAULT_GROUPS"]

DEFAULT_GROUPS: Tuple[Tuple[str, ...], ...] = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


def _same(a, b) -> bool:
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        return a is b or (isinstance(a, torch.Tensor) and isinstance(b, torch.Tensor) and a.shape == b.shape
                          and bool(torch.equal(a, b)))
    return a == b


def cat_out_features(ws: Sequence[torch.Tensor]) -> Optional[torch.Tensor]:
    """Concatenate packed weights of one class along the out-feature dimension; None when they cannot be merged
    (different class / K / quantization attributes, a layout that pads N, per-tensor scales that differ, or 128x128
    scale blocks with an N that is not a multiple of 128)."""
    from ao_b200.prototype.mx_formats.mx_tensor import MXTensor
    from ao_b200.prototype.mx_formats.nvfp4_tensor import NVFP4Tensor
    from ao_b200.quantization import Float8Tensor, Int4TilePackedTo4dTensor, Int8Tensor

    w0 = ws[0]
    cls = type(w0)
    if any(type(w) is not cls for w in ws) or any(w.dim() != 2 or w.shape[1] != w0.shape[1] for w in ws):
        return None
    n_total = sum(int(w.shape[0]) for w in ws)
    shape = torch.Size([n_total, int(w0.shape[1])])
    # every non-data attribute must agree across the group
    names = list(getattr(cls, "tensor_attribute_names", [])) + list(getattr(cls, "optional_tensor_attribute_names", []))
    for name in names:
        if name == "shape":
            continue
        if any(not _same(getattr(w, name, None), getattr(w0, name, None)) for w in ws[1:]):
            return None
    if cls is Int4TilePackedTo4dTensor:
        if any(w.qdata.shape[0] * 8 != w.shape[0] or w.act_pre_scale is not None for w in ws):
            return None   # N padded to the n-tile, or AWQ-style pre-scales (per linear)
        return cls(torch.cat([w.qdata for w in ws], 0).contiguous(), torch.cat([w.scale_and_zero for w in ws], 1).contiguous(),
                   list(w0.block_size), shape, None)
    if cls is Float8Tensor and all(list(w.block_size) == [128, 128] for w in ws):
        if any(w.shape[0] % 128 != 0 or w.scale.shape != (w.shape[0] // 128, w.shape[1] // 128) for w in ws):
            return None   # a 128x128 scale block would straddle two members
        return cls(torch.cat([w.qdata for w in ws], 0).contiguous(), torch.cat([w.scale for w in ws], 0).contiguous(),
                   block_size=[128, 128], mm_config=w0.mm_config, act_quant_kwargs=w0.act_quant_kwargs,
                   kernel_preference=w0.kernel_preference, dtype=w0.dtype)
    if cls in (Int8Tensor, Float8Tensor):
        rowwise = all(w.scale.dim() == 2 and w.scale.shape[0] == w.shape[0] and w.scale.shape[1] == 1 for w in ws)
        if not rowwise:
            return None   # per-tensor scales differ per projection
        qd = torch.cat([w.qdata for w in ws], 0).contiguous()
        sc = torch.cat([w.scale for w in ws], 0).contiguous()
        bs = [1, int(w0.shape[1])]
        if cls is Int8Tensor:
            if any(getattr(w, "act_pre_scale", None) is not None or getattr(w, "act_quant_scale", None) is not None for w in ws):
                return None
            zp = None if w0.zero_point is None else torch.cat([w.zero_point for w in ws], 0).contiguous()
            return cls(qd, sc, bs, w0.dtype, zero_point=zp, act_quant_kwargs=w0.act_quant_kwargs, reduce_range=w0.reduce_range)
        return cls(qd, sc, block_size=bs, mm_config=w0.mm_config, act_quant_kwargs=w0.act_quant_kwargs,
                   kernel_preference=w0.kernel_preference, dtype=w0.dtype)
    if cls in (MXTensor, NVFP4Tensor):
        if w0.is_swizzled_scales and any(w.shape[0] % 128 != 0 for w in ws):
            return None   # a blocked scale tile spans 128 rows
        pts = None
        if cls is NVFP4Tensor:
            from ao_b200.prototype.mx_formats.nvfp4_tensor import QuantizeTensorToFloat8ActKwargs

            has = [w.per_tensor_scale is not None for w in ws]
            if any(w.act_per_tensor_scale is not None for w in ws) or (any(has) and not all(has)):
                return None
            if all(has):
                # one fp32 scalar per member: the weight-only / fp8-activation kernel takes one scale per out-feature
                # (each member's scalar repeated over its rows); the nvfp4 x nvfp4 kernel folds a single scalar only
                if not (w0.act_quant_kwargs is None or isinstance(w0.act_quant_kwargs, QuantizeTensorToFloat8ActKwargs)):
                    return None
                pts = torch.cat([w.per_tensor_scale.reshape(-1).float().expand(int(w.shape[0])) for w in ws]).contiguous()
        qd = torch.cat([w.qdata for w in ws], 0).contiguous()
        # blocked layout: 512-byte tiles ordered [row block][column block] -> row blocks concatenate
        sc = torch.cat([w.scale.reshape(-1) if w0.is_swizzled_scales else w.scale for w in ws], 0).contiguous()
        if w0.is_swizzled_scales and w0.scale.dim() == 2:
            sc = sc.reshape(-1, w0.scale.shape[1])
        if cls is MXTensor:
            return cls(qd, sc, w0.elem_dtype, w0.block_size, w0.orig_dtype, w0.kernel_preference, w0.act_quant_kwargs,
                       w0.is_swizzled_scales)
        return cls(qd, sc, w0.block_size, w0.orig_dtype, pts, None, w0.is_swizzled_scales, w0.use_triton_kernel,
                   w0.act_quant_kwargs)
    return None


class _Group:
    """State shared by the members of one fused group (a plain object: not a registered submodule)."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], splits: List[int]):
        self.weight = weight
        self.bias = bias
        self.splits = splits
        self.offsets = [sum(splits[:i]) for i in range(len(splits))]
        self._key = None
        self._out = None
        self._served = set()

    @staticmethod
    def _key_of(x: torch.Tensor):
        return (x.data_ptr(), tuple(x.shape), tuple(x.stride()), x.dtype, x._version)

    def run(self, x: torch.Tensor, member: int) -> torch.Tensor:
        """Fused output for ``x`` on behalf of ``member``.  A cached result serves each member at most ONCE: the same
        buffer handed in again (next forward pass, next CUDA-graph capture, a replayed graph's static input -- its
        contents change without the version counter moving) is a new input and runs the fused linear again."""
        key = self._key_of(x)
        if self._key != key or self._out is None or member in self._served:
            self._out = F.linear(x, self.weight, self.bias)
            self._key = key
            self._served = set()
        self._served.add(member)
        return self._out


class FusedLinearMember(nn.Linear):
    """An ``nn.Linear`` whose weight is a view into a fused group weight; ``forward`` slices the group's output."""

    def __init__(self, group: _Group, index: int, weight_view: torch.Tensor, bias_view: Optional[torch.Tensor]):
        nn.Module.__init__(self)
        self.in_features = int(weight_view.shape[1])
        self.out_features = int(weight_view.shape[0])
        self.weight = nn.Parameter(weight_view, requires_grad=False)
        self.bias = None if bias_view is None else nn.Parameter(bias_view, requires_grad=False)
        object.__setattr__(self, "_group", group)
        self._index = index

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        g = self._group
        y = g.run(x, self._index)
        off = g.offsets[self._index]
        return y[..., off: off + g.splits[self._index]]

    def extra_repr(self) -> str:
        return f"{super().extra_repr()}, fused_member={self._index} of {len(self._group.splits)}"


def fuse_parallel_linears(model: nn.Module, groups: Iterable[Sequence[str]] = DEFAULT_GROUPS) -> int:
    """Fuse, in every submodule of ``model`` that has all the named children as quantized ``nn.Linear``s, each group
    into one launch.  Returns the number of groups fused; groups that cannot be merged are left untouched."""
    from ao_b200.utils import TorchAOBaseTensor

    fused = 0
    for parent in list(model.modules()):
        for names in groups:
            mods = [getattr(parent, n, None) for n in names]
            if any(not isinstance(m, nn.Linear) or isinstance(m, FusedLinearMember) for m in mods):
                continue
            ws = [m.weight.data if isinstance(m.weight, nn.Parameter) else m.weight for m in mods]
            if any(not isinstance(w, TorchAOBaseTensor) for w in ws):
                continue
            has_bias = [m.bias is not None for m in mods]
            if any(has_bias) and not all(has_bias):
                continue
            w_cat = cat_out_features(ws)
            if w_cat is None:
                continue
            b_cat = torch.cat([m.bias.data for m in mods], 0).contiguous() if all(has_bias) else None
            splits = [int(w.shape[0]) for w in ws]
            group = _Group(w_cat, b_cat, splits)
            off = 0
            for i, (name, n) in enumerate(zip(names, splits)):
                w_view = w_cat[off: off + n]
                b_view = None if b_cat is None else b_cat[off: off + n]
                setattr(parent, name, FusedLinearMember(group, i, w_view, b_view))
                off += n
            fused += 1
    return fused

