"""Helpers shared by the workflows (reference: torchao/quantization/utils.py)."""
from __future__ import annotations

from typing import Tuple

import torch

from .granularity import PerAxis, PerBlock, PerGroup, PerRow, PerTensor, PerToken

__all__ = ["compute_error", "pack_tinygemm_scales_and_zeros", "unpack_tinygemm_scales_and_zeros", "get_block_size"]


def compute_error(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """SQNR in dB: 20*log10(|x| / |x-y|) (reference :59-62)."""
    Ps = torch.linalg.norm(x.float())
    Pn = torch.linalg.norm((x - y).float())
    return 20 * torch.log10(Ps / Pn)


def pack_tinygemm_scales_and_zeros(scales: torch.Tensor, zeros: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """[N, K/g] x 2 -> [K/g, N, 2] (reference :299-313)."""
    assert scales.shape == zeros.shape and scales.dtype == dtype and zeros.dtype == dtype
    return torch.stack([scales, zeros], dim=-1).transpose(-3, -2).contiguous()


def unpack_tinygemm_scales_and_zeros(scale_and_zero: torch.Tensor):
    assert scale_and_zero.dim() == 3 and scale_and_zero.shape[2] == 2
    sz = scale_and_zero.transpose(0, 1)
    return sz[..., 0].contiguous(), sz[..., 1].contiguous()


def get_block_size(input_shape: Tuple[int, ...], granularity) -> Tuple[int, ...]:
    """elements per quantization block along each dim (reference :589-633)."""
    if isinstance(granularity, PerBlock):
        # a shorter block size applies to the trailing dims: padded with leading ones (reference :603-611)
        bs = (1,) * (len(input_shape) - len(granularity.block_size)) + tuple(granularity.block_size)
        assert len(bs) == len(input_shape), f"Block size {bs} must have the same number of dimensions as input shape {input_shape}"
        return bs
    if isinstance(granularity, PerTensor):
        return tuple(input_shape)
    if isinstance(granularity, PerAxis):
        bs = list(input_shape)
        bs[granularity.axis] = 1
        return tuple(bs)
    if isinstance(granularity, (PerRow, PerToken)):
        dim = getattr(granularity, "dim", -1)
        bs = [1] * len(input_shape)
        bs[dim] = input_shape[dim]
        return tuple(bs)
    if isinstance(granularity, PerGroup):
        assert input_shape[-1] % granularity.group_size == 0
        return (1,) * (len(input_shape) - 1) + (granularity.group_size,)
    raise ValueError(f"Unsupported Granularity: {granularity}")
