"""fp8 inference helpers (reference: torchao/float8/inference.py:26-39, :177-265)."""
from typing import List, NamedTuple, Optional, Tuple, Union

import torch

from ao_b200.quantization.granularity import PerBlock, PerRow, PerTensor


class Float8MMConfig(NamedTuple):
    """Matmul options carried by Float8Tensor; ``use_fast_accum`` is accepted for compatibility --
    the wgmma kernel sums every 128-k chunk into fp32 registers."""

    emulate: bool = False
    use_fast_accum: bool = False
    pad_inner_dim: bool = False


FP8Granularity = Union[PerTensor, PerRow, PerBlock]


def _is_rowwise_scaled(block_size, shape) -> bool:
    return tuple(block_size) == (1,) * (len(shape) - 1) + (shape[-1],)


def _is_tensorwise_scaled(block_size, shape) -> bool:
    return all(int(b) in (-1, int(s)) for b, s in zip(block_size, shape))


def _normalize_granularity(granularity) -> Tuple[FP8Granularity, FP8Granularity]:
    if granularity is None:
        return PerTensor(), PerTensor()
    if isinstance(granularity, (PerTensor, PerRow)):
        return granularity, granularity
    if isinstance(granularity, (tuple, list)) and len(granularity) == 2:
        a, w = granularity
        ok = (isinstance(a, PerTensor) and isinstance(w, PerTensor)) or (isinstance(a, PerRow) and isinstance(w, PerRow))
        if not ok:
            raise ValueError(f"Unsupported granularity types: {granularity}, only PerTensor or PerRow pairs are supported.")
        return a, w
    raise ValueError(f"Invalid granularity specification: {granularity}")
