"""fp8 inference helpers (reference: torchao/float8/inference.py:26-39, :177-265)."""
import math
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


def _is_1_128_scaled(block_size) -> bool:
    """1x128 blocks along the last dim (the blockwise recipe's activations; reference :197-204)."""
    return len(block_size) >= 2 and math.prod(block_size[:-1]) == 1 and block_size[-1] == 128


def _is_128_128_scaled(block_size) -> bool:
    """128x128 blocks of a 2-D weight (the blockwise recipe's weights; reference :207-214)."""
    return len(block_size) == 2 and block_size[0] == 128 and block_size[1] == 128


def _is_1_128_128_scaled(block_size) -> bool:
    """128x128 blocks of each expert of a 3-D weight [E, N, K] (or its transposed view), block_size [1, 128, 128]."""
    return len(block_size) == 3 and block_size[0] == 1 and block_size[1] == 128 and block_size[2] == 128


def _granularity_is_a_1_128_w_128_128(g) -> bool:
    """The blockwise pair, by the dataclasses' equality as the reference compares it (reference :217-228): the block
    sizes are compared as given, so PerBlock([1, 128]) matches and PerBlock((1, 128)) does not."""
    return len(g) == 2 and g[0] == PerBlock([1, 128]) and g[1] == PerBlock([128, 128])


def _normalize_granularity(granularity) -> Tuple[FP8Granularity, FP8Granularity]:
    if granularity is None:
        return PerTensor(), PerTensor()
    if isinstance(granularity, (PerTensor, PerRow)):
        return granularity, granularity
    if isinstance(granularity, (tuple, list)) and len(granularity) == 2:
        a, w = granularity
        ok = ((isinstance(a, PerTensor) and isinstance(w, PerTensor)) or (isinstance(a, PerRow) and isinstance(w, PerRow))
              or _granularity_is_a_1_128_w_128_128(granularity))
        if not ok:
            raise ValueError(f"Unsupported granularity types: {granularity}, only PerTensor or PerRow pairs and "
                             f"[PerBlock([1, 128]), PerBlock([128, 128])] are supported.")
        return a, w
    raise ValueError(f"Invalid granularity specification: {granularity}")
