"""Scale-layout helpers (reference: torchao/prototype/mx_formats/utils.py:25-134)."""
import torch


def ceil_div(a, b):
    return (a + b - 1) // b


def to_blocked(input_matrix: torch.Tensor) -> torch.Tensor:
    """[H, W] -> flat 32*ceil(H/128) x 16*ceil(W/4): the cuBLAS block-scale layout
    (each 128x4 tile becomes 32 rows of 16 bytes: (r%32)*16 + (r/32)*4 + c)."""
    rows, cols = input_matrix.shape
    rb, cb = ceil_div(rows, 128), ceil_div(cols, 4)
    padded = input_matrix
    if (rows, cols) != (rb * 128, cb * 4):
        padded = torch.zeros((rb * 128, cb * 4), device=input_matrix.device, dtype=input_matrix.dtype)
        padded[:rows, :cols] = input_matrix
    blocks = padded.view(rb, 128, cb, 4).permute(0, 2, 1, 3)
    return blocks.reshape(-1, 4, 32, 4).transpose(1, 2).reshape(-1, 32, 16).flatten()


def from_blocked(blocked: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
    rb, cb = ceil_div(rows, 128), ceil_div(cols, 4)
    t = blocked.reshape(rb * cb, 32, 4, 4).transpose(1, 2).reshape(rb, cb, 128, 4).permute(0, 2, 1, 3)
    return t.reshape(rb * 128, cb * 4)[:rows, :cols]


def hp_data_dims_to_swizzled_scale_dims_mx(M, K):
    return ceil_div(M, 128) * 32, ceil_div(K // 32, 4) * 16


def hp_data_dims_to_swizzled_scale_dims_nvfp4(M, K):
    return ceil_div(M, 128) * 32, ceil_div(K // 16, 4) * 16


def slice_qdata_and_scale(x, dim: int, start, end):
    """Row / column slice of an MXTensor or NVFP4Tensor payload: (qdata, scale) of ``x[start:end]`` along ``dim``.

    Semantics of the reference's `_swizzle_aware_slice` (`torchao/prototype/mx_formats/utils.py:247-462`, used by
    `aten.slice` of both classes, i.e. by `narrow`-based tensor-parallel weight loaders):
    * plain (row-major) scales: rows slice freely, columns at multiples of ``block_size`` (and of 2 for packed fp4);
    * blocked ("swizzled") scales are made of 128-row x 4-scale-column tiles of 512 bytes, so rows slice at multiples
      of 128 (or up to the end) and columns at multiples of ``4 * block_size`` (64 elements for nvfp4); whole tiles
      are kept, nothing is re-swizzled.
    The reference hard-codes nvfp4's 16 / 64 in the blocked column case; for block 32 (mxfp8) this function uses
    ``4 * block_size`` = 128, which is what the layout requires.
    """
    import sys

    aten = torch.ops.aten
    M, K = x.shape[-2], x.shape[-1]
    bs = x.block_size
    packed = x.qdata.dtype == torch.uint8  # two e2m1 codes per byte
    size = M if dim == 0 else K
    start = 0 if start is None else start
    end = size if end is None or end == sys.maxsize or end > size else end
    if dim not in (0, 1):
        raise ValueError(f"{type(x).__name__} only supports slicing along dimensions 0 and 1, got dim={dim}")
    if dim == 1 and packed and (start % 2 or (end != K and end % 2)):
        raise RuntimeError(f"slice [{start}:{end}] must be even for FP4 packing")
    q_lo, q_hi = (start // 2, end // 2) if (dim == 1 and packed) else (start, end)
    qdata = aten.slice.Tensor(x.qdata, dim, q_lo, q_hi, 1)
    cols = K // bs
    if x.is_swizzled_scales:
        rb, cb = ceil_div(M, 128), ceil_div(cols, 4)
        tiles = x.scale.reshape(rb, cb, 512)
        if dim == 0:
            if start % 128:
                raise RuntimeError(f"Row slicing of {type(x).__name__} with swizzled scales requires start index to be a "
                                   f"multiple of 128, got {start}")
            if end != M and end % 128:
                raise RuntimeError(f"Row slicing of {type(x).__name__} with swizzled scales requires end index to be a "
                                   f"multiple of 128 or equal to tensor size {M}, got {end}")
            tiles = tiles[start // 128: ceil_div(end, 128)]
        else:
            span = 4 * bs
            if start % span:
                raise RuntimeError(f"Column slicing of {type(x).__name__} with swizzled scales requires start index to be "
                                   f"a multiple of {span}, got {start}")
            if end != K and end % span:
                raise RuntimeError(f"Column slicing of {type(x).__name__} with swizzled scales requires end index to be a "
                                   f"multiple of {span} or equal to tensor size {K}, got {end}")
            tiles = tiles[:, start // span: ceil_div(end // bs, 4)]
        new_m, new_k = end - start if dim == 0 else M, end - start if dim == 1 else K
        dims = hp_data_dims_to_swizzled_scale_dims_nvfp4(new_m, new_k) if bs == 16 else hp_data_dims_to_swizzled_scale_dims_mx(new_m, new_k)
        scale = tiles.reshape(dims)
    else:
        plain = x.scale.reshape(M, cols)
        if dim == 0:
            scale = aten.slice.Tensor(plain, 0, start, end, 1)
        else:
            assert start % bs == 0, f"Start index {start} must be a multiple of block_size {bs}"
            assert end % bs == 0, f"End index {end} must be a multiple of block_size {bs}"
            scale = aten.slice.Tensor(plain, 1, start // bs, end // bs, 1)
    return qdata, scale
