"""Activation layouts and Meta outputs of every dense linear op on the GPU.

* Quantized activations (int8, e4m3 and fp4 codes) are contiguous; a view that does not start on 16 bytes gives the
  bits of the same call on an aligned copy.
* bf16 activations may be row-strided: a column slice of a wider buffer gives the bits of the same call on a dense
  copy, and a view that does not start on 16 bytes is rejected.
* Each op's Meta kernel states the shape, dtype and strides of its CUDA output.
"""
import pytest
import torch

import exact_operands as ex

pytestmark = pytest.mark.gpu

M, N, K, G = 37, 256, 1024, 128


def cdiv(a, b):
    return (a + b - 1) // b


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


def _codes(dtype, n, g):
    """n random activation codes of one dtype (int8, e4m3, packed fp4 bytes, or bf16 values)"""
    if dtype == torch.int8:
        return ex.randint(-128, 127, (n,), g).to(torch.int8)
    if dtype == torch.uint8:
        return ex.randint(0, 255, (n,), g).to(torch.uint8)
    return torch.randn(n, device=ex.DEV, generator=g).to(dtype)


def _dense_ops(ops):
    """Every dense linear as name -> (activation dtype, activation columns, call(x, T)); T maps each other operand to
    the device the call runs on (identity, or to the meta device)."""
    g = ex.gen(21)
    f32 = lambda *s: torch.rand(*s, device=ex.DEV, generator=g) + 0.5   # noqa: E731
    xs, ws, bias = f32(M), f32(N), torch.randn(N, device=ex.DEV, generator=g).to(torch.bfloat16)
    w8 = ex.randint(-128, 127, (N, K), g).to(torch.int8)
    w_e4m3 = torch.randn(N, K, device=ex.DEV, generator=g).to(torch.float8_e4m3fn)
    xs_t, ws_b = f32(K // 128, cdiv(M, 4) * 4), f32(N // 128, K // 128)                # 1x128 and 128x128 scales
    w_sp = torch.randn(N, K // 2, device=ex.DEV, generator=g).to(torch.float8_e4m3fn)
    w_meta = torch.full((cdiv(N, 64) * 64, cdiv(K, 128) * 16), 0x44, dtype=torch.uint8, device=ex.DEV)  # positions 0, 1
    w_fp4 = ex.randint(0, 255, (N, K // 2), g).to(torch.uint8)
    mx_sf = lambda rows: ex.randint(120, 130, (512 * cdiv(rows, 128) * cdiv(K // 32, 4),), g).to(torch.uint8)  # noqa: E731
    nv_sf = lambda rows: ex.randint(0x30, 0x3F, (512 * cdiv(rows, 128) * cdiv(K // 16, 4),), g).to(torch.uint8)  # noqa: E731
    xs_mx, ws_mx, xs_nv, ws_nv = mx_sf(M), mx_sf(N), nv_sf(M), nv_sf(N)
    a_pts, b_pts = f32(1), f32(1)
    w4 = ex.randint(-2**31, 2**31 - 1, (N // 8, K // 128, 32, 4), g).to(torch.int32)
    sz = (torch.randn(K // G, N, 2, device=ex.DEV, generator=g) * 0.1).to(torch.bfloat16)
    i8, e4m3, u8, bf16 = torch.int8, torch.float8_e4m3fn, torch.uint8, torch.bfloat16
    return {
        "int8_dyn_linear": (i8, K, lambda x, T: ops.int8_dyn_linear(x, T(xs), T(w8), T(ws), T(bias))),
        "int8_weight_linear": (bf16, K, lambda x, T: ops.int8_weight_linear(x, T(w8), T(ws), T(bias))),
        "int8_mm_i32": (i8, K, lambda x, T: ops.int8_mm_i32(x, T(w8))),
        "fp8_rowwise_linear": (e4m3, K, lambda x, T: ops.fp8_rowwise_linear(x, T(xs), T(w_e4m3), T(ws), T(bias))),
        "fp8_static_linear": (e4m3, K, lambda x, T: ops.fp8_static_linear(x, T(xs), T(w_e4m3), T(ws), T(bias), None)),
        "fp8_blockwise_linear": (e4m3, K, lambda x, T: ops.fp8_blockwise_linear(x, T(xs_t), T(w_e4m3), T(ws_b), T(bias))),
        "fp8_sparse_linear": (e4m3, K, lambda x, T: ops.fp8_sparse_linear(x, T(xs), T(w_sp), T(w_meta), T(ws), T(bias))),
        "fp8_weight_linear": (bf16, K, lambda x, T: ops.fp8_weight_linear(x, T(w_e4m3), T(ws), T(bias))),
        "mxfp8_linear": (e4m3, K, lambda x, T: ops.mxfp8_linear(x, T(xs_mx), T(w_e4m3), T(ws_mx), T(bias))),
        "mxfp4_linear": (u8, K // 2, lambda x, T: ops.mxfp4_linear(x, T(xs_mx), T(w_fp4), T(ws_mx), T(bias))),
        "nvfp4_linear": (u8, K // 2,
                         lambda x, T: ops.nvfp4_linear(x, T(xs_nv), T(a_pts), T(w_fp4), T(ws_nv), T(b_pts), T(bias))),
        "nvfp4_weight_linear": (bf16, K,
                                lambda x, T: ops.nvfp4_weight_linear(x, None, T(w_fp4), T(ws_nv), T(b_pts), T(bias))),
        "int4_tilepacked_linear": (bf16, K, lambda x, T: ops.int4_tilepacked_linear(x, T(w4), G, T(sz), T(bias))),
    }


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16)) if a.dtype == torch.bfloat16 else torch.equal(a, b)


OPS = ["int8_dyn_linear", "int8_weight_linear", "int8_mm_i32", "fp8_rowwise_linear", "fp8_static_linear",
       "fp8_blockwise_linear", "fp8_sparse_linear", "fp8_weight_linear", "mxfp8_linear", "mxfp4_linear",
       "nvfp4_linear", "nvfp4_weight_linear", "int4_tilepacked_linear"]


@pytest.mark.parametrize("op", OPS)
def test_activation_views_equal_an_aligned_copy(ops, op):
    dtype, cols, call = _dense_ops(ops)[op]
    same = lambda t: t   # noqa: E731
    g = ex.gen(22)
    # rows at a storage offset that is not on 16 bytes
    x = _codes(dtype, M * cols + 16, g)[4:4 + M * cols].view(M, cols)
    dense = x.clone()
    assert x.data_ptr() % 16 != 0 and dense.data_ptr() % 16 == 0
    if dtype == torch.bfloat16:
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            call(x, same)
        # a column slice of a wider buffer: strided rows from an aligned start
        x = _codes(dtype, M * (cols + 8), g).view(M, cols + 8)[:, 8:8 + cols]
        dense = x.contiguous()
        assert x.data_ptr() % 16 == 0 and x.stride(0) == cols + 8
    y, want = call(x, same), call(dense, same)
    assert y.shape == (M, N) and _same_bits(y, want)


@pytest.mark.parametrize("op", OPS)
def test_meta_output_matches_the_cuda_output(ops, op):
    dtype, cols, call = _dense_ops(ops)[op]
    x = _codes(dtype, M * cols, ex.gen(23)).view(M, cols)
    y = call(x, lambda t: t)
    m = call(x.to("meta"), lambda t: t.to("meta"))
    assert m.device.type == "meta"
    assert (m.shape, m.dtype, m.stride()) == (y.shape, y.dtype, y.stride())
