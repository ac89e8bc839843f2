"""CPU tests of the fp8 grouped GEMM's host side: the Meta shape of torch.ops.ao_b200.fp8_rowwise_grouped_mm, its C-ABI
argument checks (before any CUDA call), and the Float8Tensor pieces torch._grouped_mm goes through."""
import ctypes
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_meta_shape():
    import ao_b200  # noqa: F401

    xq = torch.empty(37, 256, dtype=torch.float8_e4m3fn, device="meta")
    wq = torch.empty(8, 144, 256, dtype=torch.float8_e4m3fn, device="meta")
    y = torch.ops.ao_b200.fp8_rowwise_grouped_mm(xq, torch.empty(37, device="meta"), wq,
                                                 torch.empty(8, 144, device="meta"),
                                                 torch.empty(8, dtype=torch.int32, device="meta"))
    assert y.shape == (37, 144) and y.dtype == torch.bfloat16 and y.device.type == "meta"


def test_c_abi_argument_validation_without_gpu():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_fp8_rowwise_grouped_mm
    f.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    one = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first

    def call(M=4, K=256, E=8, N=256, ptrs=(one,) * 6, ws=one):
        xq, xs, wq, wsc, offs, y = ptrs
        return f(xq, xs, M, K, wq, wsc, E, N, offs, y, ws, 1 << 20, None)

    assert call(K=100) == -1 and b"K=100" in lib.ao_b200_last_error()
    assert call(N=100) == -1 and b"N=100" in lib.ao_b200_last_error()
    assert call(E=0) == -1 and b"E=0" in lib.ao_b200_last_error()
    assert call(E=1025) == -1 and b"E=1025" in lib.ao_b200_last_error()
    assert call(E=1024, N=2**21) == -1 and b"int32" in lib.ao_b200_last_error()
    assert call(M=-1) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    for i in range(6):
        ptrs = [one] * 6
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in lib.ao_b200_last_error(), i
    assert call(ws=None) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert call(ptrs=(ctypes.c_void_p(24),) + (one,) * 5) == -1 and b"16-byte aligned" in lib.ao_b200_last_error()
    # no tokens: nothing to do, nothing dereferenced
    assert call(M=0, ptrs=(None,) * 6, ws=None) == 0


def test_float8_transpose_and_3d_quantize():
    """quantize_ with a filter_fn on a module holding a 3-D expert weight gives qdata [E, N, K] and scale [E, N, 1];
    transpose(-2, -1) is a view with qdata, scale and block_size swapped, the form torch._grouped_mm receives."""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8Tensor, PerRow, quantize_

    class Experts(torch.nn.Module):
        def __init__(self, E, K, N):
            super().__init__()
            self.weight = torch.nn.Parameter(torch.randn(E, N, K, dtype=torch.bfloat16))

    m = Experts(4, 128, 256)
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()),
              filter_fn=lambda mod, fqn: isinstance(mod, Experts))
    w = m.weight
    assert isinstance(w, Float8Tensor) and w.qdata.shape == (4, 256, 128) and w.scale.shape == (4, 256, 1)
    assert w.block_size == [1, 1, 128]
    t = w.transpose(-2, -1)
    assert isinstance(t, Float8Tensor) and t.shape == (4, 128, 256) and t.qdata.shape == (4, 128, 256)
    assert t.qdata.stride(-2) < t.qdata.stride(-1) and t.scale.shape == (4, 1, 256) and t.block_size == [1, 128, 1]
    assert torch.equal(t.qdata.transpose(-2, -1).view(torch.uint8), w.qdata.view(torch.uint8))


def test_grouped_mm_handler_rejects_unsupported_forms():
    from ao_b200.quantization import Float8Tensor, PerRow, PerTensor
    from ao_b200.quantization.quantize_.workflows.float8.float8_tensor import QuantizeTensorToFloat8Kwargs

    w = torch.randn(4, 256, 128, dtype=torch.bfloat16)
    x = torch.randn(16, 128, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    wo = Float8Tensor.from_hp(w, granularity=PerRow())
    with pytest.raises(NotImplementedError):   # weight-only: outside this engine's scope
        torch._grouped_mm(x, wo.transpose(-2, -1), offs=offs)
    pt = Float8Tensor.from_hp(w, granularity=PerRow(), act_quant_kwargs=QuantizeTensorToFloat8Kwargs(granularity=PerTensor()))
    with pytest.raises(NotImplementedError):
        torch._grouped_mm(x, pt.transpose(-2, -1), offs=offs)
    rw = Float8Tensor.from_hp(w, granularity=PerRow(), act_quant_kwargs=QuantizeTensorToFloat8Kwargs(granularity=PerRow()))
    with pytest.raises(AssertionError):        # mat_b must be the transposed view of the stored weight
        torch._grouped_mm(x, rw, offs=offs)
