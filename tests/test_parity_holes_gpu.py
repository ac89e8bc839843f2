"""GPU tests for branches of the path that shipped without one in round 1 (VERDICT "untested branches that ship"):

* int8 asymmetric dynamic activations (reference int8_tensor.py:305-359, correction at :322-330): the int32
  accumulator exactly, the final bf16 result bit-for-bit against a torch restatement of those reference lines;
* PerTensor granularity for int8 and fp8 (reference quant_api.py:782-805, float8/inference.py:259-265);
* K that is not a multiple of the kernel's 128-byte chunk (the TMA zero-fills the tail) for int8 / fp8 / mxfp8;
* the C ABI driven directly through ctypes with real device buffers (INTEGRATION.md §2), no torch.ops in between;
* torch.compile(fullgraph=True) on the default (inductor) backend.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sqnr(ref, got):
    ref, got = ref.double(), got.double()
    d = (ref - got).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


@pytest.mark.parametrize("M,N,K,bias", [(1, 256, 512, False), (7, 384, 1024, True), (32, 1024, 4096, True), (33, 128, 256, False)])
def test_int8_asymmetric_activation_branch(M, N, K, bias):
    import ao_b200  # noqa: F401
    from ao_b200.quantization import Int8DynamicActivationInt8WeightConfig, Int8Tensor, MappingType, PerRow, quantize_

    torch.manual_seed(M + N)
    lin = torch.nn.Linear(K, N, bias=bias, device="cuda", dtype=torch.bfloat16)
    quantize_(lin, Int8DynamicActivationInt8WeightConfig(act_mapping_type=MappingType.ASYMMETRIC))
    w = lin.weight
    assert w.act_quant_kwargs.mapping_type == MappingType.ASYMMETRIC
    x = (torch.randn(M, K, device="cuda") + 0.7).to(torch.bfloat16)   # shifted: a non-trivial zero point
    y = lin(x)
    # the activation quantization the handler performs
    xt = Int8Tensor.from_hp(x, PerRow(), mapping_type=MappingType.ASYMMETRIC)
    assert xt.zero_point is not None and bool((xt.zero_point != 0).any())
    # int32 accumulator: exact
    acc = torch.ops.ao_b200.int8_mm_i32(xt.qdata.contiguous(), w.qdata.contiguous())
    acc_ref = xt.qdata.cpu().to(torch.int64) @ w.qdata.cpu().to(torch.int64).t()
    assert torch.equal(acc.cpu().to(torch.int64), acc_ref)
    # reference lines 315-359 restated with torch ops on the exact accumulator
    xs = xt.scale.reshape(-1, 1).float()
    y_dot = (acc_ref.to("cuda").float() * xs).to(torch.bfloat16)
    corr = (xt.zero_point.reshape(-1, 1).float() * xs) * w.qdata.sum(dim=-1).float()
    y_ref = (y_dot - corr.to(torch.bfloat16)) * w.scale.flatten()
    if bias:
        y_ref = y_ref + lin.bias
    y_ref = y_ref.to(torch.bfloat16)
    assert torch.equal(y, y_ref)
    # and it is a sane linear: close to the unquantized one (the reference's own bar is 20 dB)
    wf = w.dequantize().float()
    y_fp = x.float() @ wf.t() + (lin.bias.float() if bias else 0)
    assert _sqnr(y_fp, y.float()) > 25.0


@pytest.mark.parametrize("fmt", ["int8", "fp8"])
@pytest.mark.parametrize("M", [1, 32, 48])
def test_per_tensor_granularity(fmt, M):
    import ao_b200  # noqa: F401
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Int8DynamicActivationInt8WeightConfig,
                                      PerTensor, quantize_)

    torch.manual_seed(M)
    N, K = 512, 1024
    lin = torch.nn.Linear(K, N, bias=True, device="cuda", dtype=torch.bfloat16)
    w_hp, b_hp = lin.weight.detach().clone(), lin.bias.detach().clone()
    cfg = (Int8DynamicActivationInt8WeightConfig(granularity=PerTensor()) if fmt == "int8"
           else Float8DynamicActivationFloat8WeightConfig(granularity=PerTensor()))
    quantize_(lin, cfg)
    w = lin.weight
    assert w.scale.numel() == 1, "PerTensor weight scale must be a single element"
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    y = lin(x)
    # exact-product restatement from the stored codes: per-tensor activation scale, per-tensor weight scale
    if fmt == "int8":
        amax = x.float().abs().max()
        xs = torch.clamp((amax.to(torch.bfloat16) / 127.5).float(), min=torch.finfo(torch.float32).eps)
        xq = torch.clamp(torch.round(x.float() * (1.0 / xs)), -128, 127)
        ref = (xq.double() @ w.qdata.double().t()) * xs.double() * w.scale.double().reshape(()) + b_hp.double()
    else:
        xs = (x.float().abs().max().to(torch.bfloat16) / 448.0).float()
        xq = torch.clamp(x.float() / xs, -448, 448).to(torch.float8_e4m3fn).double()
        ref = (xq @ w.qdata.double().t()) * xs.double() * w.scale.double().reshape(()) + b_hp.double()
    assert _sqnr(ref, y) > 40.0
    assert _sqnr(x.double() @ w_hp.double().t() + b_hp.double(), y) > (30.0 if fmt == "int8" else 24.0)


@pytest.mark.parametrize("fmt", ["int8", "fp8", "mxfp8"])
@pytest.mark.parametrize("K", [32, 160, 1056, 4128])
def test_k_tail_is_zero_filled(fmt, K):
    """K % 128 != 0 (reference requirements: int8 K % 8, fp8 K % 16, mxfp8 K % 32): the last chunk's tail comes from
    TMA's out-of-bounds zero fill on both operands; results equal the exact-product restatement of the stored codes.
    The SQNR bar below cannot see a wrong 32-element tail, so mxfp8 is also checked bit for bit on exactly
    representable operands (the int8 / fp8 tails are in test_exact_gemm_gpu.py)."""
    import ao_b200  # noqa: F401
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Int8DynamicActivationInt8WeightConfig,
                                      PerRow, quantize_)

    torch.manual_seed(K)
    N, M = 256, 9
    lin = torch.nn.Linear(K, N, bias=False, device="cuda", dtype=torch.bfloat16)
    w_hp = lin.weight.detach().clone()
    cfg = {"int8": Int8DynamicActivationInt8WeightConfig(), "fp8": Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()),
           "mxfp8": MXDynamicActivationMXWeightConfig()}[fmt]
    quantize_(lin, cfg)
    assert type(lin.weight).__name__ in ("Int8Tensor", "Float8Tensor", "MXTensor")
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    y = lin(x)
    assert bool(torch.isfinite(y.float()).all())
    ref = x.double() @ w_hp.double().t()
    assert _sqnr(ref, y) > (30.0 if fmt == "int8" else 24.0)   # quantization noise only: a wrong tail would be ~0-10 dB
    # linearity in the tail columns: zeroing them in x must change the output exactly like the dequantized weights say
    x2 = x.clone()
    x2[:, (K // 128) * 128:] = 0
    y2 = lin(x2)
    assert not torch.equal(y, y2), "the K tail did not reach the output"
    if fmt == "mxfp8":
        import exact_operands as ex

        for m in (M, 40):
            case = ex.build("mxfp8", m, N, K, seed=K)
            y = case.run()
            assert torch.equal(case.bits(y), case.bits(case.ref())), f"M={m} K={K}: {ex.first_mismatch(case, y)}"


def test_c_abi_direct_through_ctypes():
    """INTEGRATION.md §2 executed: dlopen libao_b200.so, pass raw device pointers + the stream, compare with the oracle."""
    from oracle import oracle as o

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    lib.ao_int4_pack_tile4d.argtypes = [vp, vp, i32, i32, i32, vp]
    lib.ao_int4_tilepacked_linear.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, i32, vp, ctypes.c_size_t, i32, vp]
    lib.ao_int4_tilepacked_linear_strided.argtypes = [vp, i32, i32, i32, vp, vp, i32, i32, vp, vp, i32, vp, ctypes.c_size_t, i32, vp]
    assert lib.ao_b200_device_ok() == 1
    M, N, K, g = 5, 384, 2048, 32
    gen = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randint(0, 16, (N, K), device="cuda", generator=gen, dtype=torch.int32)
    q_u8 = (q[:, ::2] << 4 | q[:, 1::2]).to(torch.uint8).contiguous()
    s = (torch.rand(N, K // g, device="cuda", generator=gen) * 0.01 + 0.002).to(torch.bfloat16)
    z = ((torch.rand(N, K // g, device="cuda", generator=gen) - 0.5) * 0.02).to(torch.bfloat16)
    sz = torch.stack([s, z], dim=-1).transpose(0, 1).contiguous()
    x_wide = torch.randn(M, K + 64, device="cuda", generator=gen).to(torch.bfloat16)
    x = x_wide[:, :K].contiguous()
    bias = torch.randn(N, device="cuda", generator=gen).to(torch.bfloat16)
    qdata = torch.empty(N // 8, K // 128, 32, 4, device="cuda", dtype=torch.int32)
    y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    y2 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ws_bytes = lib.ao_b200_workspace_bytes(M, N)
    ws = torch.zeros(ws_bytes, device="cuda", dtype=torch.uint8)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        sp = ctypes.c_void_p(st.cuda_stream)
        rc = lib.ao_int4_pack_tile4d(q_u8.data_ptr(), qdata.data_ptr(), N, K, 8, sp)
        assert rc == 0, lib.ao_b200_last_error()
        rc = lib.ao_int4_tilepacked_linear(x.data_ptr(), M, K, qdata.data_ptr(), sz.data_ptr(), g, N, bias.data_ptr(), y.data_ptr(),
                                           N, ws.data_ptr(), ws_bytes, 0, sp)
        assert rc == 0, lib.ao_b200_last_error()
        rc = lib.ao_int4_tilepacked_linear_strided(x_wide.data_ptr(), K + 64, M, K, qdata.data_ptr(), sz.data_ptr(), g, N,
                                                   bias.data_ptr(), y2.data_ptr(), N, ws.data_ptr(), ws_bytes, 0, sp)
        assert rc == 0, lib.ao_b200_last_error()
    st.synchronize()
    assert np.array_equal(qdata.cpu().numpy(), o.int4_pack_tile4d(q.cpu().numpy().astype(np.uint8), 8))
    ref = o.bf16_to_f32(o.int4_linear(o.bf16_bits(x), qdata.cpu().numpy(), o.bf16_bits(sz), g, o.bf16_bits(bias)))
    got = o.bf16_to_f32(o.bf16_bits(y))
    assert o.sqnr_db(ref, got) > 55.0
    assert torch.equal(y, y2)
    assert bool((ws[:4096] == 0).all()), "the kernels must leave the flag area of the workspace zeroed"
    # argument validation comes back as an error code + message, not a crash
    rc = lib.ao_int4_tilepacked_linear(x.data_ptr(), M, K + 1, qdata.data_ptr(), sz.data_ptr(), g, N, None, y.data_ptr(), N,
                                       ws.data_ptr(), ws_bytes, 0, None)
    assert rc == -1 and b"1024" in lib.ao_b200_last_error()


@pytest.mark.timeout(600)
def test_torch_compile_fullgraph_inductor():
    """The extern op must survive torch.compile(fullgraph=True) on the DEFAULT backend (reference:
    test_float8_tensor.py:397 / test_int4_tile_packed_to_4d_tensor.py compile tests): inductor traces through the
    tensor subclass, keeps torch.ops.ao_b200.* as an extern call and the results equal eager."""
    import ao_b200  # noqa: F401
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Int4WeightOnlyConfig, PerRow, quantize_

    torch.manual_seed(0)
    for cfg in (Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d"),
                Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())):
        m = torch.nn.Sequential(torch.nn.Linear(1024, 512, bias=True, device="cuda", dtype=torch.bfloat16), torch.nn.ReLU(),
                                torch.nn.Linear(512, 256, bias=False, device="cuda", dtype=torch.bfloat16))
        quantize_(m, cfg)
        x = torch.randn(8, 1024, device="cuda", dtype=torch.bfloat16)
        y_eager = m(x)
        n0 = torch.ops.ao_b200.launch_count()
        torch._dynamo.reset()
        compiled = torch.compile(m, fullgraph=True)
        y_comp = compiled(x)
        assert torch.ops.ao_b200.launch_count() > n0, "the compiled graph did not run this engine's kernels"
        assert torch.equal(y_eager, y_comp)
