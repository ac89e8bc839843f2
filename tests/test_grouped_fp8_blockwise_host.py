"""CPU tests of the blockwise fp8 expert GEMM (torch._grouped_mm on 3-D Float8Tensor weights with [1, 128, 128]
blocks and PerBlock([1, 128]) activations, torch.ops.ao_b200.fp8_blockwise_grouped_mm):

* the Meta shape, the op schema and the C-ABI argument checks (before any CUDA call);
* the package's 3-D weight quantizer, the select and transpose views and the per-expert activation codes against the
  reference's fixture (golden/fp8_blockwise_3d.npz), bit for bit; quantizing all routed rows at once gives the
  per-expert codes and scales;
* the handler's rejections, and that the other PerBlock pairs and PerTensor keep raising;
* quantize_ of 3-D parameters through FqnToConfig, torch.save and safetensors round trips;
* ts_gemm_kernel<Grouped<BlockwiseF8GroupedFmt>, N> exists for every token tile, has no stack or local memory and fits one
  CTA per SM beside the schedule tables.
"""
import ctypes
import io
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_decode_residency import LIB, RESERVED_PER_CTA, SMEM_PER_SM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fp8_blockwise_3d.npz")
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def bf16(bits):
    return torch.from_numpy(bits.view(np.int16).copy()).view(torch.bfloat16)


def blockwise_config(**kw):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock

    return Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])], **kw)


def _w3(E=4, N=256, K=384, dtype=torch.bfloat16, seed=0, **act):
    """A 3-D blockwise expert weight [E, N, K] as the config makes it (128x128 blocks, PerBlock([1, 128]) activations)"""
    from ao_b200.quantization import Float8Tensor, PerBlock, QuantizeTensorToFloat8Kwargs

    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(E, N, K, generator=g) * 0.05).to(dtype)
    kw = QuantizeTensorToFloat8Kwargs(granularity=PerBlock([1, 128]), **act)
    return Float8Tensor.from_hp(w, granularity=PerBlock([128, 128]), act_quant_kwargs=kw)


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
def test_meta_shape_and_schema():
    import ao_b200  # noqa: F401

    xq = torch.empty(37, 384, dtype=E4M3, device="meta")
    xs = torch.empty(3, 40, device="meta")
    wq = torch.empty(8, 256, 384, dtype=E4M3, device="meta")
    y = torch.ops.ao_b200.fp8_blockwise_grouped_mm(xq, xs, wq, torch.empty(8, 2, 3, device="meta"),
                                                   torch.empty(8, dtype=torch.int32, device="meta"))
    assert y.shape == (37, 256) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(torch.ops.ao_b200.fp8_blockwise_grouped_mm.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale, Tensor offs) -> Tensor")


def test_c_abi_argument_validation_without_gpu():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_fp8_blockwise_grouped_mm
    f.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15   # host addresses stand in for device ones: never dereferenced
    one = ctypes.c_void_p(a)

    def call(M=4, K=256, E=8, N=256, ptrs=(one,) * 7):
        xq, xs, wq, ws, offs, y, work = ptrs
        return f(xq, xs, M, K, wq, ws, E, N, offs, y, work, 1 << 20, None)

    err = lib.ao_b200_last_error
    assert call(K=200) == -1 and b"K=200 must be a multiple of 128" in err()
    assert call(N=200) == -1 and b"N=200 must be a multiple of 128" in err()
    assert call(N=136) == -1 and b"N=136" in err()
    assert call(E=0) == -1 and b"E=0" in err()
    assert call(E=1025) == -1 and b"E=1025" in err()
    assert call(E=1024, N=2**21) == -1 and b"int32" in err()
    assert call(M=-1) == -1 and b"bad sizes" in err()
    assert call(K=0) == -1 and b"bad sizes" in err()
    for i in range(7):
        ptrs = [one] * 7
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in err(), i
    assert call(ptrs=(ctypes.c_void_p(a + 8),) + (one,) * 6) == -1 and b"x must be 16-byte aligned" in err()
    assert call(ptrs=(one, ctypes.c_void_p(a + 4)) + (one,) * 5) == -1 and b"x_scale must be 16-byte aligned" in err()
    # no tokens: nothing to do, nothing dereferenced, no CUDA call (this process has no device)
    assert call(M=0, ptrs=(None,) * 7) == 0


# ------------------------------------------------------------------------------------------------ the fixture
def test_3d_weight_matches_the_reference(golden):
    from ao_b200.quantization import Float8Tensor, PerBlock

    w = Float8Tensor.from_hp(bf16(golden["w"]), granularity=PerBlock([128, 128]))
    assert list(w.block_size) == golden["block_size"].tolist() == [1, 128, 128]
    assert w.scale.shape == golden["w_scale"].shape == (3, 2, 3) and w.scale.dtype == torch.float32
    assert np.array_equal(w.qdata.view(torch.uint8).numpy(), golden["w_q"])
    assert np.array_equal(w.scale.numpy().view(np.uint32), golden["w_scale"].view(np.uint32))


def test_fixture_holds_the_edge_blocks(golden):
    s, tiny = golden["w_scale"], np.finfo(np.float32).tiny
    assert 0 < s[0, 0, 1] < tiny                                                # a subnormal weight scale
    assert s[1, 1, 0] == 0 and (golden["w_q"][1, 128:, :128] & 0x7F == 0x7F).all()   # all zero: NaN codes
    xs = golden["x_scale"]
    assert xs[0, 0] == 0 and ((xs > 0) & (xs < tiny)).any()
    offs = golden["offs"].tolist()
    assert 0 in np.diff([0] + offs) and golden["x"].shape[0] > offs[-1]        # an empty expert, rows past offs[-1]


def test_select_and_transpose_views_match_the_reference(golden):
    from ao_b200.quantization import Float8Tensor, PerBlock

    views = json.loads(str(golden["views"]))
    w = Float8Tensor.from_hp(bf16(golden["w"]), granularity=PerBlock([128, 128]))
    for e, v in enumerate(views["select"]):
        we = w[e]
        assert type(we) is Float8Tensor
        assert [list(we.shape), list(we.qdata.shape), list(we.scale.shape), list(we.block_size)] == \
            [v["shape"], v["qdata"], v["scale"], v["block_size"]], e
        assert np.array_equal(we.qdata.view(torch.uint8).numpy(), golden["w_q"][e])
        assert np.array_equal(we.scale.numpy().view(np.uint32), golden["w_scale"][e].view(np.uint32))
    t, v = w.transpose(-2, -1), views["transpose"]
    assert [list(t.shape), list(t.qdata.shape), list(t.scale.shape), list(t.block_size)] == \
        [v["shape"], v["qdata"], v["scale"], v["block_size"]]
    assert t.qdata.stride(-2) < t.qdata.stride(-1)
    back = t.transpose(-2, -1)
    assert back.qdata.is_contiguous() and back.scale.is_contiguous()   # what the handler passes to the op


def test_one_quantization_over_all_rows_equals_the_per_expert_recipe(golden):
    """The handler quantizes every routed row at once; the recipe quantizes each expert's rows on its own.  1x128
    blocks never span two rows, so the codes and scales of the rows up to offs[-1] are the reference's."""
    from ao_b200.quantization import Float8Tensor, PerBlock

    x = bf16(golden["x"])
    end = int(golden["offs"][-1])
    t = Float8Tensor.from_hp(x, granularity=PerBlock([1, 128]))
    assert np.array_equal(t.qdata.view(torch.uint8).numpy()[:end], golden["x_q"])
    assert np.array_equal(t.scale.numpy()[:end].view(np.uint32), golden["x_scale"].view(np.uint32))


def test_the_reference_grouped_mm_raises_for_this_pair(golden):
    r = json.loads(str(golden["grouped_mm"]))
    assert r["raised"] == "NotImplementedError" and "PerRow" in r["message"]


# ------------------------------------------------------------------------------------------------ the handler
def test_grouped_mm_handler_rejects_unsupported_forms():
    w = _w3()
    x = torch.randn(16, 384, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    for fn in (torch._grouped_mm, F.grouped_mm):
        with pytest.raises(AssertionError, match="transposed"):
            fn(x, w, offs=offs)
        with pytest.raises(NotImplementedError, match="bias"):
            torch._grouped_mm(x, w.transpose(-2, -1), offs=offs, bias=torch.zeros(256, dtype=torch.bfloat16))
        with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
            fn(x, w.transpose(-2, -1), offs=offs, out_dtype=torch.float32)
        with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
            fn(x.half(), w.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="2-D mat_a x 3-D mat_b"):
            fn(x.reshape(4, 4, 384), w.transpose(-2, -1), offs=offs)
        for dt in (torch.float16, torch.float32):
            with pytest.raises(NotImplementedError, match=f"quantized from {dt}"):
                fn(x, _w3(dtype=dt).transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="e4m3 weights and activations only"):
            fn(x, _w3(float8_dtype=torch.float8_e5m2).transpose(-2, -1), offs=offs)
        for bound in ({"hp_value_lb": 1e-4}, {"hp_value_ub": 100.0}):
            with pytest.raises(NotImplementedError, match="activation_value_lb / activation_value_ub"):
                fn(x, _w3(**bound).transpose(-2, -1), offs=offs)
        # a served form on CPU tensors reaches the CUDA-only ops and fails in the dispatcher
        with pytest.raises(NotImplementedError, match="fp8_quantize_1x128"):
            fn(x, w.transpose(-2, -1), offs=offs)


def test_e5m2_weights_are_rejected():
    from ao_b200.quantization import Float8Tensor, PerBlock, QuantizeTensorToFloat8Kwargs

    w = Float8Tensor.from_hp(torch.randn(2, 128, 256).to(torch.bfloat16), torch.float8_e5m2, PerBlock([128, 128]),
                             act_quant_kwargs=QuantizeTensorToFloat8Kwargs(granularity=PerBlock([1, 128])))
    x = torch.randn(4, 256, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="e4m3 weights and activations only"):
        torch._grouped_mm(x, w.transpose(-2, -1), offs=torch.tensor([2, 4], dtype=torch.int32))


@pytest.mark.parametrize("pair", ["per_tensor", "a1x64_w128x128", "a1x128_w64x64", "a128x128_w128x128"])
def test_other_granularities_keep_raising(pair):
    """Only PerBlock([1, 128]) activations on [1, 128, 128] weight blocks reach the blockwise op; PerTensor and the
    other PerBlock pairs raise as before."""
    from ao_b200.quantization import Float8Tensor, PerBlock, PerTensor, QuantizeTensorToFloat8Kwargs

    a, wb = {"per_tensor": (PerTensor(), PerTensor()), "a1x64_w128x128": (PerBlock([1, 64]), PerBlock([128, 128])),
             "a1x128_w64x64": (PerBlock([1, 128]), PerBlock([64, 64])),
             "a128x128_w128x128": (PerBlock([128, 128]), PerBlock([128, 128]))}[pair]
    w = Float8Tensor.from_hp(torch.randn(2, 128, 256).to(torch.bfloat16), E4M3, wb,
                             act_quant_kwargs=QuantizeTensorToFloat8Kwargs(granularity=a))
    x = torch.randn(4, 256, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="only supports PerRow granularity"):
        torch._grouped_mm(x, w.transpose(-2, -1), offs=torch.tensor([2, 4], dtype=torch.int32))


# ------------------------------------------------------------------------------------------------ config, serialization
class Experts(torch.nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.gate_up_proj = torch.nn.Parameter(torch.randn(E, 2 * I, H, dtype=torch.bfloat16))
        self.down_proj = torch.nn.Parameter(torch.randn(E, H, I, dtype=torch.bfloat16))


def test_quantize_3d_parameters_through_fqn_to_config():
    from ao_b200.quantization import Float8Tensor, FqnToConfig, PerBlock, quantize_

    m = Experts(3, 256, 128)
    cfg = blockwise_config()
    quantize_(m, FqnToConfig({"gate_up_proj": cfg, "down_proj": cfg}), filter_fn=None)
    for p, shape in ((m.gate_up_proj, (3, 256, 256)), (m.down_proj, (3, 256, 128))):
        E, N, K = shape
        assert isinstance(p, Float8Tensor) and p.shape == shape and list(p.block_size) == [1, 128, 128]
        assert p.scale.shape == (E, N // 128, K // 128) and p.act_quant_kwargs.granularity == PerBlock([1, 128])


def test_3d_serialization_round_trips():
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Float8Tensor

    w = _w3(3, 256, 384, seed=3)
    buf = io.BytesIO()
    torch.save({"experts.w": w}, buf)
    buf.seek(0)
    r = torch.load(buf, weights_only=True)["experts.w"]
    flat, meta = flatten_tensor_state_dict({"experts.w": w})
    assert json.loads(meta["experts.w"])["_data"]["block_size"] == [1, 128, 128]
    s, left = unflatten_tensor_state_dict(flat, meta)
    assert not left
    for got in (r, s["experts.w"]):
        assert type(got) is Float8Tensor and got.shape == (3, 256, 384) and got.dtype == torch.bfloat16
        assert list(got.block_size) == [1, 128, 128] and got.act_quant_kwargs == w.act_quant_kwargs
        assert torch.equal(got.qdata.view(torch.uint8), w.qdata.view(torch.uint8)) and torch.equal(got.scale, w.scale)


# ------------------------------------------------------------------------------------------------ kernels
TABLE_BYTES = 4 * (1024 + 1025)   # s_end[MAX_EXPERTS] + s_mbp[MAX_EXPERTS + 1]


@pytest.mark.parametrize("n_mma", [16, 32, 64])
def test_ring_and_tables_fit_one_cta_per_sm(n_mma):
    """Cfg<Grouped<BlockwiseF8GroupedFmt>, N>: a stage is the 16 KiB weight tile, the 1 KiB aux slot (the 272-byte token
    scale box) and N x 128 activation bytes; a 200 KB ring of at most 12 stages, the tables beside it."""
    stage = 16384 + 1024 + n_mma * 128
    stages = min(12, 200 * 1024 // stage)
    smem = stages * stage + 3 * stages * 8 + 1024
    assert stages == {16: 10, 32: 9, 64: 8}[n_mma]
    assert smem + TABLE_BYTES <= 227 * 1024 and smem + TABLE_BYTES + RESERVED_PER_CTA <= SMEM_PER_SM


def test_grouped_blockwise_kernels_have_no_stack_or_local_memory():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found = {}
    fn = None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_4lowp21BlockwiseF8GroupedFmtE\S*?Li(\d+)E\S*):", line)
        if m:
            fn = int(m.group(2))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", line)
        if m and fn:
            found[fn] = tuple(int(g) for g in m.groups())
        fn = None
    assert sorted(found) == [16, 32, 64], found   # MAX_N_MMA 64, as the rowwise e4m3 format
    for n_mma, (reg, stack, local) in found.items():
        assert stack == 0 and local == 0, f"ts_gemm_kernel<Grouped<BlockwiseF8GroupedFmt>, {n_mma}>: stack {stack}, local {local}"
        assert reg <= 168, (n_mma, reg)   # one CTA of 384 threads per SM: 65536 / 384, rounded down to 8
