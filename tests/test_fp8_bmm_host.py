"""CPU tests of torch.bmm on rowwise e4m3 Float8Tensor weights (the Float8Tensor bmm handler and
torch.ops.ao_b200.fp8_rowwise_bmm):

* the quantization of a [B, K, N] weight with granularity [PerRow(), PerRow(1)] (quantize_ with a filter_fn and
  FqnToConfig on a parameter) against the reference's codes and scales in tests/golden/fp8_bmm.npz;
* the handler's layout detection from qdata's strides, its rejections and its M == 0 result;
* the op's Meta shape and schema, and the C-ABI argument checks (before any CUDA call);
* torch.save and safetensors round trips of a [B, K, N] weight;
* ts_gemm_kernel<Grouped<F8NMajorFmt>, N> for every token tile: no stack, a register count that fits one CTA of 384
  threads per SM, and a ring plus transpose buffer plus schedule tables within the shared memory of one CTA.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
LIB = os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so")
E4M3 = torch.float8_e4m3fn


def _config(**kw):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow

    return Float8DynamicActivationFloat8WeightConfig(granularity=[PerRow(), PerRow(1)], **kw)


class Holder(torch.nn.Module):
    def __init__(self, w):
        super().__init__()
        self.weight = torch.nn.Parameter(w, requires_grad=False)

    def forward(self, x):
        return torch.bmm(x, self.weight)


class Experts(torch.nn.Module):
    """llama-models' MoE experts: w1 / w3 [E, D, F] and w2 [E, F, D], each used as torch.bmm(x, w)."""

    def __init__(self, E, D, F_):
        super().__init__()
        self.w1 = torch.nn.Parameter(torch.randn(E, D, F_, dtype=torch.bfloat16), requires_grad=False)
        self.w2 = torch.nn.Parameter(torch.randn(E, F_, D, dtype=torch.bfloat16), requires_grad=False)
        self.w3 = torch.nn.Parameter(torch.randn(E, D, F_, dtype=torch.bfloat16), requires_grad=False)


# ------------------------------------------------------------------------------------------------ the fixture
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "fp8_bmm.npz"))


def _cases(golden):
    for i, shape in enumerate(json.loads(str(golden["shapes"]))):
        w = torch.from_numpy(golden[f"s{i}_w"].view(np.int16)).view(torch.bfloat16)
        assert tuple(w.shape) == tuple(shape)
        yield i, w


def _check(t, golden, i):
    from ao_b200.quantization import Float8Tensor

    B, K, N = t.shape
    assert type(t) is Float8Tensor and t.act_quant_kwargs is not None
    assert list(t.block_size) == golden[f"s{i}_bs"].tolist() == [1, K, 1]
    assert tuple(t.scale.shape) == (B, 1, N) and t.scale.dtype == torch.float32
    assert np.array_equal(t.qdata.view(torch.uint8).numpy(), golden[f"s{i}_wq"]), i
    assert np.array_equal(t.scale.numpy().view(np.uint32), golden[f"s{i}_ws"].view(np.uint32)), i


def test_quantize_with_filter_fn_matches_the_reference(golden):
    from ao_b200.quantization import quantize_

    for i, w in _cases(golden):
        m = Holder(w.clone())
        quantize_(m, _config(), filter_fn=lambda *_: True)
        _check(m.weight, golden, i)


def test_fqn_to_config_on_a_parameter_matches_the_reference(golden):
    from ao_b200.quantization import FqnToConfig, quantize_

    for i, w in _cases(golden):
        m = torch.nn.Sequential()
        m.add_module("experts", Holder(w.clone()))
        quantize_(m, FqnToConfig({"experts.weight": _config()}), filter_fn=None)
        _check(m.experts.weight, golden, i)


def test_llama_experts_are_quantized_per_output_feature():
    from ao_b200.quantization import FqnToConfig, quantize_

    torch.manual_seed(0)
    m = Experts(2, 64, 96)
    quantize_(m, FqnToConfig({"w1": _config(), "w2": _config(), "w3": _config()}), filter_fn=None)
    assert tuple(m.w1.scale.shape) == (2, 1, 96) and tuple(m.w2.scale.shape) == (2, 1, 64)
    assert m.w1.qdata.is_contiguous() and m.w1.qdata.stride(-1) == 1


# ------------------------------------------------------------------------------------------------ the handler
def _weight(B, K, N, layout, seed=0, **kw):
    """A Float8Tensor of shape [B, K, N]: "kn" stored [B, K, N] (PerRow(1)), "nk" the transposed view of a stored
    [B, N, K] (PerRow())."""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow, quantize_

    g = torch.Generator().manual_seed(seed)
    if layout == "kn":
        m = Holder(torch.randn(B, K, N, generator=g).to(torch.bfloat16))
        quantize_(m, _config(**kw), filter_fn=lambda *_: True)
        return m.weight
    m = Holder(torch.randn(B, N, K, generator=g).to(torch.bfloat16))
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=PerRow(), **kw), filter_fn=lambda *_: True)
    return m.weight.transpose(-2, -1)


@pytest.fixture
def captured(monkeypatch):
    """The arguments the handler passes to the op, which returns the Meta shape (no GPU here)."""
    calls = []

    def fake(xq, x_scale, wq, w_scale):
        calls.append((xq, x_scale, wq, w_scale))
        return torch.zeros(xq.shape[0], xq.shape[1], wq.shape[2], dtype=torch.bfloat16)

    monkeypatch.setattr(torch.ops.ao_b200, "fp8_rowwise_bmm", fake)
    return calls


@pytest.mark.parametrize("layout", ["kn", "nk"])
def test_handler_reads_the_layout_from_the_strides(captured, layout):
    B, M, K, N = 3, 5, 208, 144
    w = _weight(B, K, N, layout)
    x = torch.randn(B, M, K).to(torch.bfloat16)
    for y in (torch.bmm(x, w), torch.ops.aten.bmm.default(x, w)):
        assert y.shape == (B, M, N) and y.dtype == torch.bfloat16
    xq, xs, wq, ws = captured[-1]
    assert xq.shape == (B, M, K) and xq.dtype == E4M3 and xs.shape == (B * M,) and xs.dtype == torch.float32
    assert wq.shape == (B, K, N) and ws.shape == (B, N) and ws.is_contiguous()
    if layout == "kn":
        assert wq.is_contiguous()
    else:
        assert wq.stride() == (N * K, 1, K) and wq.transpose(-2, -1).is_contiguous()
    # the weight's own codes, not a copy in another layout
    assert torch.equal(wq.view(torch.uint8), w.qdata.view(torch.uint8))
    assert torch.equal(ws, w.scale.reshape(B, N))
    # the activations: the rowwise quantizer over all B*M rows
    from ao_b200.quantization import Float8Tensor, PerRow
    ref = Float8Tensor.from_hp(x.reshape(-1, K), granularity=PerRow())
    assert torch.equal(xq.reshape(-1, K).view(torch.uint8), ref.qdata.view(torch.uint8))
    assert torch.equal(xs, ref.scale.reshape(-1))


def test_handler_rejects_other_strides(captured):
    from ao_b200.quantization import Float8Tensor

    w = _weight(2, 64, 64, "kn")
    # every other output feature: stride(-1) == 2 and stride(-2) == 64, neither layout
    odd = Float8Tensor(w.qdata[:, :, ::2], w.scale[:, :, ::2], [1, 64, 1], w.mm_config, w.act_quant_kwargs,
                       w.kernel_preference, w.dtype)
    assert odd.qdata.stride() == (64 * 64, 64, 2)
    with pytest.raises(NotImplementedError, match="strides"):
        torch.bmm(torch.randn(2, 3, 64).to(torch.bfloat16), odd)
    assert not captured


def test_handler_rejections(captured):
    from ao_b200.quantization import Float8WeightOnlyConfig, PerRow, quantize_
    from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference

    x = torch.randn(2, 3, 64).to(torch.bfloat16)
    m = Holder(torch.randn(2, 32, 64).to(torch.bfloat16))
    quantize_(m, Float8WeightOnlyConfig(), filter_fn=lambda *_: True)
    with pytest.raises(NotImplementedError, match="bmm only support float8 dynamic activation \\+ float8 weight"):
        torch.bmm(x, m.weight.transpose(-2, -1))
    with pytest.raises(AssertionError, match="bmm is not supported for TORCH"):
        torch.bmm(x, _weight(2, 64, 32, "kn", kernel_preference=KernelPreference.TORCH))
    w = _weight(2, 64, 32, "kn")
    with pytest.raises(NotImplementedError, match="bf16 x only"):
        torch.bmm(x.float(), w)
    with pytest.raises(NotImplementedError, match="bf16 x only"):
        torch.bmm(x.half(), w)
    with pytest.raises(ValueError, match="does not match"):
        torch.bmm(torch.randn(3, 3, 64).to(torch.bfloat16), w)
    with pytest.raises(ValueError, match="does not match"):
        torch.bmm(torch.randn(2, 3, 48).to(torch.bfloat16), w)
    assert not captured


def test_handler_rejects_blockwise_and_per_tensor_weights(captured):
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, PerBlock, PerRow, PerTensor,
                                      quantize_)

    x = torch.randn(2, 3, 256).to(torch.bfloat16)
    m = Holder(torch.randn(2, 128, 256).to(torch.bfloat16))
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])]),
              filter_fn=lambda *_: True)
    with pytest.raises(NotImplementedError, match="128x128 blockwise"):
        torch.bmm(x, m.weight.transpose(-2, -1))
    m = Holder(torch.randn(2, 128, 256).to(torch.bfloat16))
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=PerTensor()), filter_fn=lambda *_: True)
    with pytest.raises(AssertionError, match="per row weight quantization"):
        torch.bmm(x, m.weight.transpose(-2, -1))
    # per-row weights, per-tensor activations
    from ao_b200.quantization import Float8Tensor
    from ao_b200.quantization.quantize_.workflows.float8.float8_tensor import QuantizeTensorToFloat8Kwargs

    w = _weight(2, 256, 32, "kn")
    w2 = Float8Tensor(w.qdata, w.scale, w.block_size, w.mm_config, QuantizeTensorToFloat8Kwargs(granularity=PerTensor()),
                      w.kernel_preference, w.dtype)
    with pytest.raises(AssertionError, match="per row activation quantization"):
        torch.bmm(x, w2)
    assert not captured


def test_handler_returns_an_empty_result_without_rows(captured):
    w = _weight(3, 64, 32, "kn")
    y = torch.bmm(torch.empty(3, 0, 64, dtype=torch.bfloat16), w)
    assert y.shape == (3, 0, 32) and y.dtype == torch.bfloat16
    assert not captured


# ------------------------------------------------------------------------------------------------ op and C ABI
def test_meta_shape_and_schema():
    import ao_b200  # noqa: F401

    xq = torch.empty(4, 7, 208, dtype=E4M3, device="meta")
    for wq in (torch.empty(4, 208, 144, dtype=E4M3, device="meta"),
               torch.empty(4, 144, 208, dtype=E4M3, device="meta").transpose(-2, -1)):
        y = torch.ops.ao_b200.fp8_rowwise_bmm(xq, torch.empty(28, device="meta"), wq, torch.empty(4, 144, device="meta"))
        assert y.shape == (4, 7, 144) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    schema = str(torch.ops.ao_b200.fp8_rowwise_bmm.default._schema)
    assert schema == "ao_b200::fp8_rowwise_bmm(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale) -> Tensor"


def test_c_abi_argument_validation_without_gpu():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_fp8_rowwise_bmm
    f.restype = i32
    f.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i32, vp, vp, sz, vp]
    one = ctypes.c_void_p(4096)   # never dereferenced: every call below fails its checks or returns before a launch
    err = lib.ao_b200_last_error

    def call(B=4, M=3, K=256, N=128, w_kn=1, ptrs=(one,) * 6, ws_bytes=1 << 20):
        xq, xs, wq, ws, y, work = ptrs
        return f(xq, xs, B, M, K, wq, ws, N, w_kn, y, work, ws_bytes, None)

    assert call(B=0) == -1 and b"B=0" in err()
    assert call(B=1025) == -1 and b"B=1025" in err()
    assert call(M=-1) == -1 and b"bad sizes" in err()
    assert call(K=0) == -1 and b"bad sizes" in err()
    assert call(N=0) == -1 and b"bad sizes" in err()
    assert call(B=1024, M=2**21) == -1 and b"int32" in err()
    assert call(K=200) == -1 and b"K=200" in err()
    assert call(N=72) == -1 and b"N=72" in err()
    assert call(w_kn=2) == -1 and b"w_kn=2" in err()
    assert call(M=0, ptrs=(None,) * 6) == 0   # no rows: nothing is read
    for i in range(6):
        ptrs = [one] * 6
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in err(), i
    assert call(ws_bytes=1024) == -1 and b"workspace too small" in err()


# ------------------------------------------------------------------------------------------------ serialization
def test_torch_save_and_safetensors_round_trips():
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Float8Tensor

    w = _weight(3, 64, 48, "kn", seed=4)
    buf = io.BytesIO()
    torch.save({"experts.w1": w}, buf)
    buf.seek(0)
    r = torch.load(buf, weights_only=True)["experts.w1"]
    flat, meta = flatten_tensor_state_dict({"experts.w1": w})
    s, left = unflatten_tensor_state_dict(flat, meta)
    assert not left
    for got in (r, s["experts.w1"]):
        assert type(got) is Float8Tensor and got.shape == (3, 64, 48) and got.qdata.stride() == (64 * 48, 48, 1)
        assert list(got.block_size) == [1, 64, 1] and got.act_quant_kwargs is not None
        assert torch.equal(got.qdata.view(torch.uint8), w.qdata.view(torch.uint8)) and torch.equal(got.scale, w.scale)


# ------------------------------------------------------------------------------------------------ kernel budget
def _usage():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_4lowp11F8NMajorFmtE\S*?Li(\d+)E\S*):", line)
        if m:
            fn = int(m.group(2))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
        if m and fn:
            found[fn] = tuple(int(v) for v in m.groups())
        fn = None
    return found


def test_n_major_kernels_have_no_stack_and_fit_one_cta_per_sm():
    found = _usage()
    assert sorted(found) == [16, 32, 64], found   # e4m3 keeps a second accumulator: token tiles up to 64
    for n_mma, (reg, stack, static_smem) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<F8NMajorFmt>, {n_mma}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (n_mma, reg)   # one CTA of 384 threads per SM: 65536 / 384, rounded down to 8
        # Cfg: a 200 KiB ring less the 16 KiB transpose buffer, then the buffer, the barriers and the alignment pad
        stage = 128 * 128 + n_mma * 128
        stages = min((200 * 1024 - 16384) // stage, 12)
        dyn = stages * stage + 16384 + 3 * stages * 8 + 1024
        assert stages >= 6, (n_mma, stages)
        assert dyn + static_smem <= 227 * 1024 and dyn + static_smem + 1024 <= 228 * 1024, (n_mma, dyn, static_smem)
