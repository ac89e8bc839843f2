"""NF4 weights (NF4Tensor, NF4WeightOnlyConfig) without a GPU: the package's quantizer and a restatement of the
dequantization and the linear against the reference's fixture, the handler's assertion, skips and errors, tensor
plumbing (detach, clone, copy_, device moves, torch.save), Meta shapes and the op schema, C-ABI rejections, the
fusion leaving NF4 linears alone, and the register and shared-memory budget of the GEMM's format policy."""
import ctypes
import json
import logging
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import streamk_model as sk
from test_decode_residency import SMEM_PER_SM, RESERVED_PER_CTA, resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ---------------------------------------------------------------- the restatement (shared with the GPU tests)
def bf16(t):
    return t.to(torch.bfloat16)


def restated_weight(quantized_data, quantized_scalers, quantization_factor, scaler_mean, nf4, shape, block_size,
                    scaler_block_size):
    """w~ = bf16(fp32(nf4[code]) * fp32(s[b])), s[b] = bf16(fp32(bf16(fp32(qs[b]) / fp32(f[b / sbs]))) + fp32(mean)),
    every operation an IEEE fp32 one on the device of the inputs."""
    qs = quantized_scalers.to(torch.float32)
    f = quantization_factor.float().repeat_interleave(scaler_block_size)
    s = bf16(bf16(qs / f).float() + scaler_mean.float())
    codes = torch.stack([quantized_data >> 4, quantized_data & 15], -1).flatten().long()
    vals = nf4.float()[codes]
    return bf16(vals * s.float().repeat_interleave(block_size)).reshape(shape)


def restated_linear(x, w, bias):
    """F.linear on the dequantized weight (one bf16 rounding of the fp32 sum), then a bf16 add of the bias."""
    y = F.linear(x, w)
    return y if bias is None else y + bias


def u16(a):
    return torch.from_numpy(a.astype(np.int16)).view(torch.bfloat16)


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "nf4.npz"))
    return z, json.loads(str(z["cases"]))


def _case(z, ci):
    b = u16(z[f"c{ci}_b"]) if f"c{ci}_b" in z else None
    return u16(z[f"c{ci}_w"]), b, u16(z[f"c{ci}_x"]), u16(z[f"c{ci}_xe"])


def test_package_quantizer_matches_the_fixture(golden):
    from ao_b200.quantization import NF4Tensor

    z, cases = golden
    for ci, (M, K, N, bs, sbs, has_bias) in enumerate(cases):
        w, _, _, _ = _case(z, ci)
        t = NF4Tensor.from_tensor(w, bs, sbs)
        assert t.shape == (N, K) and t.dtype == torch.bfloat16 and t.n_blocks == N * K // bs
        assert np.array_equal(t.quantized_data.numpy(), z[f"c{ci}_quantized_data"])
        assert np.array_equal(t.quantized_scalers.numpy(), z[f"c{ci}_quantized_scalers"])
        assert torch.equal(t.quantization_factor.view(torch.int16), u16(z[f"c{ci}_quantization_factor"]).view(torch.int16))
        assert torch.equal(t.scaler_mean.reshape(1).view(torch.int16), u16(z[f"c{ci}_scaler_mean"]).view(torch.int16))
        assert torch.equal(t.nf4.view(torch.int16), u16(z[f"c{ci}_nf4"]).view(torch.int16))
        assert torch.equal(t.get_original_weight().view(torch.int16), u16(z[f"c{ci}_orig"]).view(torch.int16))


def test_restatement_reproduces_the_reference(golden):
    z, cases = golden
    for ci, (M, K, N, bs, sbs, has_bias) in enumerate(cases):
        _, b, x, xe = _case(z, ci)
        w = restated_weight(torch.from_numpy(z[f"c{ci}_quantized_data"]), torch.from_numpy(z[f"c{ci}_quantized_scalers"]),
                            u16(z[f"c{ci}_quantization_factor"]), u16(z[f"c{ci}_scaler_mean"])[0], u16(z[f"c{ci}_nf4"]),
                            (N, K), bs, sbs)
        assert torch.equal(w.view(torch.int16), u16(z[f"c{ci}_orig"]).view(torch.int16)), ci
        for inp, key in ((x, "y"), (xe, "ye")):
            y = restated_linear(inp, w, b)
            assert torch.equal(y.view(torch.int16), u16(z[f"c{ci}_{key}"]).view(torch.int16)), (ci, key)


def test_config_and_exports():
    from ao_b200.core.config import AOBaseConfig
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig, nf4_weight_only
    from ao_b200.quantization import NF4Tensor, to_nf4
    from ao_b200.quantization.quantize_.workflows.nf4.nf4_tensor import linear_nf4  # noqa: F401
    from ao_b200.quantization.transform_module import _QUANTIZE_CONFIG_HANDLER

    assert nf4_weight_only is NF4WeightOnlyConfig and issubclass(NF4WeightOnlyConfig, AOBaseConfig)
    assert NF4WeightOnlyConfig.block_size == 64 and NF4WeightOnlyConfig.scaler_block_size == 256
    assert not hasattr(NF4WeightOnlyConfig, "__dataclass_fields__")
    assert NF4WeightOnlyConfig in _QUANTIZE_CONFIG_HANDLER
    t = to_nf4(torch.randn(128, 128, dtype=torch.bfloat16))
    assert isinstance(t, NF4Tensor) and t.block_size == 64 and t.scaler_block_size == 256
    names, ctx = t.__tensor_flatten__()
    assert names == ["quantized_data", "scaler_mean", "quantization_factor", "quantized_scalers", "nf4"]
    u = NF4Tensor.__tensor_unflatten__({n: getattr(t, n) for n in names}, ctx, t.shape, t.stride())
    assert torch.equal(u.get_original_weight(), t.get_original_weight())


def test_handler_assertion_skips_and_quantized_layers(caplog):
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import NF4Tensor, quantize_

    with pytest.raises(AssertionError):   # N*K % (64 * 256) != 0: the reference asserts as well
        quantize_(nn.Sequential(nn.Linear(128, 64)).to(torch.bfloat16), NF4WeightOnlyConfig())
    small_blocks = NF4WeightOnlyConfig()
    small_blocks.block_size = 8
    skipped = [
        (nn.Linear(256, 256).half(), NF4WeightOnlyConfig(), "dtype"),          # not bf16
        (nn.Linear(96, 512).to(torch.bfloat16), NF4WeightOnlyConfig(), "multiple of block_size"),
        (nn.Linear(64, 32).to(torch.bfloat16), small_blocks, "multiple of 16"),
    ]
    sixteen = NF4WeightOnlyConfig()
    sixteen.block_size = 16
    skipped.append((nn.Linear(16, 256).to(torch.bfloat16), sixteen, "multiple of 32"))
    for lin, cfg, why in skipped:
        m = nn.Sequential(lin)
        with caplog.at_level(logging.INFO):
            caplog.clear()
            quantize_(m, cfg)
        assert not isinstance(m[0].weight, NF4Tensor), why
        assert any("Skipping nf4" in r.message and why in r.message for r in caplog.records), (why, caplog.text)
    m = nn.Sequential(nn.Linear(256, 192, bias=True)).to(torch.bfloat16)
    w = m[0].weight.detach().clone()
    quantize_(m, NF4WeightOnlyConfig())
    assert isinstance(m[0].weight, NF4Tensor) and isinstance(m[0].weight, nn.Parameter)
    assert not m[0].weight.requires_grad
    assert torch.equal(m[0].weight.get_original_weight(), NF4Tensor.from_tensor(w, 64, 256).get_original_weight())


def test_linear_raises_where_the_kernel_does_not_serve():
    from ao_b200.quantization import to_nf4
    from ao_b200.quantization.quantize_.workflows.nf4.nf4_tensor import linear_nf4

    w16 = to_nf4(torch.randn(128, 128, dtype=torch.float16))
    with pytest.raises(NotImplementedError, match="bf16 models"):
        F.linear(torch.randn(2, 128, dtype=torch.float16), w16)
    w = to_nf4(torch.randn(128, 128, dtype=torch.bfloat16))
    with pytest.raises(NotImplementedError, match="activations"):
        F.linear(torch.randn(2, 128), w)
    with pytest.raises(NotImplementedError, match="backward"):
        linear_nf4(torch.randn(2, 128, dtype=torch.bfloat16, requires_grad=True), w)
    with pytest.raises(NotImplementedError):
        w.split(64)
    with pytest.raises(NotImplementedError):
        w.new_zeros(4)
    with pytest.raises(NotImplementedError):
        w.as_strided((128, 128), (128, 1))


def test_tensor_plumbing_and_save_load(tmp_path):
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import NF4Tensor, quantize_, to_nf4

    t = to_nf4(torch.randn(256, 128, dtype=torch.bfloat16))
    for u in (t.detach(), t.clone(), t.cpu(), t.to("cpu")):
        assert isinstance(u, NF4Tensor) and u.shape == t.shape and u.dtype == t.dtype and u.block_size == 64
        assert torch.equal(u.get_original_weight(), t.get_original_weight())
    assert torch.equal(t.to(torch.float32), t.get_original_weight().float())   # to(dtype) dequantizes
    c = t.clone()
    assert c.quantized_data.data_ptr() != t.quantized_data.data_ptr()
    other = to_nf4(torch.randn(256, 128, dtype=torch.bfloat16))
    c.copy_(other)
    assert torch.equal(c.get_original_weight(), other.get_original_weight())
    with pytest.raises(NotImplementedError):
        c.copy_(to_nf4(torch.randn(128, 256, dtype=torch.bfloat16), 128, 64))

    def model():
        torch.manual_seed(0)
        m = nn.Sequential(nn.Linear(256, 192), nn.Linear(192, 256, bias=False)).to(torch.bfloat16)
        quantize_(m, NF4WeightOnlyConfig())
        return m

    m = model()
    torch.save(m.state_dict(), tmp_path / "sd.pt")
    sd = torch.load(tmp_path / "sd.pt", weights_only=True)
    assert isinstance(sd["0.weight"], NF4Tensor)
    m2 = nn.Sequential(nn.Linear(256, 192), nn.Linear(192, 256, bias=False)).to(torch.bfloat16)
    quantize_(m2, NF4WeightOnlyConfig())
    m2.load_state_dict(sd)
    for a, b in zip(m.parameters(), m2.parameters()):
        if isinstance(a, NF4Tensor):
            assert torch.equal(a.get_original_weight(), b.get_original_weight())
        else:
            assert torch.equal(a, b)


def test_fusion_leaves_nf4_linears_alone():
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import NF4Tensor, quantize_

    class Attn(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj, self.v_proj = (nn.Linear(256, 256, bias=False) for _ in range(3))

    m = Attn().to(torch.bfloat16)
    quantize_(m, NF4WeightOnlyConfig())
    assert fuse_parallel_linears(m) == 0
    assert all(type(getattr(m, n)) is nn.Linear and isinstance(getattr(m, n).weight, NF4Tensor)
               for n in ("q_proj", "k_proj", "v_proj"))


def test_meta_shapes_and_schema():
    import ao_b200  # noqa: F401

    N, K = 200, 256
    meta = lambda *s, dt=torch.bfloat16: torch.empty(*s, dtype=dt, device="meta")
    y = torch.ops.ao_b200.nf4_linear(meta(130, K), meta(N * K // 2, dt=torch.uint8), meta(N * K // 64, dt=torch.int8),
                                     meta(N * K // 64 // 256), meta(()), meta(16), 64, 256, None)
    assert y.shape == (130, N) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(torch.ops.ao_b200.nf4_linear.default._schema).endswith(
        "(Tensor x, Tensor quantized_data, Tensor quantized_scalers, Tensor quantization_factor, Tensor scaler_mean, "
        "Tensor nf4, int block_size, int scaler_block_size, Tensor? bias) -> Tensor")


def test_c_abi_rejections():
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    z = ctypes.c_size_t(0)
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15

    def call(ldx, M, K, N, bs=64, sbs=256, x=None, p=None):
        P = ctypes.c_void_p(p)
        return lib.ao_nf4_linear(ctypes.c_void_p(x), ldx, M, K, P, P, P, P, P, bs, sbs, N, None, P, None, z, None)

    err = lambda: lib.ao_b200_last_error()
    assert call(4096, 4, 4096, 128, bs=40) == -1 and b"multiple of 16" in err()
    assert call(4096, 4, 4096, 128, bs=0) == -1 and b"block_size" in err()
    assert call(4160, 4, 4160, 128, bs=128) == -1 and b"multiple of block_size" in err()
    assert call(4112, 4, 4112, 256, bs=16, sbs=1) == -1 and b"multiple of 32" in err()
    assert call(4096, 4, 4096, 130, sbs=256) == -1 and b"scaler_block_size" in err()   # 8320 scalers
    assert call(4096, 4, 4096, 130, sbs=0) == -1 and b"scaler_block_size" in err()
    assert call(4096, 4, 4096, 1 << 24, bs=16, sbs=1) == -1 and b"int32 range" in err()
    assert call(4096, 4, 0, 128) == -1 and b"bad sizes" in err()
    assert call(4100, 4, 4096, 128) == -1 and b"multiple of 8" in err()
    assert call(4088, 4, 4096, 128) == -1 and b"ldx" in err()
    assert call(4096, 4, 4096, 130, sbs=65) == -1 and b"null pointer" in err()   # any N is a valid size
    assert call(4096, 4, 4096, 128, x=a + 8, p=a) == -1 and b"x must be 16-byte aligned" in err()
    assert call(4096, 4, 4096, 128, x=a) == -1 and b"null pointer" in err()
    assert call(4096, 0, 4096, 128) == 0   # no rows: nothing is read


def _policy():
    src = open(os.path.join(ROOT, "ao_b200", "csrc", "lowp_linear.cu")).read()
    body = src[src.index("struct Nf4Fmt {"):]
    return body[:body.index("struct Raw")]


@pytest.fixture
def nf4_model(monkeypatch):
    """Nf4Fmt in the stream-K model for the test that needs it: its widths and its stage layout (W_BYTES, AUX_BYTES,
    X_ELEM_BYTES, DECODE_2CTA, PROMOTE, MAX_N_MMA), 8 KiB of codes and 2 KiB of decoded scalers plus the 32-byte code
    table.  The model's own tables stay as they are: the plan tests pin their set of formats."""
    monkeypatch.setitem(sk.WIDTHS, "nf4", (16, 32, 64, 128))
    monkeypatch.setitem(sk.POLICIES, "nf4", (8192, 128 * 16 + 32, 2, False, False, 128))


@pytest.mark.parametrize("n_mma", [16, 32, 64, 128])
def test_tiles_registers_stack_and_shared_memory(n_mma, nf4_model):
    """ts_gemm_kernel<Nf4Fmt, N>: one CTA per SM (its aux fillers run at the kernel's register count), every tile at
    most 168 registers and a ring within 200 KB, never any stack."""
    body = _policy()
    assert "W_BYTES = ROWS * KCHUNK / 2;" in body and "AUX_BYTES = LUT_OFF + 32;" in body and "LUT_OFF = ROWS * 16;" in body
    assert "static constexpr bool DECODE_2CTA = false;" in body and "AUX_FILL = true;" in body
    assert sk.POLICIES["nf4"][:2] == (8192, 128 * 16 + 32)
    usage = resource_usage()
    assert ("Nf4Fmt", n_mma) in usage, f"ts_gemm_kernel<Nf4Fmt, {n_mma}> not built"
    reg, stack = usage[("Nf4Fmt", n_mma)]
    assert reg <= 168, reg
    assert stack == 0, f"ts_gemm_kernel<Nf4Fmt, {n_mma}>: {stack} bytes of stack"
    _, ctas, stages, _ = sk.ring("nf4", n_mma)
    assert ctas == 1 and stages >= 2
    assert sk.ring_smem("nf4", n_mma) + RESERVED_PER_CTA <= SMEM_PER_SM
