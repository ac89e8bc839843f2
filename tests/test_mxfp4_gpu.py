"""mxfp4 on the GPU: the quantizer bit for bit against the torch restatement run on CUDA, the exactness of both
operands' dequantization, the GEMM bit for bit on exact operands (every forced stream-K grid, every token tile, K and N
tails, bias, several activation slabs, the Llama-3-8B projections), the MXTensor handler's accuracy and the golden
linear, and the execution modes (CUDA graph, PDL chain, torch.compile, fusion, narrow + copy_ loading).

Exact operands: e2m1 codes of every value times e8m0 scales whose bytes vary over a wide range from row to row (bytes
80..171) and by at most one within a row.  Every product is then a multiple of the output's quantum u = 2^-2 x
2^(lowest x byte + lowest w byte - 254) and the sum of K of them stays below 2^24 u, so the fp32 accumulation is exact
in any order and the only rounding is bf16(sum + bias), which the reference computes the same way."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import streamk_model as sk
from test_block_quantizers_gpu import to_blocked
from test_mxfp4_host import mxfp4_dequant, mxfp4_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"
FP4 = torch.float4_e2m1fn_x2


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def sqnr(ref, got):
    ref, got = ref.float(), got.float()
    d = (ref - got).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


def bits(t):
    return t.contiguous().view(torch.int16)


# ---------------------------------------------------------------- quantizer
def bf16_sweep():
    """Every bf16 bit pattern, in blocks of 32, plus blocks built around each rounding tie, the amax extremes, zero
    blocks, +-inf and NaN."""
    allb = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).reshape(-1, 32)
    rows = [allb]
    # ties: amax 6 * 2^j puts the scale at 2^j, so element t * 2^j is exactly the tie t of the e2m1 grid
    ties = torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, 0.3, 4.9, 5.1, 6.0], dtype=torch.float32)
    for j in (-126, -100, -20, -1, 0, 1, 7, 60, 120):
        blk = torch.zeros(len(ties) * 2 + 2, 32, dtype=torch.float32)
        for i, t in enumerate(ties):
            blk[2 * i, 0], blk[2 * i, 1] = 6.0 * 2.0**j, t * 2.0**j
            blk[2 * i + 1, 0], blk[2 * i + 1, 1] = -6.0 * 2.0**j, -t * 2.0**j
        blk[-2, 0] = 6.0 * 2.0**j * 1.0078125          # amax just above a power of two: the scale rounds up
        blk[-1, :] = torch.linspace(-1, 1, 32) * 2.0**j
        rows.append(blk.to(torch.bfloat16))
    big = torch.finfo(torch.bfloat16).max
    ext = torch.zeros(8, 32, dtype=torch.bfloat16)
    ext[0, 0] = big                                   # amax > 6 * 2^125: byte 253, code 4 dequantizes to inf
    ext[1, :] = torch.tensor(2.0**-133).to(torch.bfloat16)   # the smallest subnormal: byte 0
    ext[2, 5] = float("inf")
    ext[3, 7] = float("-inf")
    ext[4, 9] = float("nan")
    ext[5, :] = -big
    ext[6, 3] = 6.0 * 2.0**126                        # byte 253 with code 4 and 6 present
    ext[6, 4] = 4.0 * 2.0**126
    rows.append(ext)                                   # (row 7: a zero block)
    return torch.cat(rows).reshape(-1, 256)


def test_quantizer_bit_exact_over_every_bf16_value(ops):
    x = bf16_sweep().to(DEV)
    M, K = x.shape
    q, s = ops.mxfp4_quantize(x, False)
    qr, sr = mxfp4_ref(x)
    assert torch.equal(s, sr), f"{int((s != sr).sum())} scale bytes differ"
    assert int(s.max()) == 255 and int(s.min()) == 0 and bool((s == 253).any())
    ok = (sr != 255).repeat_interleave(16, dim=1)       # the codes of NaN blocks are not restated
    assert torch.equal(q[ok], qr[ok]), f"{int((q[ok] != qr[ok]).sum())} code bytes differ"
    qb, sb = ops.mxfp4_quantize(x, True)
    assert torch.equal(qb, q) and torch.equal(sb.reshape(-1), to_blocked(sr))   # padding included (zero)
    # dequantize = the reference's dequantize of the reference's bytes
    from ao_b200.prototype.mx_formats import MXTensor

    t = MXTensor.to_mx(x, FP4)
    d = t.dequantize(torch.float32)
    want = mxfp4_dequant(qr, sr)
    assert torch.equal(torch.isnan(d), torch.isnan(want)) and torch.equal(d[~torch.isnan(d)], want[~torch.isnan(want)])
    assert bool(torch.isinf(d).any())                   # code 4 / 6 at byte 253


@pytest.mark.parametrize("M,K", [(1, 32), (130, 96), (257, 4128)])
def test_quantizer_blocked_padding_and_row_strides(ops, M, K):
    g = torch.Generator(device="cpu").manual_seed(M + K)
    wide = (torch.randn(M, K + 64, generator=g) * torch.logspace(-4, 4, M)[:, None]).to(torch.bfloat16).to(DEV)
    x = wide[:, 32:32 + K]                              # a column slice: row pitch K + 64
    qr, sr = mxfp4_ref(x.contiguous())
    for swz in (False, True):
        q, s = ops.mxfp4_quantize(x, swz)
        assert torch.equal(q, qr)
        assert torch.equal(s.reshape(-1), to_blocked(sr) if swz else sr.reshape(-1))


# ---------------------------------------------------------------- dequantization exactness (one-hot reads)
def _blocked(s):
    return to_blocked(s).contiguous()


def test_weight_and_activation_dequant_exact_for_every_code_and_byte(ops):
    """Weight row n = one (code, byte) pair at k = 0; a one-hot activation (code 2 = 1.0 at byte 127) reads it back.
    The activation side the same with the roles swapped.  Bytes 0x00..0xFE exact (inf where the product overflows,
    as in the reference's fp32 dequantize), 0xFF NaN."""
    K = 32
    codes = torch.arange(16, dtype=torch.uint8).repeat_interleave(256)
    bytes_ = torch.arange(256, dtype=torch.int32).repeat(16).to(torch.uint8)
    N = codes.numel()
    wq = torch.zeros(N, K // 2, dtype=torch.uint8)
    wq[:, 0] = codes
    ws = bytes_.reshape(N, 1)
    want = mxfp4_dequant(wq, ws)[:, 0]                  # fp32, the reference's dequantize
    xq = torch.zeros(1, K // 2, dtype=torch.uint8)
    xq[0, 0] = 2
    xs = torch.full((1, 1), 127, dtype=torch.uint8)
    y = ops.mxfp4_linear(xq.to(DEV), _blocked(xs.to(DEV)), wq.to(DEV), _blocked(ws.to(DEV)), None)
    got = y[0].float().cpu()
    nan = bytes_ == 255
    assert bool(torch.isnan(got[nan]).all())
    assert torch.equal(got[~nan], want[~nan].to(torch.bfloat16).float()) and torch.equal(got[~nan], want[~nan])
    # activation side: M = N rows of (code, byte), one weight row reading k = 0
    y = ops.mxfp4_linear(wq.to(DEV), _blocked(ws.to(DEV)), xq.to(DEV), _blocked(xs.to(DEV)), None)
    got = y[:, 0].float().cpu()
    assert bool(torch.isnan(got[nan]).all()) and torch.equal(got[~nan], want[~nan])
    assert bool(torch.isinf(got).any()) and float(got[~nan & ~torch.isinf(got)].abs().max()) == 1.5 * 2.0**127


# ---------------------------------------------------------------- exact operands
class Exact:
    def __init__(self, M, N, K, seed=0, bias=True):
        g = torch.Generator(device="cpu").manual_seed(seed * 1000003 + M * 131 + N * 7 + K)
        self.M, self.N, self.K = M, N, K
        nb = -(-K // 32)
        xc = torch.randint(0, 16, (M, K), generator=g, dtype=torch.uint8)
        wc = torch.randint(0, 16, (N, K), generator=g, dtype=torch.uint8)
        xs = (torch.randint(80, 171, (M, 1), generator=g) + torch.randint(0, 2, (M, nb), generator=g)).to(torch.uint8)
        ws = (torch.randint(80, 171, (N, 1), generator=g) + torch.randint(0, 2, (N, nb), generator=g)).to(torch.uint8)
        self.xq, self.wq = (xc[:, 0::2] | xc[:, 1::2] << 4), (wc[:, 0::2] | wc[:, 1::2] << 4)
        X, W = mxfp4_dequant(self.xq, xs).double(), mxfp4_dequant(self.wq, ws).double()
        u = 0.25 * torch.pow(2.0, xs.double().min(1).values[:, None] + ws.double().min(1).values[None, :] - 254)
        acc = X.to(DEV) @ W.to(DEV).t()
        assert bool(((X.abs().to(DEV) @ W.abs().to(DEV).t()) < 2.0**24 * u.to(DEV)).all()), "premise"
        assert torch.equal(acc.float().double(), acc), "premise: the sums are fp32 values"
        self.bias = (torch.randn(N, generator=g) * 2.0**20).to(torch.bfloat16).to(DEV) if bias else None
        y = acc.float() + (self.bias.float() if bias else 0.0)
        self.ref = y.to(torch.bfloat16)
        self.xq, self.wq = self.xq.to(DEV), self.wq.to(DEV)
        self.xs, self.ws = _blocked(xs.to(DEV)), _blocked(ws.to(DEV))
        self.xs_plain, self.ws_plain = xs.to(DEV), ws.to(DEV)

    def run(self, ops, m=None):
        m = self.M if m is None else m
        xs = self.xs if m == self.M else _blocked(self.xs_plain[:m])
        return ops.mxfp4_linear(self.xq[:m], xs, self.wq, self.ws, self.bias)

    def check(self, ops, m=None, what=""):
        m = self.M if m is None else m
        y = self.run(ops, m)
        bad = bits(y) != bits(self.ref[:m])
        assert not bool(bad.any()), f"M={m} N={self.N} K={self.K} {what}: {int(bad.sum())} wrong, first at {bad.nonzero()[0].tolist()}"


def grids(M, N, K):
    # mxfp4 splits work as mxfp8 does: the same token-tile widths (16, 32, 64, 128) and 128-k chunks (K tail included)
    U = sk.plan("mxfp8", M, N, K, grid=1).U
    return list(range(1, min(U, 132) + 1))


@pytest.mark.parametrize("M,N,K", [(16, 256, 1024), (129, 384, 2048), (300, 200, 4128)])
def test_every_forced_grid_bit_exact(ops, set_ctas, M, N, K):
    case = Exact(M, N, K)
    for G in grids(M, N, K):
        set_ctas(G)
        case.check(ops, what=f"grid={G}")
    set_ctas(0)
    case.check(ops, what="default grid")


@pytest.mark.parametrize("K", [160, 1024, 4128])
@pytest.mark.parametrize("N", [200, 256])
def test_token_tiles_and_tails_bit_exact(ops, set_ctas, N, K):
    case = Exact(300, N, K, seed=1)
    for G in (0, 1, 3, 7, 132):
        set_ctas(G)
        for m in (1, 16, 17, 32, 64, 128, 129, 300):
            case.check(ops, m, what=f"grid={G}")


def test_without_bias_bit_exact(ops):
    Exact(33, 136, 512, seed=2, bias=False).check(ops)


@pytest.mark.parametrize("rows", [37, 128])
def test_activation_slabs_bit_exact(rows):
    """ao_mxfp4_linear through ctypes with a workspace holding `rows` bf16 activation rows: several slabs."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.ao_mxfp4_linear.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, sz, vp]
    M, N, K = 300, 200, 1056
    c = Exact(M, N, K, seed=3)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    act_off = (64 * 1024 + sm * 128 * 128 * 4 + (1 << 20) - 1) & ~((1 << 20) - 1)
    ws_bytes = act_off + rows * K * 2
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    y = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    rc = lib.ao_mxfp4_linear(c.xq.data_ptr(), c.xs.data_ptr(), M, K, c.wq.data_ptr(), c.ws.data_ptr(), N,
                             c.bias.data_ptr(), y.data_ptr(), ws.data_ptr(), ws_bytes,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.ao_b200_last_error()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(c.ref))
    assert not bool(ws[:16384].ne(0).any()), "flags left raised"


LLAMA3_8B = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}


@pytest.mark.parametrize("proj", sorted(LLAMA3_8B))
def test_llama3_8b_projections_bit_exact(ops, proj):
    N, K = LLAMA3_8B[proj]
    case = Exact(512, N, K, seed=4)
    for m in (1, 32, 512):
        case.check(ops, m, what=proj)


# ---------------------------------------------------------------- the MXTensor handler
def _quantized_linear(K, N, bias=True, seed=0):
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.quantization import quantize_

    torch.manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref.load_state_dict(lin.state_dict())
    quantize_(lin, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4))
    return lin, ref


@pytest.mark.parametrize("shape", [(1, 4096), (5, 3, 4096), (64, 4096)])
def test_handler_accuracy(shape):
    from ao_b200.prototype.mx_formats import MXTensor

    lin, ref = _quantized_linear(4096, 1024)
    w = lin.weight
    assert isinstance(w, MXTensor) and w.elem_dtype == FP4 and tuple(w.shape) == (1024, 4096)
    assert w.qdata.shape == (1024, 2048) and w.qdata.dtype == torch.uint8
    x = torch.randn(*shape, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y = lin(x)
        x2 = x.reshape(-1, 4096)
        xd = MXTensor.to_mx(x2, FP4).dequantize(torch.float32)
        emu = xd @ w.dequantize(torch.float32).t() + lin.bias.float()
        assert y.shape == (*shape[:-1], 1024) and y.dtype == torch.bfloat16
        assert sqnr(emu.to(torch.bfloat16), y.reshape(-1, 1024)) >= 80.0   # both rounded to the bf16 output
        assert sqnr(ref(x), y) >= 12.0
        # non-bf16 input, M == 0 and a column-sliced input
        assert lin(x.float()).dtype == torch.float32
        assert lin(torch.empty(0, 4096, device=DEV, dtype=torch.bfloat16)).shape == (0, 1024)
        wide = torch.randn(x2.shape[0], 4096 + 256, device=DEV, dtype=torch.bfloat16)
        assert torch.equal(lin(wide[:, 128:128 + 4096]), lin(wide[:, 128:128 + 4096].contiguous()))


def test_golden_linear():
    d = np.load(os.path.join(GOLDEN, "mxfp4.npz"))
    b16 = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).to(DEV)
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.quantization import quantize_

    lin = nn.Linear(256, 192, bias=True, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(b16(d["lin_w"]))
        lin.bias.copy_(b16(d["lin_b"]))
    quantize_(lin, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4))
    assert np.array_equal(lin.weight.qdata.cpu().numpy(), d["lin_q"])
    assert np.array_equal(lin.weight.scale.view(torch.uint8).cpu().numpy().reshape(-1), d["lin_scale"].reshape(-1))
    with torch.no_grad():
        y = lin(b16(d["lin_x"]))
    assert sqnr(b16(d["lin_y"]), y) >= 60.0
    # the golden quantizer input through the CUDA op: the reference's bytes
    q, s = torch.ops.ao_b200.mxfp4_quantize(b16(d["x"]), True)
    assert np.array_equal(q.cpu().numpy(), d["q"]) and np.array_equal(s.cpu().numpy().reshape(-1), d["scale_blocked"].reshape(-1))


# ---------------------------------------------------------------- execution modes
def test_cuda_graph_replay(ops):
    case = Exact(32, 384, 1024, seed=5)
    other = Exact(32, 384, 1024, seed=6)
    xq, xs = case.xq.clone(), case.xs.clone()
    ops.mxfp4_linear(xq, xs, case.wq, case.ws, case.bias)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = ops.mxfp4_linear(xq, xs, case.wq, case.ws, case.bias)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(case.ref))
    # new activations in the static buffers; other's weights share case's, not its activations: recompute the ref
    xq.copy_(other.xq)
    xs.copy_(other.xs)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(ops.mxfp4_linear(other.xq, other.xs, case.wq, case.ws, case.bias)))


def test_pdl_chain_matches_serialized():
    """mxfp4 -> mxfp8 -> mxfp4 linears back to back (each quantizer and GEMM launched with PDL) against the same
    launches separated by synchronisations."""
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.quantization import quantize_

    torch.manual_seed(7)
    mk = lambda: nn.Linear(2048, 2048, bias=True, device=DEV, dtype=torch.bfloat16)
    l1, l2, l3 = mk(), mk(), mk()
    quantize_(l1, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4))
    quantize_(l2, MXDynamicActivationMXWeightConfig())
    quantize_(l3, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4))
    for M in (1, 32, 300):
        x = torch.randn(M, 2048, device=DEV, dtype=torch.bfloat16)
        with torch.no_grad():
            chained = l3(l2(l1(x)))
            a = l1(x)
            torch.cuda.synchronize()
            b = l2(a)
            torch.cuda.synchronize()
            serial = l3(b)
            torch.cuda.synchronize()
        assert torch.equal(bits(chained), bits(serial)), f"M={M}"


def test_torch_compile_fullgraph():
    lin, _ = _quantized_linear(1024, 512, seed=8)
    x = torch.randn(7, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        eager = lin(x)
        compiled = torch.compile(lin, fullgraph=True)(x)
    assert torch.equal(bits(eager), bits(compiled))


class Attn(nn.Module):
    def __init__(self, h=1024, kv=256, inter=2048, bias=False):
        super().__init__()
        mk = lambda k, n: nn.Linear(k, n, bias=bias, device=DEV, dtype=torch.bfloat16)
        self.q_proj, self.k_proj, self.v_proj = mk(h, h), mk(h, kv), mk(h, kv)
        self.gate_proj, self.up_proj = mk(h, inter), mk(h, inter)

    def forward(self, x):
        return self.q_proj(x), self.k_proj(x), self.v_proj(x), self.gate_proj(x), self.up_proj(x)


@pytest.mark.parametrize("M,bias", [(1, False), (32, True)])
def test_fusion_matches_separate(M, bias):
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig, MXTensor
    from ao_b200.quantization import quantize_

    torch.manual_seed(9)
    m = Attn(bias=bias)
    quantize_(m, MXDynamicActivationMXWeightConfig(activation_dtype=FP4, weight_dtype=FP4))
    x = torch.randn(M, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        ref = m(x)
    assert fuse_parallel_linears(m) == 2
    with torch.no_grad():
        got = m(x)
    for r, g in zip(ref, got):
        assert r.shape == g.shape and sqnr(r, g) > 60.0

    # exact weights: the fused launch equals each member bit for bit
    kw, pref = m.gate_proj.weight.act_quant_kwargs, m.gate_proj.weight.kernel_preference
    m2 = Attn(bias=bias)
    for i, name in enumerate(("q_proj", "k_proj", "v_proj", "gate_proj", "up_proj")):
        lin = getattr(m2, name)
        c = Exact(1, lin.out_features, 1024, seed=20 + i, bias=False)
        w = MXTensor(c.wq, c.ws.view(torch.float8_e8m0fnu).reshape(-1, 16 * 8), FP4, 32, torch.bfloat16, pref, kw, True)
        lin.weight = nn.Parameter(w, requires_grad=False)
    xs = Exact(M, 8, 1024, seed=30, bias=False)
    xe = mxfp4_dequant(xs.xq.cpu(), xs.xs_plain.cpu()).to(torch.bfloat16).to(DEV)   # exact in bf16
    with torch.no_grad():
        sep = m2(xe)
        assert fuse_parallel_linears(m2) == 2
        fused = m2(xe)
    for r, g in zip(sep, fused):
        assert torch.equal(bits(r), bits(g))


def test_narrow_and_copy_loading():
    """A tensor-parallel loader narrows the quantized parameter and copies a shard into it (reference mx_slice)."""
    src, _ = _quantized_linear(1024, 512, seed=10)
    dst, _ = _quantized_linear(1024, 512, seed=11)
    for lo, hi in ((0, 256), (256, 512)):
        d = dst.weight.narrow(0, lo, hi - lo)
        d.copy_(src.weight.narrow(0, lo, hi - lo))
    with torch.no_grad():
        dst.bias.copy_(src.bias)
    x = torch.randn(4, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        assert torch.equal(bits(dst(x)), bits(src(x)))
