"""float8 weight-only on the GPU: the e4m3 -> bf16 dequantization of the register-A fragment for every byte in every
fragment position and every kind of scale, the GEMM bit for bit on exact operands (every forced stream-K grid, every
token tile, K and N tails, bias, per-tensor scales, scales that are not bf16 values, the Llama-3-8B projections and
lm_head), the reference's CPU outputs of the golden fixture, the Float8Tensor handler, and the execution modes (CUDA
graph, PDL chain, torch.compile, fusion, narrow + copy_ loading and device moves, quantize_ -> forward launch counts).

Exact operands: codes c/8 (|c| <= 7) are e4m3 values, and every dequantized weight w~ = bf16(fp32(c/8 * s)) has 8
significant bits.  With bf16 scales of 3 bits (c * s exact) and activations -8..8 times 2^-3, a product is at most 392
quanta; with fp32 scales (w~ rounds) codes 1/8 and 3/8 keep a row's w~ within 2^10 quanta of its smallest step, and
activations -1..1.  Either way the sum of K products stays below 2^24 quanta: fp32 accumulates exactly in any order and
under any stream-K split, and the recipe's roundings bf16(bf16(sum) + bias) are what torch computes on any device."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import streamk_model as sk
from exact_operands import POISON_BF16, fp32_exact, gen, pick, pow2, randint
from test_float8_weight_only_host import f32, golden_cases, same_codes, within_one_step_of_the_sum

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"
E4M3 = torch.float8_e4m3fn


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


def bits(t):
    return t.contiguous().view(torch.int16)


def same_or_nan_or_zero(got, want):
    """bf16 tensors equal bit for bit, NaN matching NaN and +0 matching -0.  The sign of a zero weight cannot reach
    the linear's output: every product with it is a zero, and on the H100 the wgmma sum of a row whose every weight
    dequantizes to -0 (byte 0x80, or negative codes at the scale 2^-149) is +0, while torch's CPU sum keeps -0."""
    g, w = got.float().cpu(), want.float().cpu()
    nan_g, nan_w = torch.isnan(g), torch.isnan(w)
    zero = (g == 0) & (w == 0)
    same = bits(got).cpu() == bits(want).cpu()
    return bool(torch.equal(nan_g, nan_w) and (same | nan_g | zero).all())


def sqnr(ref, got):
    ref, got = ref.float(), got.float()
    d = (ref - got).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


# ---------------------------------------------------------------- the dequantization
FINITE = [b for b in range(256) if b & 0x7F != 0x7F]   # 254 bytes; 0x7F and 0xFF are NaN
LARGE = [b for b in FINITE if (b & 0x7F) >= 0x77]      # |value| >= 240


def dense_layout():
    """Row 128 v + i holds FINITE[(v + i + k) mod 254] at column k: position (i, k) of the 128 x 128 chunk sees every
    finite byte as v runs."""
    v = torch.arange(254)[:, None, None]
    i = torch.arange(128)[None, :, None]
    k = torch.arange(128)[None, None, :]
    return torch.tensor(FINITE, dtype=torch.uint8)[(v + i + k) % 254].reshape(254 * 128, 128)


def one_byte_layout(byte_set):
    """Row (b, v, i) holds byte_set[b] at column (i + v) mod 128 and zeros elsewhere: every position sees every byte
    of the set, alone in its row (so a one-hot read of an inf or NaN is not hidden by 0 * inf in the same row)."""
    b = torch.arange(len(byte_set))[:, None, None]
    v = torch.arange(128)[None, :, None]
    i = torch.arange(128)[None, None, :]
    n = ((b * 128 + v) * 128 + i).reshape(-1)
    q = torch.zeros(n.numel(), 128, dtype=torch.uint8)
    q[n, ((i + v) % 128).expand(len(byte_set), 128, 128).reshape(-1)] = torch.tensor(byte_set, dtype=torch.uint8)[
        b.expand(len(byte_set), 128, 128).reshape(-1)]
    return q


def scales(kind, n, seed):
    """n fp32 row scales: "bf16" values (8 significant bits) in [2^-4, 2^4); "fp32" with 24 significant bits in the same
    range; "tiny" 2^-140 .. 2^-118 (fp32 subnormal scales among them; most products are bf16 subnormals); "large"
    2^119 .. 2^121 (the largest codes overflow, in fp32 or in the rounding to bf16); "zero"."""
    g = torch.Generator().manual_seed(seed)
    mant = torch.randint(2**23, 2**24, (n,), generator=g).double() * 2.0**-23
    e = {"bf16": (-4, 3), "fp32": (-4, 3), "tiny": (-140, -118), "large": (119, 120), "zero": (0, 0)}[kind]
    ex = torch.randint(e[0], e[1] + 1, (n,), generator=g).double()
    if kind == "bf16":
        mant = torch.randint(128, 256, (n,), generator=g).double() / 128
    s = (mant * torch.pow(2.0, ex)).float()
    return torch.zeros(n) if kind == "zero" else s


def one_hot_reads(q, s):
    """What F.linear(eye(128), w~) gives for w~ = bf16(fp32(q) * s) computed by torch on the CPU: out[m, n] = w~[n, m]
    where the rest of row n is finite, NaN where another element of the row is inf or NaN (0 * inf)."""
    wt = (q.view(E4M3).float() * s[:, None]).to(torch.bfloat16)
    bad = ~torch.isfinite(wt.float())
    other = (bad.sum(1, keepdim=True) - bad.int()) > 0
    return torch.where(other, torch.full_like(wt, float("nan")), wt).t()


@pytest.mark.parametrize("layout", ["dense", "large", "nan"])
@pytest.mark.parametrize("kind", ["bf16", "fp32", "tiny", "large", "zero"])
def test_every_e4m3_byte_in_every_fragment_position(ops, layout, kind):
    """One-hot activations (the identity) read the dequantized weights back: each output is bf16(fp32(q) * s) itself
    (1 * w~ plus zero products), compared with torch's CPU dequantization bit for bit, NaN as NaN."""
    q = {"dense": dense_layout, "large": lambda: one_byte_layout(LARGE), "nan": lambda: one_byte_layout([0x7F, 0xFF])}[layout]()
    s = scales(kind, q.shape[0], seed=len(layout) * 31 + len(kind))
    want = one_hot_reads(q, s)
    x = torch.eye(128, device=DEV, dtype=torch.bfloat16)
    wq, sd = q.to(DEV).view(E4M3), s.to(DEV)
    y = ops.fp8_weight_linear(x, wq, sd, None)
    assert same_or_nan_or_zero(y, want), f"{layout} {kind}"
    if layout == "dense" and kind != "zero":
        assert bool(torch.isfinite(want.float()).any())
    if kind == "fp32" and layout == "dense":   # the same through a narrow token tile: 16 one-hot rows at a time
        for m0 in (0, 48, 112):
            assert same_or_nan_or_zero(ops.fp8_weight_linear(x[m0:m0 + 16], wq, sd, None), want[m0:m0 + 16])


def test_subnormal_and_overflow_products_occur():
    """The scale kinds above reach the ranges they are meant for."""
    q = dense_layout()
    tiny = (q.view(E4M3).float() * scales("tiny", q.shape[0], 1)[:, None]).to(torch.bfloat16).float()
    sub = (tiny != 0) & (tiny.abs() < 2.0**-126)
    assert int(sub.sum()) > 1000
    big = (one_byte_layout(LARGE).view(E4M3).float() * scales("large", 16 * 128 * 128, 2)[:, None]).to(torch.bfloat16)
    assert bool(torch.isinf(big.float()).any()) and bool((torch.isfinite(big.float()) & (big.float().abs() > 2.0**126)).any())
    assert bool((scales("tiny", 4096, 3).abs() < 2.0**-126).any())   # fp32 subnormal scales


# ---------------------------------------------------------------- exact operands
class Exact:
    """scales: "bf16" = bf16 values (c * s exact), "odd" = fp32 values with 24 significant bits (w~ rounds), "tensor" =
    one bf16 value expanded to [N] as the handler expands a per-tensor scale."""

    def __init__(self, M, N, K, seed=0, bias=True, scales="bf16", n_block=8192):
        g = gen(seed * 1000003 + M * 131 + N * 7 + K)
        self.M, self.N, self.K = M, N, K
        if scales == "odd":
            X = randint(-1, 1, (M, K), g).double()
            codes = pick([-3, -1, 0, 1, 3], (N, K), g) * 2.0**-3
            s = (randint(2**23, 2**24 - 1, (N,), g).double() * 2.0**-23 * pow2(randint(-12, -4, (N,), g))).float()
            assert not torch.equal(s.to(torch.bfloat16).float(), s)
            units = 2**10   # w~ in [s/8, 3s/8] rounded to 8 bits: under 2^10 steps of the smallest; |x| <= 1 step
        else:
            X = randint(-8, 8, (M, K), g).double() * 2.0**-3
            codes = randint(-7, 7, (N, K), g).double() * 2.0**-3
            s = (pick([3, 5, 7], (N,), g) * pow2(randint(-12, -4, (N,), g))).float()
            if scales == "tensor":
                s = s[:1].expand(N).contiguous()
            units = 7 * 7 * 8
        assert K * units < 2**24, "premise: K products stay below 2^24 quanta"
        self.x = X.to(torch.bfloat16)
        self.wq = codes.to(E4M3)
        assert torch.equal(self.wq.double(), codes)
        self.scale = s
        wt = (self.wq.float() * s[:, None]).to(torch.bfloat16)   # the reference's dequantize
        if scales != "odd":
            assert torch.equal(wt.double(), codes * s.double()[:, None]), "premise: c * s exact in bf16"
        else:
            assert not torch.equal(wt.double(), codes * s.double()[:, None])
        self.bias = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16) if bias else None
        self.ref = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        for n0 in range(0, N, n_block):   # the fp64 sums of n_block features at a time
            n1 = min(N, n0 + n_block)
            acc = X @ wt[n0:n1].double().t()
            fp32_exact(acc, "the sums")
            y = acc.float().to(torch.bfloat16)
            self.ref[:, n0:n1] = y if self.bias is None else y + self.bias[n0:n1]
        del wt

    def run(self, ops, m=None):
        return ops.fp8_weight_linear(self.x[: self.M if m is None else m], self.wq, self.scale, self.bias)

    def check(self, ops, m=None, what=""):
        m = self.M if m is None else m
        y = self.run(ops, m)
        bad = bits(y) != bits(self.ref[:m])
        assert not bool(bad.any()), f"M={m} N={self.N} K={self.K} {what}: {int(bad.sum())} wrong, first at {bad.nonzero()[0].tolist()}"
        bits(y).fill_(POISON_BF16)   # a later launch cannot inherit these values through the caching allocator


def grids(M, N, K):
    # the work splits as mxfp8's does: the same token-tile widths (16, 32, 64, 128) and 128-k chunks (K tail included)
    U = sk.plan("mxfp8", M, N, K, grid=1).U
    return list(range(1, min(U, 132) + 1))


@pytest.mark.parametrize("M,N,K", [(16, 256, 1024), (129, 384, 2048), (300, 200, 4112)])
def test_every_forced_grid_bit_exact(ops, set_ctas, M, N, K):
    case = Exact(M, N, K, scales="odd")
    for G in grids(M, N, K):
        set_ctas(G)
        case.check(ops, what=f"grid={G}")
    set_ctas(0)
    case.check(ops, what="default grid")


@pytest.mark.parametrize("K", [144, 1024, 4112])
@pytest.mark.parametrize("N", [77, 200, 256])
def test_token_tiles_and_tails_bit_exact(ops, set_ctas, N, K):
    case = Exact(300, N, K, seed=1)
    for G in (0, 1, 3, 7, 132):
        set_ctas(G)
        for m in (1, 16, 17, 32, 33, 64, 65, 128, 129, 300):
            case.check(ops, m, what=f"grid={G}")


@pytest.mark.parametrize("scales", ["odd", "bf16", "tensor"])
@pytest.mark.parametrize("bias", [False, True])
def test_scale_kinds_and_bias_bit_exact(ops, set_ctas, scales, bias):
    case = Exact(130, 136, 528, seed=2, bias=bias, scales=scales)
    for G in (0, 5):
        set_ctas(G)
        for m in (3, 130):
            case.check(ops, m, what=f"{scales} bias={bias} grid={G}")


def test_row_strided_activations_and_unaligned_scales(ops):
    case = Exact(40, 200, 528, seed=3)
    wide = torch.zeros(40, 528 + 72, device=DEV, dtype=torch.bfloat16)
    wide[:, 64:64 + 528] = case.x
    y = ops.fp8_weight_linear(wide[:, 64:64 + 528], case.wq, case.scale, case.bias)
    assert torch.equal(bits(y), bits(case.ref))
    # a scale view that does not start on 16 bytes (rows 1.. of a longer vector) is copied by the op for the TMA load
    s = torch.cat([torch.ones(1, device=DEV), case.scale])[1:]
    assert s.data_ptr() % 16 != 0
    assert torch.equal(bits(ops.fp8_weight_linear(case.x, case.wq, s, case.bias)), bits(case.ref))


SERVED = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336), "lm_head": (128256, 4096)}


@pytest.mark.parametrize("proj", sorted(SERVED))
def test_llama3_8b_shapes_bit_exact(ops, proj):
    N, K = SERVED[proj]
    case = Exact(512, N, K, seed=4, scales="odd")
    for m in (1, 32, 512):
        case.check(ops, m, what=proj)


# ---------------------------------------------------------------- the reference's CPU outputs
def test_golden_fixture():
    """The fixture's one-hot inputs (xe): bit for bit (each output is one product).  Its random inputs (x): the fp32
    sums round in each implementation's own order, so within one bf16 step of the sum carried through the add
    (within_one_step_of_the_sum states the bound).  The zero row's NaN reaches every token, as in the reference."""
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, PerRow, PerTensor, quantize_

    d = np.load(os.path.join(GOLDEN, "float8_weight_only.npz"))
    b16 = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).to(DEV)
    for i, c, a in golden_cases(d):
        lin = nn.Linear(c["K"], c["N"], bias=c["bias"], device=DEV, dtype=torch.bfloat16)
        with torch.no_grad():
            lin.weight.copy_(b16(a["w"]))
            if c["bias"]:
                lin.bias.copy_(b16(a["b"]))
        quantize_(lin, Float8WeightOnlyConfig(granularity=PerTensor() if c["granularity"] == "PerTensor" else PerRow()))
        w = lin.weight
        assert isinstance(w, Float8Tensor) and w.act_quant_kwargs is None and list(w.block_size) == c["block_size"]
        assert same_codes(w.qdata.view(torch.uint8).cpu().numpy(), a["q"]), c
        assert np.array_equal(w.scale.cpu().numpy(), a["scale"]), c
        with torch.no_grad():
            ye, y = lin(b16(a["xe"])), lin(b16(a["x"]))
        want_e = torch.from_numpy(a["ye"].view(np.int16).copy()).view(torch.bfloat16)
        assert same_or_nan_or_zero(ye, want_e), c
        assert bool(torch.isnan(y[:, 1].float()).all()) != (c["granularity"] == "PerTensor")
        bias = None if a["b"] is None else f32(a["b"])
        got = y.cpu().view(torch.int16).numpy().view(np.uint16)
        assert within_one_step_of_the_sum(got, a["y"], f32(a["x"]), a["q"], a["scale"].reshape(-1), bias), c


# ---------------------------------------------------------------- the handler
def _quantized_linear(K, N, bias=True, seed=0, gran=None):
    from ao_b200.quantization import Float8WeightOnlyConfig, quantize_

    torch.manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref.load_state_dict(lin.state_dict())
    quantize_(lin, Float8WeightOnlyConfig() if gran is None else Float8WeightOnlyConfig(granularity=gran))
    return lin, ref


@pytest.mark.parametrize("shape", [(1, 4096), (5, 3, 4096), (300, 4096)])
def test_handler_accuracy(ops, shape):
    from ao_b200.quantization import Float8Tensor

    lin, ref = _quantized_linear(4096, 1000)
    w = lin.weight
    assert isinstance(w, Float8Tensor) and w.act_quant_kwargs is None and w.qdata.dtype == E4M3
    x = torch.randn(*shape, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        n0 = ops.launch_count()
        y = lin(x)
        assert ops.launch_count() - n0 == 1   # one kernel per linear: no activation quantizer
        assert y.shape == (*shape[:-1], 1000) and y.dtype == torch.bfloat16
        assert sqnr(ref(x), y) > 25.0   # the reference's own bar for this config
        # F.linear on the dequantized weight is the same arithmetic up to the order of the fp32 sums
        assert sqnr(F.linear(x, w.dequantize(), lin.bias), y) > 45.0
        # other activation dtypes are cast to bf16 and the result back
        for dt in (torch.float16, torch.float32):
            xd = x.to(dt)
            yd = lin(xd)
            assert yd.dtype == dt and torch.equal(yd, lin(xd.to(torch.bfloat16)).to(dt))
        assert lin(torch.empty(0, 4096, device=DEV, dtype=torch.bfloat16)).shape == (0, 1000)
        x2 = x.reshape(-1, 4096)
        wide = torch.randn(x2.shape[0], 4096 + 256, device=DEV, dtype=torch.bfloat16)
        assert torch.equal(lin(wide[:, 128:128 + 4096]), lin(wide[:, 128:128 + 4096].contiguous()))


def test_handler_per_tensor():
    from ao_b200.quantization import PerTensor

    lin, ref = _quantized_linear(1024, 520, gran=PerTensor(), seed=1)
    assert lin.weight.scale.shape == (1, 1)
    x = torch.randn(9, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        assert sqnr(ref(x), lin(x)) > 25.0
        assert sqnr(F.linear(x, lin.weight.dequantize(), lin.bias), lin(x)) > 45.0


# ---------------------------------------------------------------- execution modes
def test_cuda_graph_replay(ops):
    case, other = Exact(32, 384, 1024, seed=5), Exact(32, 384, 1024, seed=6)
    x = case.x.clone()
    ops.fp8_weight_linear(x, case.wq, case.scale, case.bias)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = ops.fp8_weight_linear(x, case.wq, case.scale, case.bias)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(case.ref))
    x.copy_(other.x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(ops.fp8_weight_linear(other.x, case.wq, case.scale, case.bias)))


CHAIN = """
import sys, torch, torch.nn as nn
sys.path.insert(0, {root!r})
from ao_b200.quantization import Float8WeightOnlyConfig, quantize_
torch.manual_seed(7)
ls = [nn.Linear(2048, 2048, bias=True, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
for l in ls:
    quantize_(l, Float8WeightOnlyConfig())
outs = []
with torch.no_grad():
    for M in (1, 32, 300):
        x = torch.randn(M, 2048, device="cuda", dtype=torch.bfloat16)
        outs.append(ls[2](ls[1](ls[0](x))))
torch.cuda.synchronize()
sys.stdout.buffer.write(b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs))
"""


def test_pdl_chain_matches_serialized_and_no_pdl():
    """Three weight-only linears back to back (each GEMM prefetches its weights under the previous one) against the
    same launches separated by synchronisations, and against a process that launches without PDL."""
    from ao_b200.quantization import Float8WeightOnlyConfig, quantize_

    torch.manual_seed(7)
    ls = [nn.Linear(2048, 2048, bias=True, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
    for l in ls:
        quantize_(l, Float8WeightOnlyConfig())
    outs = []
    with torch.no_grad():
        for M in (1, 32, 300):
            x = torch.randn(M, 2048, device=DEV, dtype=torch.bfloat16)
            chained = ls[2](ls[1](ls[0](x)))
            a = ls[0](x)
            torch.cuda.synchronize()
            b = ls[1](a)
            torch.cuda.synchronize()
            serial = ls[2](b)
            torch.cuda.synchronize()
            assert torch.equal(bits(chained), bits(serial)), f"M={M}"
            outs.append(chained)
    here = b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs)
    for no_pdl in ("0", "1"):
        env = dict(os.environ, AO_B200_NO_PDL=no_pdl)
        r = subprocess.run([sys.executable, "-c", CHAIN.format(root=ROOT)], env=env, stdout=subprocess.PIPE, check=True)
        assert r.stdout == here, f"AO_B200_NO_PDL={no_pdl}: the chain's outputs differ"


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


def _exact_weights(lin):
    """Weights c * 2^-6 (|c| <= 7) with c = 7 in every row: the row scale is 7 2^-6 / 448 = 2^-12 and the codes 64 c,
    so the dequantized weights are the weights themselves and the sums with activations -8..8 2^-3 are exact."""
    with torch.no_grad():
        w = torch.randint(-7, 8, lin.weight.shape, device=DEV).float()
        w[:, 0] = 7
        lin.weight.copy_((w * 2.0**-6).to(torch.bfloat16))
    return lin


@pytest.mark.parametrize("M,bias", [(1, False), (32, True), (200, True)])
def test_fusion_matches_separate(ops, M, bias):
    """q|k|v and gate|up as one launch each (cat_out_features already merges weight-only members: act_quant_kwargs is
    None in each).  On exact sums the fused launch equals the members bit for bit, whatever its stream-K split; the
    members stay loader-compatible views."""
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, quantize_

    torch.manual_seed(9)
    m = Attn(bias=bias)
    for lin in (m.q_proj, m.k_proj, m.v_proj, m.gate_proj, m.up_proj):
        _exact_weights(lin)
    quantize_(m, Float8WeightOnlyConfig())
    x = (torch.randint(-8, 9, (M, 1024), device=DEV).float() * 2.0**-3).to(torch.bfloat16)
    with torch.no_grad():
        ref = m(x)
    assert fuse_parallel_linears(m) == 2
    with torch.no_grad():
        n0 = ops.launch_count()
        got = m(x)
        assert ops.launch_count() - n0 == 2
    for r, g in zip(ref, got):
        assert r.shape == g.shape and torch.equal(bits(r), bits(g))
    k = m.k_proj.weight
    assert isinstance(k, Float8Tensor) and k.act_quant_kwargs is None and tuple(k.shape) == (256, 1024)
    # narrow + copy_ into a fused member writes through to the group's weight
    src = _exact_weights(nn.Linear(1024, 256, bias=False, device=DEV, dtype=torch.bfloat16))
    quantize_(src, Float8WeightOnlyConfig())
    for lo in (0, 128):
        m.k_proj.weight.narrow(0, lo, 128).copy_(src.weight.narrow(0, lo, 128))
    with torch.no_grad():
        want = src(x) if not bias else F.linear(x, src.weight, m.k_proj.bias)
        assert torch.equal(bits(m(x)[1]), bits(want))


def test_narrow_and_copy_loading_and_device_moves(tmp_path):
    src, _ = _quantized_linear(1024, 512, seed=10)
    dst, _ = _quantized_linear(1024, 512, seed=11)
    for lo, hi in ((0, 256), (256, 512)):
        dst.weight.narrow(0, lo, hi - lo).copy_(src.weight.narrow(0, lo, hi - lo))
    with torch.no_grad():
        dst.bias.copy_(src.bias)
    x = torch.randn(4, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        want = src(x)
        assert torch.equal(bits(dst(x)), bits(want))
        # a checkpoint saved from the GPU, loaded on the CPU and moved back
        torch.save(src.state_dict(), tmp_path / "w.pt")
        sd = torch.load(tmp_path / "w.pt", weights_only=True, map_location="cpu")
        assert sd["weight"].act_quant_kwargs is None and sd["weight"].device.type == "cpu"
        back = nn.Linear(1024, 512, bias=True, dtype=torch.bfloat16)
        back.load_state_dict(sd, assign=True)
        assert torch.equal(bits(back.to(DEV)(x)), bits(want))


def test_quantize_then_forward_launches(ops):
    """quantize_ on CUDA: the rowwise quantizer, then the fence that completes the weights before any GEMM may prefetch
    them; the forward right behind it is one launch and equals the forward after a synchronisation."""
    from ao_b200.quantization import Float8WeightOnlyConfig, quantize_

    torch.manual_seed(12)
    a = nn.Linear(4096, 256, bias=True, device=DEV, dtype=torch.bfloat16)
    b = nn.Linear(4096, 256, bias=True, device=DEV, dtype=torch.bfloat16)
    b.load_state_dict(a.state_dict())
    x = torch.randn(32, 4096, device=DEV, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    with torch.no_grad():
        quantize_(b, Float8WeightOnlyConfig())
        torch.cuda.synchronize()
        want = b(x)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        quantize_(a, Float8WeightOnlyConfig())
        n1 = ops.launch_count()
        got = a(x)
        n2 = ops.launch_count()
    torch.cuda.synchronize()
    assert n1 - n0 == 2 and n2 - n1 == 1, (n1 - n0, n2 - n1)
    assert torch.equal(bits(got), bits(want))
