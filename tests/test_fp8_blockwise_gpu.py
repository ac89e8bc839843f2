"""Blockwise fp8 on the GPU: the 1x128 activation quantizer bit for bit against the torch rule (Float8Tensor.from_hp
with PerBlock([1, 128]) on CUDA tensors: all-zero, NaN, inf, zero-scale and subnormal-scale blocks, row-strided
input), the GEMM
bit for bit on exact operands (every forced stream-K grid, every token tile and M tail, bias or not, the Llama-3-8B
projections), random operands against an fp64 restatement of the reference's Triton loop, the handler through
quantize_ (2-D and 3-D inputs), and the execution modes (CUDA graph, PDL chain, torch.compile, fusion, launches).

Exact operands: e4m3 codes that are small integers and power-of-two scales.  Each 128-k chunk's wgmma sum is an
integer below 2^13 (exact in the tensor core's adder), its scaled value a power-of-two multiple of it, and the sum over
the chunks stays below 2^24 quanta: fp32 accumulates exactly in any order and under any stream-K split, so the output
is the fp64 sum rounded to bf16, then the bf16 bias add."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import streamk_model as sk
from exact_operands import POISON_BF16, gen, pow2, randint

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def transposed_scales(s):
    """[M, K/128] -> the kernel's [K/128, round_up(M, 4)] layout, pads zero."""
    M, KB = s.shape
    out = torch.zeros(KB, (M + 3) // 4 * 4, dtype=torch.float32, device=s.device)
    out[:, :M] = s.t()
    return out


def torch_rule(x):
    """Float8Tensor.from_hp(x, PerBlock([1, 128])) as the package's torch path computes it on the device."""
    from ao_b200.quantization import Float8Tensor, PerBlock

    t = Float8Tensor.from_hp(x, granularity=PerBlock([1, 128]))
    return t.qdata, t.scale


def sqnr(ref, y):
    ref, y = ref.double(), y.double()
    return float(20 * torch.log10(ref.norm() / (ref - y).norm()))


def same_f32(a, b):
    """fp32 tensors equal bit for bit, NaN matching NaN"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return bool(torch.equal(na, nb) and torch.equal(a.view(torch.int32)[~na], b.view(torch.int32)[~nb]))


def same_codes(a, b):
    """e4m3 codes equal, every NaN code (0x7F / 0xFF) matching every other"""
    ua, ub = a.view(torch.uint8).int(), b.view(torch.uint8).int()
    na, nb = (ua & 0x7F) == 0x7F, (ub & 0x7F) == 0x7F
    return bool(torch.equal(na, nb) and torch.equal(ua[~na], ub[~nb]))


# ---------------------------------------------------------------- the 1x128 quantizer
def edge_input(M, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, device=DEV, generator=g) * torch.logspace(-3, 3, K, device=DEV)[None, :]
    x[0, :128] = 0                                                     # all-zero block: s = 0, codes NaN
    if K >= 256:
        x[0, 128:256] = torch.randn(128, device=DEV, generator=g) * 2.0**-128    # scale rounds to 0: codes +-448
    if K >= 384:
        x[0, 256:384] = torch.randn(128, device=DEV, generator=g) * 2.0**-118    # subnormal fp32 scale
    if M > 1:
        x[1, 5] = float("nan")                                         # NaN block
        x[1, -3] = float("inf")                                        # inf amax: s = inf
    if M > 2:
        x[2, :128] = -0.0                                              # negative zeros
        x[2, 130] = torch.finfo(torch.bfloat16).max
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("M,K", [(1, 128), (3, 256), (5, 4096), (33, 14336), (300, 7168), (4097, 1024)])
def test_quantizer_matches_the_torch_rule(ops, M, K):
    x = edge_input(M, K, seed=M * 7 + K)
    q, st = ops.fp8_quantize_1x128(x)
    rq, rs = torch_rule(x)
    assert q.dtype == E4M3 and tuple(q.shape) == (M, K) and tuple(st.shape) == (K // 128, (M + 3) // 4 * 4)
    assert same_codes(q, rq), "codes"
    assert same_f32(st[:, :M].t().contiguous(), rs.contiguous()), "scales"
    assert bool((st[:, M:] == 0).all()), "pad entries"


def test_quantizer_row_strided_input(ops):
    x = edge_input(40, 1024, seed=3)
    wide = torch.full((40, 1024 + 192), float("nan"), device=DEV, dtype=torch.bfloat16)
    wide[:, 64:64 + 1024] = x
    q, st = ops.fp8_quantize_1x128(wide[:, 64:64 + 1024])
    rq, rs = torch_rule(x)
    assert same_codes(q, rq) and same_f32(st[:, :40].t().contiguous(), rs)


# ---------------------------------------------------------------- the GEMM on exact operands
class Exact:
    """codes x in -2..2, w in -2..2 (e4m3 integers); a_s = 2^[-2, 1], w_s = 2^[-1, 1]: a chunk's sum is below 2^9,
    its scaled value a multiple of 2^-3 below 2^11, and KT <= 128 chunks stay below 2^24 quanta"""

    def __init__(self, M, N, K, seed=0, bias=True):
        g = gen(seed * 1000003 + M * 131 + N * 7 + K)
        self.M, self.N, self.K = M, N, K
        KB = K // 128
        assert KB * 2**14 < 2**24, "premise: the sum stays below 2^24 quanta"
        X = randint(-2, 2, (M, K), g).double()
        W = randint(-2, 2, (N, K), g).double()
        self.a_s = pow2(randint(-2, 1, (M, KB), g)).float()
        self.w_s = pow2(randint(-1, 1, (N // 128, KB), g)).float()
        self.xq, self.wq = X.to(E4M3), W.to(E4M3)
        self.bias = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16) if bias else None
        acc = torch.zeros(M, N, dtype=torch.float64, device=DEV)
        for kb in range(KB):   # the reference's loop: acc += dot(a_kb, b_kb) * a_s[:, kb] * b_s[n/128, kb]
            part = X[:, kb * 128:(kb + 1) * 128] @ W[:, kb * 128:(kb + 1) * 128].t()
            acc += part * self.a_s[:, kb, None].double() * self.w_s[:, kb].double().repeat_interleave(128)[None, :]
        assert torch.equal(acc.float().double(), acc), "premise: the sums are exact in fp32"
        y = acc.float().to(torch.bfloat16)
        self.ref = y if self.bias is None else y + self.bias

    def run(self, ops, m=None):
        m = self.M if m is None else m
        return ops.fp8_blockwise_linear(self.xq[:m], transposed_scales(self.a_s[:m]), self.wq, self.w_s, self.bias)

    def check(self, ops, m=None, what=""):
        m = self.M if m is None else m
        y = self.run(ops, m)
        bad = bits(y) != bits(self.ref[:m])
        assert not bool(bad.any()), f"M={m} N={self.N} K={self.K} {what}: {int(bad.sum())} wrong, first at {bad.nonzero()[0].tolist()}"
        assert not bool(ops.debug_workspace(y).view(torch.int32)[:4096].ne(0).any()), f"M={m} {what}: flags left raised"
        bits(y).fill_(POISON_BF16)


def grids(M, N, K):
    U = sk.plan("fp8_blockwise", M, N, K, grid=1).U
    return list(range(1, min(U, 132) + 1))


@pytest.mark.parametrize("M,N,K", [(16, 256, 1024), (64, 384, 2048), (129, 128, 4096)])
def test_every_forced_grid_bit_exact(ops, set_ctas, M, N, K):
    case = Exact(M, N, K)
    for G in grids(M, N, K):
        set_ctas(G)
        case.check(ops, what=f"grid={G}")
    set_ctas(0)
    case.check(ops, what="default grid")


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("N,K", [(128, 128), (384, 1152)])
def test_token_tiles_and_tails_bit_exact(ops, set_ctas, N, K, bias):
    case = Exact(300, N, K, seed=1, bias=bias)
    for G in (0, 1, 3, 7, 132):
        set_ctas(G)
        for m in (1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 128, 129, 300):
            case.check(ops, m, what=f"grid={G}")


SERVED = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}


@pytest.mark.parametrize("proj", sorted(SERVED))
def test_llama3_8b_shapes_bit_exact(ops, proj):
    N, K = SERVED[proj]
    case = Exact(512, N, K, seed=4)
    for m in (1, 32, 512):
        case.check(ops, m, what=proj)


# ---------------------------------------------------------------- random operands
def triton_loop_fp64(xq, a_s, wq, w_s, bias):
    """The reference's loop in fp64 on the same codes and scales, then its roundings: bf16(acc), bf16 + bias."""
    M, K = xq.shape
    X, W = xq.double(), wq.double()
    acc = torch.zeros(M, W.shape[0], dtype=torch.float64, device=DEV)
    for kb in range(K // 128):
        part = X[:, kb * 128:(kb + 1) * 128] @ W[:, kb * 128:(kb + 1) * 128].t()
        acc += part * a_s[:, kb, None].double() * w_s[:, kb].double().repeat_interleave(128)[None, :]
    return acc


@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (77, 1024, 7168), (600, 512, 2048)])
def test_random_operands_within_tolerance(ops, M, N, K):
    from ao_b200.quantization import Float8Tensor, PerBlock

    torch.manual_seed(M + N + K)
    w = Float8Tensor.from_hp((torch.randn(N, K, device=DEV) * 0.02).to(torch.bfloat16), granularity=PerBlock([128, 128]))
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV).to(torch.bfloat16)
    xq, st = ops.fp8_quantize_1x128(x)
    y = ops.fp8_blockwise_linear(xq, st, w.qdata, w.scale, bias)
    acc = triton_loop_fp64(xq, st[:, :M].t(), w.qdata, w.scale, None)
    # the rowwise fp8 linear's bar against its fp64 sum (test_lowp_gpu.py): the e4m3 wgmma chain of a chunk adds in
    # the tensor core's reduced-precision accumulator
    assert sqnr(acc + bias.double(), y) > 45.0


# ---------------------------------------------------------------- the handler
def exact_module(lin):
    """Weights c 2^-6 (|c| <= 7) with c = 7 in every row of every 128-k block: each 128x128 block's scale is
    bf16(7 2^-6 / 448) = 2^-12 and the codes 64 c, exact"""
    with torch.no_grad():
        w = torch.randint(-7, 8, lin.weight.shape, device=DEV).float()
        w[:, ::128] = 7
        lin.weight.copy_((w * 2.0**-6).to(torch.bfloat16))
    return lin


def exact_input(*shape):
    """Activations r 2^-9 (|r| <= 4) with 448 2^-9 at the start of every 128-block: each block's scale is 2^-9 and its
    codes the integers r and 448, exact; every chunk's sum stays below 2^13 quanta of 64 (weight codes 64 c)"""
    x = torch.randint(-4, 5, shape, device=DEV).float()
    x[..., ::128] = 448
    return (x * 2.0**-9).to(torch.bfloat16)


def blockwise_config():
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock

    return Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])])


def reference_linear(x, w, bias):
    """The reference's handler restated: from_hp(x, PerBlock([1, 128])), the Triton loop in fp64, bf16, + bias"""
    xq, xs = torch_rule(x.reshape(-1, x.shape[-1]))
    acc = triton_loop_fp64(xq, xs, w.qdata, w.scale, None)
    y = acc.float().to(torch.bfloat16)
    if bias is not None:
        y = y + bias
    return y.reshape(*x.shape[:-1], -1)


@pytest.mark.parametrize("shape", [(7, 1024), (2, 3, 1024), (1, 130, 1024)])
def test_handler_bit_exact_through_quantize(ops, shape):
    from ao_b200.quantization import Float8Tensor, quantize_

    torch.manual_seed(5)
    lin = exact_module(nn.Linear(1024, 384, bias=True, device=DEV, dtype=torch.bfloat16))
    quantize_(lin, blockwise_config())
    assert isinstance(lin.weight, Float8Tensor) and list(lin.weight.block_size) == [128, 128]
    x = exact_input(*shape)
    with torch.no_grad():
        y = lin(x)
    assert y.shape == (*shape[:-1], 384) and y.dtype == torch.bfloat16
    assert torch.equal(bits(y), bits(reference_linear(x, lin.weight, lin.bias)))


def test_handler_random_within_tolerance():
    from ao_b200.quantization import quantize_

    torch.manual_seed(6)
    lin = nn.Linear(2048, 512, bias=True, device=DEV, dtype=torch.bfloat16)
    ref_w = lin.weight.detach().clone()
    quantize_(lin, blockwise_config())
    x = torch.randn(3, 11, 2048, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y = lin(x)
        assert sqnr(reference_linear(x, lin.weight, lin.bias), y) > 45.0
        assert sqnr(F.linear(x, ref_w, lin.bias), y) > 25.0


# ---------------------------------------------------------------- execution modes
def test_cuda_graph_replay(ops):
    torch.manual_seed(7)
    lin = exact_module(nn.Linear(1024, 256, bias=True, device=DEV, dtype=torch.bfloat16))
    quantize_blockwise(lin)
    x, other = exact_input(32, 1024), exact_input(32, 1024)
    with torch.no_grad():
        lin(x)   # warm-up outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = lin(x)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(y), bits(reference_linear(x, lin.weight, lin.bias)))
        x.copy_(other)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(y), bits(reference_linear(other, lin.weight, lin.bias)))


def quantize_blockwise(m):
    from ao_b200.quantization import quantize_

    quantize_(m, blockwise_config())
    return m


CHAIN = """
import sys, torch, torch.nn as nn
sys.path.insert(0, {root!r})
from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock, quantize_
torch.manual_seed(8)
ls = [nn.Linear(2048, 2048, bias=True, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
for l in ls:
    quantize_(l, Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])]))
outs = []
with torch.no_grad():
    for M in (1, 32, 300):
        x = torch.randn(M, 2048, device="cuda", dtype=torch.bfloat16)
        outs.append(ls[2](ls[1](ls[0](x))))
torch.cuda.synchronize()
sys.stdout.buffer.write(b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs))
"""


def test_pdl_chain_matches_serialized_and_no_pdl():
    """Three blockwise linears back to back (each quantizer and GEMM start under the kernel ahead of them) against the
    same launches separated by synchronisations, and against a process that launches without PDL."""
    torch.manual_seed(8)
    ls = [nn.Linear(2048, 2048, bias=True, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
    for l in ls:
        quantize_blockwise(l)
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
    torch.manual_seed(9)
    lin = quantize_blockwise(nn.Linear(1024, 512, bias=True, device=DEV, dtype=torch.bfloat16))
    x = torch.randn(7, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        eager = lin(x)
        compiled = torch.compile(lin, fullgraph=True)(x)
    assert torch.equal(bits(eager), bits(compiled))


class Attn(nn.Module):
    """Llama-3-8B's q|k|v (4096 + 1024 + 1024) and gate|up (14336 + 14336) over h = 4096"""

    def __init__(self, h=4096, kv=1024, inter=14336, bias=False):
        super().__init__()
        mk = lambda k, n: nn.Linear(k, n, bias=bias, device=DEV, dtype=torch.bfloat16)
        self.q_proj, self.k_proj, self.v_proj = mk(h, h), mk(h, kv), mk(h, kv)
        self.gate_proj, self.up_proj = mk(h, inter), mk(h, inter)

    def forward(self, x):
        return self.q_proj(x), self.k_proj(x), self.v_proj(x), self.gate_proj(x), self.up_proj(x)


@pytest.mark.parametrize("M,bias", [(1, False), (32, True), (200, True)])
def test_fusion_matches_separate(ops, M, bias):
    """q|k|v and gate|up fused into one blockwise weight each: one quantizer and one GEMM per group.  On exact operands
    the fused launch equals the members bit for bit, whatever its stream-K split."""
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.quantization import Float8Tensor

    torch.manual_seed(10)
    m = Attn(bias=bias)
    for lin in (m.q_proj, m.k_proj, m.v_proj, m.gate_proj, m.up_proj):
        exact_module(lin)
    quantize_blockwise(m)
    x = exact_input(M, 4096)
    with torch.no_grad():
        ref = m(x)
    assert fuse_parallel_linears(m) == 2
    with torch.no_grad():
        n0 = ops.launch_count()
        got = m(x)
        assert ops.launch_count() - n0 == 4
    for r, g in zip(ref, got):
        assert r.shape == g.shape and torch.equal(bits(r), bits(g))
    k = m.k_proj.weight
    assert isinstance(k, Float8Tensor) and list(k.block_size) == [128, 128] and tuple(k.scale.shape) == (8, 32)


def test_two_launches_per_linear_and_device_moves(ops, tmp_path):
    torch.manual_seed(11)
    lin = quantize_blockwise(nn.Linear(4096, 1024, bias=True, device=DEV, dtype=torch.bfloat16))
    x = torch.randn(5, 4096, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        lin(x)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        want = lin(x)
        assert ops.launch_count() - n0 == 2
        torch.save(lin.state_dict(), tmp_path / "w.pt")
        sd = torch.load(tmp_path / "w.pt", weights_only=True, map_location="cpu")
        assert sd["weight"].device.type == "cpu" and list(sd["weight"].block_size) == [128, 128]
        back = nn.Linear(4096, 1024, bias=True, dtype=torch.bfloat16)
        back.load_state_dict(sd, assign=True)
        assert torch.equal(bits(back.to(DEV)(x)), bits(want))
