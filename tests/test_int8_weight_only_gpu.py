"""int8 weight-only on the GPU: the int8 -> bf16 conversion of the register-A fragment for every value in every
fragment position, the GEMM bit for bit on exact operands (every forced stream-K grid, every token tile, K and N tails,
bias, per-tensor scales, scales that are not bf16 values, the Llama-3-8B projections and lm_head), the reference's CPU
outputs of the golden fixture, the Int8Tensor handler, and the execution modes (CUDA graph, PDL chain, torch.compile,
fusion, narrow + copy_ loading, quantize_ -> forward launch counts).

Exact operands: activations are integers -8..8 times 2^-3 and the weights any int8, so every product is a multiple of
2^-3 and the sum of K <= 14336 of them stays below 2^24 of those: fp32 accumulates exactly in any order and under any
stream-K split.  What remains are the recipe's three roundings, bf16(bf16(bf16(sum) * bf16(scale)) + bias), which torch
computes the same way on any device."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import streamk_model as sk
from exact_operands import POISON_BF16, fp32_exact, gen, randint
from test_int8_weight_only_host import f32, golden_cases, within_one_step_of_the_sum

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"


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


def sqnr(ref, got):
    ref, got = ref.float(), got.float()
    d = (ref - got).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


def recipe(acc, scale, bias):
    """The three roundings on an exact fp32 sum [M, n], as torch computes them: scale fp32 [n], bias bf16 [n] or None."""
    y = acc.to(torch.bfloat16) * scale.to(torch.bfloat16)
    return y if bias is None else y + bias


# ---------------------------------------------------------------- the conversion
def test_every_int8_value_in_every_fragment_position(ops):
    """Weight row 128 v + i holds int8((v + i + k) mod 256 - 128) at column k: position (i, k) of the 128 x 128 chunk
    sees all 256 values as v runs.  One-hot activations (the identity) read each column back; the scales have
    mantissa bits, so the output is bf16(q * bf16(s)) with a rounding."""
    i = torch.arange(128, device=DEV)
    v = torch.arange(256, device=DEV)
    q = ((v[:, None, None] + i[None, :, None] + i[None, None, :]) % 256 - 128).reshape(256 * 128, 128)
    wq = q.to(torch.int8)
    assert all(int((wq.reshape(256, 128, 128)[:, a, b].long() + 128).unique().numel()) == 256 for a, b in ((0, 0), (77, 9), (127, 127)))
    scale = ((torch.arange(256 * 128, device=DEV) % 61 + 64).float() * 2.0**-9)   # 64..124 x 2^-9: up to 7 bits
    x = torch.eye(128, device=DEV, dtype=torch.bfloat16)
    y = ops.int8_weight_linear(x, wq, scale, None)
    want = (q.t().float() * scale.to(torch.bfloat16).float()[None, :]).to(torch.bfloat16)
    assert torch.equal(bits(y), bits(want))
    # the same through the narrow tiles: 16 one-hot rows at a time
    for m0 in (0, 48, 112):
        assert torch.equal(bits(ops.int8_weight_linear(x[m0:m0 + 16], wq, scale, None)), bits(want[m0:m0 + 16]))


# ---------------------------------------------------------------- exact operands
class Exact:
    """scales: "odd" = fp32 values with 12 mantissa bits (the cast to bf16 rounds), "bf16" = bf16 values, "tensor" = one
    value expanded to [N] as the handler expands a per-tensor scale."""

    def __init__(self, M, N, K, seed=0, bias=True, scales="odd", n_block=8192):
        g = gen(seed * 1000003 + M * 131 + N * 7 + K)
        self.M, self.N, self.K = M, N, K
        assert K * 8 * 128 < 2**24, "premise: |x| <= 8 x 2^-3 and |q| <= 128, so K products stay below 2^24 x 2^-3"
        X = randint(-8, 8, (M, K), g).double() * 2.0**-3
        self.x = X.to(torch.bfloat16)
        self.wq = randint(-128, 127, (N, K), g).to(torch.int8)
        s = (randint(2048, 4095, (N,), g).float() * 2.0**-20) * torch.pow(2.0, randint(-6, 6, (N,), g).float())
        if scales == "bf16":
            s = s.to(torch.bfloat16).float()
        elif scales == "tensor":
            s = s[:1].expand(N).contiguous()
        else:
            assert not torch.equal(s.to(torch.bfloat16).float(), s)
        self.scale = s
        self.bias = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16) if bias else None
        self.ref = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        for n0 in range(0, N, n_block):   # the fp64 sums of n_block features at a time
            n1 = min(N, n0 + n_block)
            acc = X @ self.wq[n0:n1].double().t()
            fp32_exact(acc, "the sums")
            self.ref[:, n0:n1] = recipe(acc.float(), s[n0:n1], None if self.bias is None else self.bias[n0:n1])

    def run(self, ops, m=None):
        return ops.int8_weight_linear(self.x[: self.M if m is None else m], self.wq, self.scale, self.bias)

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
    case = Exact(M, N, K)
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


def test_one_hot_without_bias(ops):
    x = torch.zeros(2, 128, device=DEV, dtype=torch.bfloat16)
    x[0, 0], x[1, 0] = -1.0, 1.0
    wq = torch.zeros(16, 128, dtype=torch.int8, device=DEV)
    wq[1, 0] = 3
    y = ops.int8_weight_linear(x, wq, torch.full((16,), 0.5, device=DEV), None)
    want = recipe(x.float() @ wq.float().t(), torch.full((16,), 0.5, device=DEV), None)
    assert torch.equal(bits(y), bits(want)) and float(y[0, 1]) == -1.5 and float(y[1, 1]) == 1.5


def test_row_strided_activations(ops):
    case = Exact(40, 200, 528, seed=3)
    wide = torch.zeros(40, 528 + 72, device=DEV, dtype=torch.bfloat16)
    wide[:, 64:64 + 528] = case.x
    y = ops.int8_weight_linear(wide[:, 64:64 + 528], case.wq, case.scale, case.bias)
    assert torch.equal(bits(y), bits(case.ref))


SERVED = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336), "lm_head": (128256, 4096)}


@pytest.mark.parametrize("proj", sorted(SERVED))
def test_llama3_8b_shapes_bit_exact(ops, proj):
    N, K = SERVED[proj]
    case = Exact(512, N, K, seed=4)
    for m in (1, 32, 512):
        case.check(ops, m, what=proj)


# ---------------------------------------------------------------- the reference's CPU outputs
def test_golden_fixture():
    """The fixture's exact inputs (xe): bit for bit, the accumulation order cannot matter.  Its random inputs (x): the
    fp32 sums round in each implementation's own order, so within one bf16 step of the sum carried through the multiply
    and the add (within_one_step_of_the_sum states the bound)."""
    from ao_b200.quantization import Int8Tensor, Int8WeightOnlyConfig, PerRow, PerTensor, quantize_

    d = np.load(os.path.join(GOLDEN, "int8_weight_only.npz"))
    b16 = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).to(DEV)
    for i, c, a in golden_cases(d):
        lin = nn.Linear(c["K"], c["N"], bias=c["bias"], device=DEV, dtype=torch.bfloat16)
        with torch.no_grad():
            lin.weight.copy_(b16(a["w"]))
            if c["bias"]:
                lin.bias.copy_(b16(a["b"]))
        quantize_(lin, Int8WeightOnlyConfig(granularity=PerTensor() if c["granularity"] == "PerTensor" else PerRow()))
        w = lin.weight
        assert isinstance(w, Int8Tensor) and w.act_quant_kwargs is None and list(w.block_size) == c["block_size"]
        assert np.array_equal(w.qdata.cpu().numpy(), a["q"]) and np.array_equal(w.scale.cpu().numpy(), a["scale"]), c
        with torch.no_grad():
            ye, y = lin(b16(a["xe"])), lin(b16(a["x"]))
        assert np.array_equal(ye.cpu().view(torch.int16).numpy().view(np.uint16), a["ye"]), c
        bias = None if a["b"] is None else f32(a["b"])
        got = y.cpu().view(torch.int16).numpy().view(np.uint16)
        assert within_one_step_of_the_sum(got, a["y"], f32(a["x"]), a["q"], a["scale"].reshape(-1), bias), c


# ---------------------------------------------------------------- the handler
def _quantized_linear(K, N, bias=True, seed=0, gran=None):
    from ao_b200.quantization import Int8WeightOnlyConfig, quantize_

    torch.manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    ref.load_state_dict(lin.state_dict())
    quantize_(lin, Int8WeightOnlyConfig() if gran is None else Int8WeightOnlyConfig(granularity=gran))
    return lin, ref


@pytest.mark.parametrize("shape", [(1, 4096), (5, 3, 4096), (300, 4096)])
def test_handler_accuracy(ops, shape):
    from ao_b200.quantization import Int8Tensor

    lin, ref = _quantized_linear(4096, 1000)
    w = lin.weight
    assert isinstance(w, Int8Tensor) and w.act_quant_kwargs is None and w.qdata.dtype == torch.int8
    x = torch.randn(*shape, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        n0 = ops.launch_count()
        y = lin(x)
        assert ops.launch_count() - n0 == 1   # one kernel per linear: no activation quantizer
        assert y.shape == (*shape[:-1], 1000) and y.dtype == torch.bfloat16
        assert sqnr(ref(x), y) > 35.0
        # F.linear on the dequantized weight rounds q * s to bf16 before the sum instead of after: close, not equal
        assert sqnr(F.linear(x, w.dequantize(), lin.bias), y) > 40.0
        # other activation dtypes are cast to bf16 and the result back
        for dt in (torch.float16, torch.float32):
            xd = x.to(dt)
            yd = lin(xd)
            assert yd.dtype == dt and torch.equal(yd, lin(xd.to(torch.bfloat16)).to(dt))
        assert lin(torch.empty(0, 4096, device=DEV, dtype=torch.bfloat16)).shape == (0, 1000)
        x2 = x.reshape(-1, 4096)
        wide = torch.randn(x2.shape[0], 4096 + 256, device=DEV, dtype=torch.bfloat16)
        assert torch.equal(lin(wide[:, 128:128 + 4096]), lin(wide[:, 128:128 + 4096].contiguous()))


def test_handler_per_tensor_and_act_pre_scale():
    from ao_b200.quantization import Int8Tensor, PerTensor

    lin, ref = _quantized_linear(1024, 520, gran=PerTensor(), seed=1)
    assert lin.weight.scale.shape == (1, 1)
    x = torch.randn(9, 1024, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        assert sqnr(ref(x), lin(x)) > 30.0   # one scale for the whole weight
        w = lin.weight
        pre = (torch.rand(1024, device=DEV) + 0.5).to(torch.bfloat16)
        wp = Int8Tensor(w.qdata, w.scale, list(w.block_size), w.dtype, zero_point=w.zero_point, act_pre_scale=pre)
        assert torch.equal(bits(F.linear(x, wp, lin.bias)), bits(lin(x * pre)))


# ---------------------------------------------------------------- execution modes
def test_cuda_graph_replay(ops):
    case, other = Exact(32, 384, 1024, seed=5), Exact(32, 384, 1024, seed=6)
    x = case.x.clone()
    ops.int8_weight_linear(x, case.wq, case.scale, case.bias)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = ops.int8_weight_linear(x, case.wq, case.scale, case.bias)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(case.ref))
    x.copy_(other.x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(ops.int8_weight_linear(other.x, case.wq, case.scale, case.bias)))


CHAIN = """
import sys, torch, torch.nn as nn
sys.path.insert(0, {root!r})
from ao_b200.quantization import Int8WeightOnlyConfig, quantize_
torch.manual_seed(7)
ls = [nn.Linear(2048, 2048, bias=True, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
for l in ls:
    quantize_(l, Int8WeightOnlyConfig())
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
    from ao_b200.quantization import Int8WeightOnlyConfig, quantize_

    torch.manual_seed(7)
    ls = [nn.Linear(2048, 2048, bias=True, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
    for l in ls:
        quantize_(l, Int8WeightOnlyConfig())
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


@pytest.mark.parametrize("M,bias", [(1, False), (32, True), (200, True)])
def test_fusion_matches_separate(ops, M, bias):
    """q|k|v and gate|up as one launch each (cat_out_features already merges weight-only members: act_quant_kwargs is
    None in each).  On exact sums the fused launch equals the members bit for bit, whatever its stream-K split; the
    members stay loader-compatible views."""
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.quantization import Int8Tensor, Int8WeightOnlyConfig, quantize_

    torch.manual_seed(9)
    m = Attn(bias=bias)
    quantize_(m, Int8WeightOnlyConfig())
    x = (torch.randint(-8, 9, (M, 1024), device=DEV).float() * 2.0**-3).to(torch.bfloat16)   # exact sums: any split agrees
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
    assert isinstance(k, Int8Tensor) and k.act_quant_kwargs is None and tuple(k.shape) == (256, 1024)
    # narrow + copy_ into a fused member writes through to the group's weight
    src = nn.Linear(1024, 256, bias=False, device=DEV, dtype=torch.bfloat16)
    quantize_(src, Int8WeightOnlyConfig())
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
    from ao_b200.quantization import Int8WeightOnlyConfig, quantize_

    torch.manual_seed(12)
    a = nn.Linear(4096, 256, bias=True, device=DEV, dtype=torch.bfloat16)
    b = nn.Linear(4096, 256, bias=True, device=DEV, dtype=torch.bfloat16)
    b.load_state_dict(a.state_dict())
    x = torch.randn(32, 4096, device=DEV, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    with torch.no_grad():
        quantize_(b, Int8WeightOnlyConfig())
        torch.cuda.synchronize()
        want = b(x)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        quantize_(a, Int8WeightOnlyConfig())
        n1 = ops.launch_count()
        got = a(x)
        n2 = ops.launch_count()
    torch.cuda.synchronize()
    assert n1 - n0 == 2 and n2 - n1 == 1, (n1 - n0, n2 - n1)
    assert torch.equal(bits(got), bits(want))
