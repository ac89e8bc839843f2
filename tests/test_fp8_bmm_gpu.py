"""torch.bmm on rowwise e4m3 Float8Tensor weights (torch.ops.ao_b200.fp8_rowwise_bmm and the Float8Tensor bmm handler)
on the GPU, in both weight layouts: the transposed view of a stored [B, N, K] weight (the grouped e4m3 kernel) and a
stored [B, K, N] weight (the N-major kernel, which transposes each weight tile on chip).

* bit-exact under every forced stream-K grid with exact-product operands (the scheme of tests/exact_operands.py),
  with K and N tails, M from 1 to 200 and B = 1; the workspace flags must be back to zero after each launch;
* random operands: both layouts give the same bits, and match the fp64 product of the codes and bf16 torch.bmm;
* the reference's test_bmm and test_bmm_weight_in_bkn_layout through quantize_, and a llama-models expert block
  with [E, K, N] weights against the same block run batch by batch;
* Llama-4-Scout expert shapes with B = 2;
* a CUDA graph replay, torch.compile(fullgraph=True), a PDL chain against a serialized run and the launch count.
"""
import copy
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

import exact_operands as ex
from test_grouped_int4_gpu import Chain, Head

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    d = (ref - out).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


def as_layout(w_nk, layout):
    """[B, K, N] view of the codes w_nk [B, N, K]: "nk" the transposed view of w_nk, "kn" a stored [B, K, N] copy."""
    t = w_nk.transpose(-2, -1)
    return t.contiguous() if layout == "kn" else t


def host_units(B, M, K, N):
    """The units launch_gemm sizes the grid for (ts_gemm.cuh: per-expert m-blocks bounded by ceil(BM / N_MMA) + B)."""
    BM = B * M
    n_mma = 16 if BM <= 16 else 32 if BM <= 32 else 64
    return -(-N // 128) * (-(-BM // n_mma) + min(B, BM)) * -(-K // 128)


# ------------------------------------------------------------------------------------------------ exact operands
# (B, M, K, N): K and N tails, every token tile, B = 1
EXACT_CASES = [(1, 1, 256, 128), (3, 5, 208, 144), (2, 16, 512, 256), (1, 33, 1024, 144), (4, 64, 208, 128),
               (2, 200, 384, 272), (1, 200, 2048, 128)]


class ExactCase:
    """X in {-7..7} / 4, W in {-7..7} / 8 and scales of three significant bits: every product, chunk sum and scaled
    output is exact (exact_operands.premise), so the output must equal the fp64 reference rounded once to bf16."""

    def __init__(self, B, M, K, N, seed):
        g = ex.gen(seed * 7919 + B * 131 + M * 31 + N * 7 + K)
        X = ex.randint(-7, 7, (B, M, K), g).double() * 2.0**-2
        W = ex.randint(-7, 7, (B, N, K), g).double() * 2.0**-3
        self.xq, self.wq = X.to(E4M3), W.to(E4M3)
        assert torch.equal(self.xq.double(), X) and torch.equal(self.wq.double(), W)
        for b in range(B):
            ex.premise(X[b], W[b], chunk=True)
        rs = ex.pick(ex.ODD, (B, M), g) * 2.0**-8
        sw = ex.pick(ex.ODD, (B, N), g) * 2.0**-9
        ref = torch.bmm(X, W.transpose(-2, -1)) * rs[:, :, None] * sw[:, None, :]
        ex.fp32_exact(rs[:, :, None] * sw[:, None, :], "bmm: x_scale * w_scale")
        ex.fp32_exact(ref, "bmm: acc * scales")
        self.rs, self.sw = rs.float().reshape(-1), sw.float()
        self.ref = ref.float().to(torch.bfloat16)
        self.B, self.M, self.K, self.N = B, M, K, N

    def run(self, ops, layout):
        return ops.fp8_rowwise_bmm(self.xq, self.rs, as_layout(self.wq, layout), self.sw)


@pytest.mark.parametrize("layout", ["kn", "nk"])
@pytest.mark.parametrize("ci", range(len(EXACT_CASES)))
def test_exact_operands_every_grid(ops, set_ctas, ci, layout):
    B, M, K, N = EXACT_CASES[ci]
    case = ExactCase(B, M, K, N, seed=ci)
    w = as_layout(case.wq, layout)
    flags = ops.debug_workspace(case.xq).view(torch.int32)[:4096]
    grids = [None] + list(range(1, min(host_units(B, M, K, N), ex.sm_count()) + 1))
    bad = torch.zeros(len(grids), dtype=torch.int64, device=ex.DEV)
    raised = torch.zeros(len(grids), dtype=torch.int64, device=ex.DEV)
    for i, G in enumerate(grids):
        set_ctas(G or 0)
        y = ops.fp8_rowwise_bmm(case.xq, case.rs, w, case.sw)
        bad[i] = (y.view(torch.int16) != case.ref.view(torch.int16)).sum()
        raised[i] = flags.ne(0).sum()
        y.view(torch.int16).fill_(ex.POISON_BF16)
    set_ctas(0)
    wrong = [(G, b, r) for G, b, r in zip(grids, bad.cpu().tolist(), raised.cpu().tolist()) if b or r]
    assert not wrong, (f"{layout} B={B} M={M} K={K} N={N}: (grid, wrong elements, raised flags) {wrong[:5]}; "
                       f"{len(wrong)} of {len(grids)} launches wrong")


# ------------------------------------------------------------------------------------------------ random operands
def _random_operands(ops, B, M, K, N, seed):
    g = ex.gen(seed)
    x = torch.randn(B * M, K, device=ex.DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(B * N, K, device=ex.DEV, generator=g) * 0.05).to(torch.bfloat16)
    xq, sx = ops.fp8_quantize_rowwise(x)
    wq, sw = ops.fp8_quantize_rowwise(w)
    return x.reshape(B, M, K), xq.reshape(B, M, K), sx.reshape(-1), w.reshape(B, N, K), wq.reshape(B, N, K), sw.reshape(B, N)


@pytest.mark.parametrize("B,M,K,N", [(4, 1, 1024, 512), (3, 33, 2048, 784), (2, 128, 5120, 1024), (1, 200, 768, 256)])
def test_random_operands_layouts_agree(ops, set_ctas, B, M, K, N):
    """Same codes in both layouts: the same bits at every grid.  Against the fp64 product of the codes > 45 dB and the
    dense fp8 GEMM run batch by batch > 70 dB (the bars of test_grouped_mm_gpu.py: the e4m3 wgmma adds each chunk in
    the tensor core's reduced-precision accumulator), against bf16 torch.bmm > 20 dB (the reference's bar)."""
    x, xq, sx, w, wq, sw = _random_operands(ops, B, M, K, N, seed=B * M + K + N)
    ref64 = torch.bmm(xq.double(), wq.double().transpose(-2, -1)) * sx.double().reshape(B, M, 1) * sw.double()[:, None, :]
    dense = torch.stack([ops.fp8_rowwise_linear(xq[b], sx.reshape(B, M)[b], wq[b], sw[b], None) for b in range(B)])
    for G in (None, 1, 7, 64):
        set_ctas(G or 0)
        y_kn = ops.fp8_rowwise_bmm(xq, sx, as_layout(wq, "kn"), sw)
        y_nk = ops.fp8_rowwise_bmm(xq, sx, as_layout(wq, "nk"), sw)
        assert torch.equal(y_kn.view(torch.int16), y_nk.view(torch.int16)), f"grid {G}: the layouts differ"
        assert sqnr(ref64, y_kn) > 45.0, G
        assert sqnr(dense, y_kn) > 70.0, G
    set_ctas(0)
    assert sqnr(torch.bmm(x, w.transpose(-2, -1)), y_kn) > 20.0


# ------------------------------------------------------------------------------------------------ the reference's tests
class BmmModel(torch.nn.Module):
    def __init__(self, weight, transpose):
        super().__init__()
        self.weight = torch.nn.Parameter(weight, requires_grad=False)
        self.transpose = transpose

    def forward(self, x):
        return torch.bmm(x, self.weight.transpose(-2, -1) if self.transpose else self.weight)


@torch.no_grad()
def test_bmm():
    """The reference's test_bmm: torch.bmm(x, w.transpose(-2, -1)) with w [B, N, K] quantized PerRow()."""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8Tensor, PerRow, quantize_

    torch.manual_seed(0)
    B, M, K, N = 10, 32, 128, 256
    x = torch.randn(B, M, K, dtype=torch.bfloat16, device="cuda")
    m = BmmModel(torch.randn(B, N, K, dtype=torch.bfloat16, device="cuda"), transpose=True).eval()
    original = m(x)
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()), filter_fn=lambda *_: True)
    assert isinstance(m.weight, Float8Tensor)
    y = m(x)
    assert y.shape == (B, M, N) and y.dtype == torch.bfloat16
    assert sqnr(original, y) > 20


@torch.no_grad()
def test_bmm_weight_in_bkn_layout():
    """The reference's test_bmm_weight_in_bkn_layout: torch.bmm(x, w) with w [B, K, N] quantized [PerRow(), PerRow(1)]."""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow, quantize_

    torch.manual_seed(0)
    B, M, K, N = 10, 32, 128, 256
    x = torch.randn(B, M, K, dtype=torch.bfloat16, device="cuda")
    m = BmmModel(torch.randn(B, K, N, dtype=torch.bfloat16, device="cuda"), transpose=False).eval()
    original = m(x)
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=[PerRow(), PerRow(1)]),
              filter_fn=lambda *_: True)
    assert m.weight.scale.shape == (B, 1, N), m.weight.scale.shape
    y = m(x)
    assert sqnr(original, y) > 20


class LlamaExperts(torch.nn.Module):
    """llama-models' MoE experts (the reference's model_architectures.py): w1 / w3 [E, D, F] and w2 [E, F, D] in their
    native [E, K, N] layout, x [E, tokens, D]."""

    def __init__(self, E, D, F_, device="cuda"):
        super().__init__()
        g = torch.Generator(device=device).manual_seed(E + D + F_)
        for name, shape in (("w1", (E, D, F_)), ("w2", (E, F_, D)), ("w3", (E, D, F_))):
            w = (torch.randn(shape, device=device, generator=g) * D ** -0.5).to(torch.bfloat16)
            setattr(self, name, torch.nn.Parameter(w, requires_grad=False))

    def forward(self, x):
        h = F.silu(torch.bmm(x, self.w1)) * torch.bmm(x, self.w3)
        return torch.bmm(h, self.w2)


def _quantized_experts(E, D, F_):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, FqnToConfig, PerRow, quantize_

    ref = LlamaExperts(E, D, F_)
    m = copy.deepcopy(ref)
    cfg = Float8DynamicActivationFloat8WeightConfig(granularity=[PerRow(), PerRow(1)])
    quantize_(m, FqnToConfig({"w1": cfg, "w2": cfg, "w3": cfg}), filter_fn=None)
    return ref, m


@torch.no_grad()
def test_llama_expert_block_equals_the_block_run_per_batch(set_ctas):
    """One grid for both runs (a single CTA sums each tile's K in order), so batch b's rows of the batched block equal
    the same block on batch b alone, bit for bit."""
    E, D, F_, T = 4, 512, 768, 24
    ref, m = _quantized_experts(E, D, F_)
    assert m.w1.qdata.is_contiguous() and m.w1.scale.shape == (E, 1, F_)
    x = torch.randn(E, T, D, device="cuda", dtype=torch.bfloat16)
    set_ctas(1)
    y = m(x)
    for b in range(E):
        one = torch.bmm(F.silu(torch.bmm(x[b:b + 1], m.w1[b:b + 1])) * torch.bmm(x[b:b + 1], m.w3[b:b + 1]),
                        m.w2[b:b + 1])
        assert torch.equal(y[b:b + 1].view(torch.int16), one.view(torch.int16)), b
    set_ctas(0)
    assert sqnr(ref(x), m(x)) > 20


@pytest.mark.parametrize("M", [1, 8, 128])
@torch.no_grad()
def test_llama4_scout_expert_shapes(ops, M):
    """Llama-4-Scout experts (D = 5120, F = 8192) with B = 2: w1 [2, 5120, 8192] and w2 [2, 8192, 5120]."""
    for K, N in ((5120, 8192), (8192, 5120)):
        x, xq, sx, w, wq, sw = _random_operands(ops, 2, M, K, N, seed=M + K)
        y_kn = ops.fp8_rowwise_bmm(xq, sx, as_layout(wq, "kn"), sw)
        y_nk = ops.fp8_rowwise_bmm(xq, sx, as_layout(wq, "nk"), sw)
        assert torch.equal(y_kn.view(torch.int16), y_nk.view(torch.int16)), (M, K, N)
        ref64 = torch.bmm(xq.double(), wq.double().transpose(-2, -1)) * sx.double().reshape(2, M, 1) * sw.double()[:, None, :]
        assert sqnr(ref64, y_kn) > 45.0, (M, K, N)


# ------------------------------------------------------------------------------------------------ integration
@torch.no_grad()
def test_cuda_graph_replay():
    _, m = _quantized_experts(2, 256, 512)
    x = torch.randn(2, 16, 256, device="cuda", dtype=torch.bfloat16)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(x)   # warm-up on the capture stream: creates its workspace outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        y = m(x)
    for seed in range(3):
        x.copy_(torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)))
        g.replay()
        want = m(x)
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), seed


@pytest.mark.parametrize("transpose", [False, True], ids=["bkn", "bnk"])
@torch.no_grad()
def test_torch_compile_fullgraph(transpose):
    """One bmm per layout: the compiled graph runs the same ops and gives the eager bits.  (Not the whole expert block:
    inductor fuses silu(a) * b in fp32 with one rounding where eager rounds silu(a) to bf16 first.)"""
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow, quantize_

    shape = (2, 512, 256) if transpose else (2, 256, 512)
    m = BmmModel(torch.randn(shape, dtype=torch.bfloat16, device="cuda"), transpose=transpose)
    gran = PerRow() if transpose else [PerRow(), PerRow(1)]
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=gran), filter_fn=lambda *_: True)
    x = torch.randn(2, 9, 256, device="cuda", dtype=torch.bfloat16)
    want = m(x)
    got = torch.compile(m, fullgraph=True)(x)
    assert got.shape == (2, 9, 512)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@torch.no_grad()
def test_launch_count_of_one_forward(ops):
    """Per bmm: the rowwise quantizer, the row ends and the GEMM."""
    _, m = _quantized_experts(2, 256, 512)
    x = torch.randn(2, 9, 256, device="cuda", dtype=torch.bfloat16)
    m(x)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    m(x)
    assert ops.launch_count() - n0 == 3 * 3


def _lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.ao_fp8_quantize_rowwise.argtypes = [vp, i32, i32, vp, vp, vp]
    lib.ao_fp8_rowwise_bmm.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i32, vp, vp, sz, vp]
    return lib


def test_pdl_chain_equals_serialized():
    """An upstream kernel writes x, then quantize -> [B, K, N] bmm (B = 4) -> quantize -> [B, N, K] bmm (B = 2, other
    row ends in the same workspace), parked behind a long kernel: bit for bit the same launches run one at a time, and
    as a graph."""
    lib = _lib()
    head = Head(lib)
    g = ex.gen(41)
    K, N1, N2 = 1024, 512, 256
    x0 = torch.randn(300, K, device=ex.DEV, generator=g).to(torch.bfloat16)
    w1 = torch.randn(4, K, N1, device=ex.DEV, generator=g).to(E4M3)                    # stored [B, K, N]
    w2 = torch.randn(2, N2, N1, device=ex.DEV, generator=g).to(E4M3)                   # stored [B, N, K]
    s1 = torch.rand(4, N1, device=ex.DEV, generator=g) * 0.01 + 0.001
    s2 = torch.rand(2, N2, device=ex.DEV, generator=g) * 0.01 + 0.001
    buf = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=ex.DEV)
    c = Chain(lib, "upstream x -> quantize -> bmm [B, K, N] -> quantize -> bmm [B, N, K]")
    x = c.out((300, K), torch.bfloat16)
    q1, a1 = c.out((300, K), torch.uint8), c.out((300,), torch.float32)
    y1 = c.out((300, N1), torch.bfloat16)
    q2, a2 = c.out((300, N1), torch.uint8), c.out((300,), torch.float32)
    y2 = c.out((300, N2), torch.bfloat16)
    c.torch(lambda: torch.mul(x0, 3.0, out=x))
    c.call("ao_fp8_quantize_rowwise", x, 300, K, q1, a1)
    c.call("ao_fp8_rowwise_bmm", q1, a1, 4, 75, K, w1, s1, N1, 1, y1, buf, buf.numel())
    c.call("ao_fp8_quantize_rowwise", y1, 300, N1, q2, a2)
    c.call("ao_fp8_rowwise_bmm", q2, a2, 2, 150, N1, w2, s2, N2, 0, y2, buf, buf.numel())
    want = c.result(sync_each=True)
    assert bool(torch.isfinite(want[-1].float()).all())
    got = c.result(head=head)
    for i, (p, q) in enumerate(zip(got, want)):
        assert torch.equal(p.view(torch.uint8), q.view(torch.uint8)), f"{c.name}: output {i} differs (eager)"
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        c.run(head=head)
    for t in c.outs:
        t.view(torch.uint8).fill_(0xFF)
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    for i, (p, q) in enumerate(zip(c.outs, want)):
        assert torch.equal(p.view(torch.uint8), q.view(torch.uint8)), f"{c.name}: output {i} differs (graph replay)"
