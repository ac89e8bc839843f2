"""torch._grouped_mm on 3-D blockwise e4m3 expert weights (torch.ops.ao_b200.fp8_blockwise_grouped_mm and the
Float8Tensor handler) on the GPU:

* the GEMM bit for bit on exact operands against an fp64 restatement of the per-expert recipe (select, then the dense
  blockwise loop) under every forced stream-K grid up to the host bound and the default one: the grouped cases of
  test_grouped_mm_gpu.py with N a multiple of 128, E = 256, experts of several 64-token blocks, clamped malformed offs;
  the workspace flags are back to zero after each launch and rows past offs[-1] keep their poison;
* random operands: bit-identical to fp8_blockwise_linear run expert by expert when one CTA computes every tile of both
  launches, and within the dense op's fp64 bound at the default grid;
* the handler through torch._grouped_mm and F.grouped_mm against select + F.linear per expert;
* CUDA-graph replay on new routings, torch.compile fullgraph, opcheck, save / load, a PDL chain against a serialized
  run, misaligned activation views and the launch count.

Exact operands: the scheme of test_fp8_blockwise_gpu.py::Exact per expert.  Codes in -2..2, token scales 2^[-2, 1] and
weight block scales 2^[-1, 1] divided by 2^(e % 3), so a wrong expert's scale block cannot pass: each chunk's wgmma sum
is an integer below 2^9, its scaled value a multiple of 2^-5 below 2^11 (2^16 quanta), and K <= 16384 (128 chunks)
keeps the sum below 2^24 quanta, exact in fp32 in any order and under any stream-K split (fp32_exact asserts it).
"""
import copy
import ctypes
import io
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import exact_operands as ex
import grouped_model as gm
from test_grouped_int4_gpu import Chain, Head

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
E4M3 = torch.float8_e4m3fn

# (rows per expert, N, K, rows past the last expert, forced grids; None = every grid up to the host bound):
# test_grouped_mm_gpu.py's cases with N a multiple of 128, and E = 256 with top-8-like routing
GROUPED_CASES = [
    ([13], 256, 1024, 0, None),                                   # E = 1, N_MMA 16
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 1024, 2, None),              # E = 8, empty experts, rows past offs[-1]
    ([150, 0, 70, 1], 256, 512, 0, None),                         # experts of three and two 64-token blocks
    ([7, 9, 0, 12], 128, 512, 3, None),                           # N_MMA 32, one n-tile
    ([20, 30], 640, 1024, 0, (3, 6, 7, 11)),                      # five n-tiles: CONTRIB, FULL and OWNER in one CTA
    ([1, 0, 2, 1, 0, 0, 3, 1] * 8, 128, 256, 5, None),            # E = 64
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 0, (1, 2, 5, 16, 64)),  # E = 64, one expert with every row
    ([1, 0, 2, 0, 0, 3, 1, 1] * 32, 256, 512, 3, (1, 2, 7, 50, 131, 132)),   # E = 256
    # K = 16384, one tile split over up to 128 CTAs: owners gather 32 to 127 partials (N_MMA 16, 32 and 64; at 32
    # also 4 and 5, and 25 valid token columns of the 32)
    ([0, 16, 0], 128, 16384, 0, (33, 64, 65, 127, 128)),
    ([0, 25, 0], 128, 16384, 0, (5, 6, 33, 64, 65, 127, 128)),
    ([0, 64, 0], 128, 16384, 0, (33, 64, 65, 127, 128)),
]
# offs values that are not cumulative row ends: the kernel clamps each into [end[e-1], M]
MALFORMED = [([9, 4, -3, 30, 12, 500], 40), ([-5, -1, 0, 3], 8), ([100, 200], 64)]


def gm_offs(rows):
    out, s = [], 0
    for r in rows:
        s += r
        out.append(s)
    return out


def grids_of(case_rows, N, K, tail, grids, sm):
    M = sum(case_rows) + tail
    p = gm.plan(gm_offs(case_rows), M, N, K, grid=1, sm=sm, fmt="fp8_blockwise")
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def transposed_scales(s):
    """[M, K/128] -> the kernel's [K/128, round_up(M, 4)] layout, pads zero."""
    M, KB = s.shape
    out = torch.zeros(KB, (M + 3) // 4 * 4, dtype=torch.float32, device=s.device)
    out[:, :M] = s.t()
    return out


class GroupedCase:
    """Exact operands (see the top of the file): the output rows up to offs[-1] must equal the fp64 per-expert loop
    rounded once to bf16."""

    def __init__(self, offs, M, N, K, seed):
        E, KB = len(offs), K // 128
        g = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E)
        X = ex.randint(-2, 2, (M, K), g).double()
        W = ex.randint(-2, 2, (E, N, K), g).double()
        self.a_s = ex.pow2(ex.randint(-2, 1, (M, KB), g)).float()
        shift = (torch.arange(E, device=DEV) % 3)[:, None, None]
        self.w_s = ex.pow2(ex.randint(-1, 1, (E, N // 128, KB), g) - shift).float()
        self.xq, self.wq = X.to(E4M3), W.to(E4M3)
        self.xs = transposed_scales(self.a_s)
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                for kb in range(KB):
                    ks = slice(kb * 128, (kb + 1) * 128)
                    part = X[start:end, ks] @ W[e, :, ks].t()
                    ref[start:end] += (part * self.a_s[start:end, kb, None].double()
                                       * self.w_s[e, :, kb].double().repeat_interleave(128)[None, :])
            start = end
        ex.fp32_exact(ref, "grouped fp8 blockwise: acc")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.offs = torch.tensor(offs, dtype=torch.int32, device=DEV)
        self.M, self.N, self.K, self.E = M, N, K, E

    def run(self):
        return torch.ops.ao_b200.fp8_blockwise_grouped_mm(self.xq, self.xs, self.wq, self.w_s, self.offs)


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def _sweep(ops, set_ctas, case, grids, what):
    flags = ops.debug_workspace(case.xq).view(torch.int32)[:4096]
    bad = torch.zeros(len(grids), dtype=torch.int64, device=DEV)
    raised = torch.zeros(len(grids), dtype=torch.int64, device=DEV)
    for i, G in enumerate(grids):
        set_ctas(G or 0)
        y = case.run()
        bad[i] = (y[: case.valid].view(torch.int16) != case.ref.view(torch.int16)).sum()
        raised[i] = flags.ne(0).sum()
        y.view(torch.int16).fill_(ex.POISON_BF16)
    set_ctas(0)
    bad, raised = bad.cpu().tolist(), raised.cpu().tolist()
    wrong = [(G, b, r) for G, b, r in zip(grids, bad, raised) if b or r]
    if wrong:
        G, nb, nr = wrong[0]
        p = gm.plan(case.offs.tolist(), case.M, case.N, case.K, grid=G, sm=ex.sm_count(), fmt="fp8_blockwise")
        pytest.fail(f"{what} M={case.M} N={case.N} K={case.K} E={case.E} grid={G or 'default'}: {nb} wrong elements, "
                    f"{nr} flags left raised (U={p.U}, device grid {p.G} of {p.G_host}); "
                    f"{len(wrong)} of {len(grids)} launches wrong")


@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, ci):
    rows, N, K, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(gm_offs(rows), sum(rows) + tail, N, K, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(rows, N, K, tail, grids, ex.sm_count()), f"case {ci}")


@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(offs, M, 256, 512, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


def test_all_experts_empty(ops, set_ctas):
    case = GroupedCase([0, 0, 0], 20, 256, 512, seed=7)
    flags = ops.debug_workspace(case.xq).view(torch.int32)[:4096]
    for G in (0, 5):
        set_ctas(G)
        out = case.run()
        torch.cuda.synchronize()
        assert out.shape == (20, 256) and not bool(flags.ne(0).any())


def _lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    lib.ao_fp8_blockwise_grouped_mm.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, ctypes.c_size_t, vp]
    lib.ao_fp8_quantize_1x128.argtypes = [vp, i32, i32, vp, vp, vp]
    lib.ao_fp8_quantize_rowwise.argtypes = [vp, i32, i32, vp, vp, vp]
    return lib


def test_rows_past_the_last_expert_are_not_written():
    """Through the C ABI into a poisoned y: the rows from offs[-1] on keep their bytes, the rest is the reference."""
    lib = _lib()
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    for offs, M in (([5, 5, 20], 37), ([3, 40, 90], 130)):
        case = GroupedCase(offs, M, 256, 1024, seed=3)
        y = torch.full((case.M, case.N), ex.POISON_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        rc = lib.ao_fp8_blockwise_grouped_mm(case.xq.data_ptr(), case.xs.data_ptr(), case.M, case.K, case.wq.data_ptr(),
                                             case.w_s.data_ptr(), case.E, case.N, case.offs.data_ptr(), y.data_ptr(),
                                             ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, lib.ao_b200_last_error()
        torch.cuda.synchronize()
        assert torch.equal(y[: case.valid].view(torch.int16), case.ref.view(torch.int16))
        assert bool((y[case.valid:].view(torch.int16) == ex.POISON_BF16).all())


# ------------------------------------------------------------------------------------------------ random operands
def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    dd = (ref - out).norm()
    return float("inf") if dd == 0 else float(20 * torch.log10(ref.norm() / dd))


def random_experts(E, N, K, seed):
    from ao_b200.quantization import Float8Tensor, PerBlock

    torch.manual_seed(seed)
    return Float8Tensor.from_hp((torch.randn(E, N, K, device=DEV) * 0.02).to(torch.bfloat16),
                                granularity=PerBlock([128, 128]))


@pytest.mark.parametrize("E,N,K,rows", [(8, 512, 1024, [16, 0, 48, 3, 0, 16, 70, 1]), (4, 4096, 2048, [9] * 4),
                                        (16, 768, 7168, [0, 1, 32, 0, 2, 0, 0, 48, 16, 0, 0, 5, 32, 0, 1, 1])])
def test_random_operands_equal_the_dense_op_per_expert(ops, set_ctas, E, N, K, rows):
    """One CTA computes every tile of both launches (forced grid 1): each tile's chunks are summed in order in one
    segment, so the grouped op equals fp8_blockwise_linear on each expert's own quantized rows bit for bit.  At the
    default grid the stream-K split reorders the fp32 sums: within the dense op's fp64 bound."""
    w = random_experts(E, N, K, seed=E + N + K)
    x = torch.randn(sum(rows), K, device=DEV).to(torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device=DEV)
    xq, xs = ops.fp8_quantize_1x128(x)
    set_ctas(1)
    y1 = ops.fp8_blockwise_grouped_mm(xq, xs, w.qdata, w.scale, offs)
    dense = torch.empty_like(y1)
    acc = torch.empty(sum(rows), N, dtype=torch.float64, device=DEV)
    start = 0
    for e, end in enumerate(gm_offs(rows)):
        if end > start:
            q, s = ops.fp8_quantize_1x128(x[start:end])
            dense[start:end] = ops.fp8_blockwise_linear(q, s, w.qdata[e], w.scale[e], None)
            X, W = q.double(), w.qdata[e].double()
            a_s = s[:, : end - start].t().double()
            acc[start:end] = 0
            for kb in range(K // 128):
                ks = slice(kb * 128, (kb + 1) * 128)
                acc[start:end] += ((X[:, ks] @ W[:, ks].t()) * a_s[:, kb, None]
                                   * w.scale[e, :, kb].double().repeat_interleave(128)[None, :])
        start = end
    set_ctas(0)
    assert torch.equal(y1.view(torch.int16), dense.view(torch.int16))
    y = ops.fp8_blockwise_grouped_mm(xq, xs, w.qdata, w.scale, offs)
    # the dense op's bar against its fp64 sum (test_fp8_blockwise_gpu.py::test_random_operands_within_tolerance)
    assert sqnr(acc, y) > 45.0


# ------------------------------------------------------------------------------------------------ handler
def blockwise_config():
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock

    return Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])])


class GroupedMMModel(nn.Module):
    def __init__(self, E, K, N):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16) * 0.05)

    def forward(self, x, offs, functional=False):
        fn = F.grouped_mm if functional else torch._grouped_mm
        return fn(x, self.weight.transpose(-2, -1), offs=offs)


def _quantized(model):
    from ao_b200.quantization import FqnToConfig, quantize_

    m = copy.deepcopy(model)
    quantize_(m, FqnToConfig({"weight": blockwise_config()}), filter_fn=None)
    return m


@torch.no_grad()
@pytest.mark.parametrize("functional", [False, True])
def test_handler_equals_select_and_linear(set_ctas, functional):
    from ao_b200.quantization import Float8Tensor

    torch.manual_seed(5)
    E, K, N = 6, 2048, 1024
    rows = [3, 17, 0, 70, 1, 9]
    ref = GroupedMMModel(E, K, N)
    m = _quantized(ref)
    w = m.weight
    assert isinstance(w, Float8Tensor) and list(w.block_size) == [1, 128, 128] and w.scale.shape == (E, N // 128, K // 128)
    x = torch.randn(sum(rows) + 4, K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device=DEV)
    end = gm_offs(rows)[-1]
    for G in (1, 0):
        set_ctas(G)
        y = m(x, offs, functional)
        assert y.shape == (x.shape[0], N) and y.dtype == torch.bfloat16
        loop = torch.empty_like(y)
        start = 0
        for e, stop in enumerate(gm_offs(rows)):
            if stop > start:
                loop[start:stop] = F.linear(x[start:stop], w[e])   # the eager loop: select + the dense handler
            start = stop
        if G == 1:   # one CTA per launch: whole tiles in both
            assert torch.equal(y[:end].view(torch.int16), loop[:end].view(torch.int16))
        else:
            assert sqnr(loop[:end], y[:end]) > 45.0
        assert sqnr(ref(x, offs)[:end], y[:end]) > 25.0


@torch.no_grad()
def test_two_launches_per_grouped_call(ops):
    torch.manual_seed(6)
    m = _quantized(GroupedMMModel(8, 1024, 512))
    x = torch.randn(40, 1024, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs([5] * 8), dtype=torch.int32, device=DEV)
    m(x, offs)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    m(x, offs)
    assert ops.launch_count() - n0 == 2   # the 1x128 quantizer and the grouped GEMM


# ------------------------------------------------------------------------------------------------ graph and compile
@torch.no_grad()
def test_cuda_graph_replay_with_new_routing():
    """Capture the quantized expert forward, then write new routings into the static offs and x: the replay must
    equal eager bit for bit, so the host never read offs."""
    E, K, N, M = 8, 2048, 1024, 48
    torch.manual_seed(1)
    m = _quantized(GroupedMMModel(E, K, N))
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs([6] * 8), dtype=torch.int32, device=DEV)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(x, offs)   # warm-up on the capture stream: creates its workspace outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        y = m(x, offs)
    for rows in ([6] * 8, [0, 30, 0, 0, 1, 17, 0, 0], [48, 0, 0, 0, 0, 0, 0, 0], [0] * 7 + [40]):
        x.copy_(torch.randn(M, K, device=DEV, dtype=torch.bfloat16))
        offs.copy_(torch.tensor(gm_offs(rows), dtype=torch.int32))
        g.replay()
        want = m(x, offs)
        torch.cuda.synchronize()
        n = gm_offs(rows)[-1]
        assert torch.equal(y[:n].view(torch.int16), want[:n].view(torch.int16)), f"routing {rows}"


@torch.no_grad()
@pytest.mark.parametrize("backend", ["inductor", "aot_eager"])
def test_compile_fullgraph_through_the_handler(backend):
    torch.manual_seed(2)
    m = _quantized(GroupedMMModel(4, 1024, 640))
    x = torch.randn(20, 1024, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([3, 3, 12, 20], dtype=torch.int32, device=DEV)
    y = m(x, offs)
    yc = torch.compile(m, fullgraph=True, backend=backend)(x, offs)
    assert torch.equal(y[:20].view(torch.int16), yc[:20].view(torch.int16))


def test_opcheck(ops):
    case = GroupedCase([2, 5, 10], 10, 256, 512, seed=9)
    # test_schema is left out: it multiplies the inputs, and torch has no mul for float8_e4m3fn
    torch.library.opcheck(ops.fp8_blockwise_grouped_mm.default, (case.xq, case.xs, case.wq, case.w_s, case.offs),
                          test_utils=("test_faketensor", "test_autograd_registration"))


@torch.no_grad()
def test_save_load_then_grouped_forward():
    from ao_b200.quantization import Float8Tensor

    torch.manual_seed(6)
    base = GroupedMMModel(4, 512, 384)
    x = torch.randn(40, 512, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([10, 10, 25, 40], dtype=torch.int32, device=DEV)
    m = _quantized(base)
    buf = io.BytesIO()
    torch.save(m.state_dict(), buf)
    buf.seek(0)
    m2 = GroupedMMModel(4, 512, 384)
    m2.load_state_dict(torch.load(buf, weights_only=True), assign=True)
    assert type(m2.weight) is Float8Tensor and list(m2.weight.block_size) == [1, 128, 128]
    assert torch.equal(m2(x, offs).view(torch.int16), m(x, offs).view(torch.int16))


# ------------------------------------------------------------------------------------------------ activation layouts
@pytest.mark.parametrize("layout", ["column_slice", "storage_offset"])
def test_misaligned_activation_views_equal_a_contiguous_copy(ops, layout):
    """xq as a column slice of a wider buffer or rows at an odd storage offset, neither on 16 bytes: the bits of the
    same call on a dense, aligned copy."""
    M, K = 37, 1024
    case = GroupedCase([10, 10, 30, 35], M, 256, K, seed=12)
    wide = torch.zeros(M, K + 8, dtype=E4M3, device=DEV)
    x = wide[:, 4:4 + K] if layout == "column_slice" else wide.flatten()[4:4 + M * K].view(M, K)
    x.copy_(case.xq)
    assert x.data_ptr() % 16 != 0
    y = ops.fp8_blockwise_grouped_mm(x, case.xs, case.wq, case.w_s, case.offs)
    assert torch.equal(y[:35].view(torch.int16), case.ref.view(torch.int16))
    xs_view = torch.zeros(case.xs.numel() + 1, device=DEV)[1:].view(case.xs.shape)   # x_scale off 16 bytes as well
    xs_view.copy_(case.xs)
    y = ops.fp8_blockwise_grouped_mm(case.xq, xs_view, case.wq, case.w_s, case.offs)
    assert torch.equal(y[:35].view(torch.int16), case.ref.view(torch.int16))


# ------------------------------------------------------------------------------------------------ PDL handoffs
def test_pdl_overlapped_equals_serialized():
    """offs from a torch cumsum, then quantizer -> grouped gate/up -> torch SiLU-mul -> quantizer -> grouped down,
    parked behind a long kernel (tests/test_pdl_handoffs_gpu.py's stall head), against the same launches run one at a
    time, and as a graph."""
    lib = _lib()
    head = Head(lib)
    M, E, H, I = 300, 4, 2048, 1024
    wg = random_experts(E, 2 * I, H, seed=32)
    wd = random_experts(E, H, I, seed=33)
    x = (torch.randn(M, H, device=DEV) * 0.25).to(torch.bfloat16)
    counts = torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    ws2 = torch.zeros_like(ws)
    c = Chain(lib, "cumsum offs -> quantize -> grouped gate/up -> silu-mul -> quantize -> grouped down")
    offs = c.out((E,), torch.int32)
    xq = c.out((M, H), torch.uint8)
    xs = c.out((H // 128, (M + 3) // 4 * 4), torch.float32)
    h = c.out((M, 2 * I), torch.bfloat16)
    a = c.out((M, I), torch.bfloat16)
    aq = c.out((M, I), torch.uint8)
    as_ = c.out((I // 128, (M + 3) // 4 * 4), torch.float32)
    y = c.out((M, H), torch.bfloat16)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    c.call("ao_fp8_quantize_1x128", x, M, H, xq, xs)
    c.call("ao_fp8_blockwise_grouped_mm", xq, xs, M, H, wg.qdata, wg.scale, E, 2 * I, offs, h, ws, ws.numel())
    c.torch(lambda: torch.mul(F.silu(h[:, :I]), h[:, I:], out=a))
    c.call("ao_fp8_quantize_1x128", a, M, I, aq, as_)
    c.call("ao_fp8_blockwise_grouped_mm", aq, as_, M, I, wd.qdata, wd.scale, E, H, offs, y, ws2, ws2.numel())
    want = c.result(sync_each=True)
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
