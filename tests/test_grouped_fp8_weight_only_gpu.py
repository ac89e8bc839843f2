"""torch._grouped_mm on 3-D weight-only e4m3 expert weights (torch.ops.ao_b200.fp8_weight_grouped_mm and the
Float8Tensor handler) on the GPU:

* the GEMM bit for bit on exact operands against an fp64 restatement under every forced stream-K grid, at every token
  tile (16 / 32 / 64 / 128), with N and K tails, empty experts, malformed (clamped) offs, all experts empty, and rows
  past the last expert left untouched; per-row scales carry a power of two of their expert's own, so a wrong expert
  offset in the scale map cannot pass;
* a NaN weight row in the part of a tile past N (the next expert's rows) never reaches a stored output;
* the handler through torch._grouped_mm and F.grouped_mm: equal to select + F.linear bit for bit on exact operands,
  within the accumulation-order bound of the recipe on random ones, the reference's fixture (PerRow and PerTensor)
  and the reference's own test case (quantize_ with filter_fn and FqnToConfig, SQNR > 25 dB against bf16);
* CUDA-graph replay on new routings, a PDL chain against a serialized run, torch.compile fullgraph, opcheck, and
  torch.save / torch.load of a 3-D weight-only model followed by a grouped forward.

Exact operands: codes c/8 (|c| <= 7) are e4m3 values, row scales odd * 2^p (odd in 3, 5, 7) make every dequantized
weight c * odd * 2^(p-3) exact in bf16, and activations -8..8 times 2^-3: every product of one output is a multiple
of 2^(p-6), at most 392 of them, and K products stay below 2^24 such quanta, so fp32 sums exactly in any order.
"""
import copy
import ctypes
import io
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import exact_operands as ex
import grouped_model as gm
import grouped_nvfp4_model as gnm
from test_float8_weight_only_host import f32
from test_grouped_int4_gpu import Chain, Head

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda"
E4M3 = torch.float8_e4m3fn

# (rows per expert, N, K, rows past the last expert, forced grids; None = every grid up to the bound)
GROUPED_CASES = [
    ([13], 128, 1024, 0, None),                                              # E = 1, N_MMA 16
    ([7, 9, 0, 12], 200, 1040, 3, None),                                     # N and K tails, empty expert, N_MMA 32
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 2048, 2, (1, 2, 3, 5, 8, 13, 21, 34, 64, 132)),   # E = 8, N_MMA 64
    ([150, 0, 70, 1], 264, 1024, 0, (1, 2, 3, 5, 8, 13, 21, 34)),            # N_MMA 128, two m-blocks, N tail
    ([20, 30], 640, 2048, 0, (3, 6, 7, 11)),                                 # five n-tiles: CONTRIB, FULL and OWNER
    ([1, 0, 2, 1, 0, 0, 3, 1] * 16, 136, 1024, 5, (1, 7, 50, 132)),          # E = 128, N tail 136, N_MMA 128
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 0, (1, 2, 5, 16, 64)),           # E = 64, one expert with every row
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
    p = gnm.plan(gm_offs(case_rows), M, N, K, grid=1, sm=sm, fmt="fp8wo")
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def exact_experts(E, N, K, gen):
    """Exact e4m3 expert weights: codes c/8, row scales odd * 2^p with p = -(4 + e % 24) for expert e (distinct per
    expert up to 24 experts).  Returns (w~ fp64 [E, N, K], qdata e4m3 [E, N, K], scale fp32 [E, N])."""
    codes = ex.randint(-7, 7, (E, N, K), gen).double() * 2.0**-3
    p = -(4 + torch.arange(E, device=DEV) % 24)
    s = (ex.pick([3, 5, 7], (E, N), gen) * ex.pow2(p)[:, None]).float()
    q = codes.to(E4M3)
    assert torch.equal(q.double(), codes)
    wt = (q.float() * s[..., None]).to(torch.bfloat16)   # the reference's dequantize
    assert torch.equal(wt.double(), codes * s.double()[..., None]), "premise: c * s exact in bf16"
    assert K * 7 * 7 * 8 < 2**24, "premise: K products stay below 2^24 quanta"
    return wt.double(), q, s


class GroupedCase:
    """Exact operands (exact_experts) and activations -8..8 times 2^-3: the output must equal the fp64 reference
    rounded once to bf16.  Weight rows past N belong to the next expert: a tail tile computes them, never stores them."""

    def __init__(self, offs, M, N, K, seed):
        E = len(offs)
        gen = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E)
        W, self.wq, self.scale = exact_experts(E, N, K, gen)
        X = ex.randint(-8, 8, (M, K), gen).double() * 2.0**-3
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                ref[start:end] = X[start:end] @ W[e].t()
            start = end
        ex.fp32_exact(ref, "grouped fp8 weight-only: acc")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.x = X.to(torch.bfloat16)
        self.offs = torch.tensor(offs, dtype=torch.int32, device=DEV)
        self.M, self.N, self.K, self.E = M, N, K, E

    def run(self):
        return torch.ops.ao_b200.fp8_weight_grouped_mm(self.x, self.wq, self.scale, self.offs)


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
    flags = ops.debug_workspace(case.x).view(torch.int32)[:4096]
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
        p = gnm.plan(case.offs.tolist(), case.M, case.N, case.K, grid=G, sm=ex.sm_count(), fmt="fp8wo")
        pytest.fail(f"{what} M={case.M} N={case.N} K={case.K} E={case.E} grid={G or 'default'}: {nb} wrong elements, "
                    f"{nr} flags left raised (U={p.U}, width {p.width}, device grid {p.G} of {p.G_host}); "
                    f"{len(wrong)} of {len(grids)} launches wrong")


@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, ci):
    rows, N, K, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(gm_offs(rows), sum(rows) + tail, N, K, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(rows, N, K, tail, grids, ex.sm_count()), f"case {ci}")


@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(offs, M, 200, 1040, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


def test_all_experts_empty(ops, set_ctas):
    case = GroupedCase([0, 0, 0], 20, 256, 1024, seed=7)
    flags = ops.debug_workspace(case.x).view(torch.int32)[:4096]
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
    lib.ao_fp8_weight_grouped_mm.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, ctypes.c_size_t, vp]
    lib.ao_fp8_quantize_rowwise.argtypes = [vp, i32, i32, vp, vp, vp]
    return lib


def _call(lib, x, M, K, wq, scale, E, N, offs, y, ws):
    rc = lib.ao_fp8_weight_grouped_mm(x.data_ptr(), M, K, wq.data_ptr(), scale.data_ptr(), E, N, offs.data_ptr(),
                                      y.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.ao_b200_last_error()


def test_rows_past_the_last_expert_are_not_written():
    """Through the C ABI into a poisoned y: the rows from offs[-1] on keep their bytes, the rest is the reference."""
    lib = _lib()
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    for offs, M in (([5, 5, 20], 37), ([3, 40, 90], 130)):
        case = GroupedCase(offs, M, 200, 1040, seed=3)
        y = torch.full((case.M, case.N), ex.POISON_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        _call(lib, case.x, case.M, case.K, case.wq, case.scale, case.E, case.N, case.offs, y, ws)
        torch.cuda.synchronize()
        assert torch.equal(y[: case.valid].view(torch.int16), case.ref.view(torch.int16))
        assert bool((y[case.valid:].view(torch.int16) == ex.POISON_BF16).all())


def test_nan_rows_past_n_do_not_reach_stored_outputs(ops, set_ctas):
    """N = 200: the second n-tile of expert e covers its rows 128..199 and expert e+1's rows 0..55, which are all-zero
    weight rows (scale 0, NaN codes, as the quantizer leaves them).  Expert e's outputs stay finite and exact; the
    NaN rows of expert e+1 appear only in expert e+1's own outputs."""
    E, N, K = 3, 200, 1024
    rows = [20, 33, 70]
    case = GroupedCase(gm_offs(rows), sum(rows), N, K, seed=11)
    nan_rows = torch.arange(0, 56, device=DEV)
    for e in (1, 2):
        case.wq.view(torch.uint8)[e, nan_rows] = 0x7F
        case.scale[e, nan_rows] = 0.0
    for G in (0, 1, 4, 17):
        set_ctas(G)
        y = case.run()
        torch.cuda.synchronize()
        assert torch.equal(y[:20].view(torch.int16), case.ref[:20].view(torch.int16)), f"grid {G}"
        for e, (r0, r1) in ((1, (20, 53)), (2, (53, 123))):
            assert bool(torch.isnan(y[r0:r1, :56].float()).all()), (G, e)
            assert torch.equal(y[r0:r1, 56:].view(torch.int16), case.ref[r0:r1, 56:].view(torch.int16)), (G, e)


# ------------------------------------------------------------------------------------------------ handler
def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    dd = (ref - out).norm()
    return float("inf") if dd == 0 else float(20 * torch.log10(ref.norm() / dd))


class GroupedMMModel(nn.Module):
    def __init__(self, E, K, N):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16))

    def forward(self, x, offs, functional=False):
        fn = F.grouped_mm if functional else torch._grouped_mm
        return fn(x, self.weight.transpose(-2, -1), offs=offs)


def _quantized(model, gran=None, fqn=True):
    from ao_b200.quantization import Float8WeightOnlyConfig, FqnToConfig, quantize_

    m = copy.deepcopy(model)
    cfg = Float8WeightOnlyConfig() if gran is None else Float8WeightOnlyConfig(granularity=gran)
    if fqn:
        quantize_(m, FqnToConfig({"weight": cfg}), filter_fn=None)
    else:
        quantize_(m, cfg, filter_fn=lambda mod, name: isinstance(mod, GroupedMMModel))
    return m


@torch.no_grad()
@pytest.mark.parametrize("functional", [False, True])
def test_handler_exact_equals_select_and_linear(functional):
    from ao_b200.quantization import Float8Tensor

    gen = ex.gen(5)
    E, N, K = 6, 1000, 2064
    rows = [3, 17, 0, 40, 1, 9]
    W, q, s = exact_experts(E, N, K, gen)
    w = Float8Tensor(q, s[..., None], [1, 1, K], dtype=torch.bfloat16)
    X = ex.randint(-8, 8, (sum(rows), K), gen).double() * 2.0**-3
    x = X.to(torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device=DEV)
    fn = F.grouped_mm if functional else torch._grouped_mm
    y = fn(x, w.transpose(-2, -1), offs=offs)
    assert y.shape == (sum(rows), N) and y.dtype == torch.bfloat16
    start = 0
    for e, end in enumerate(gm_offs(rows)):
        if end > start:
            ref = (X[start:end] @ W[e].t()).float().to(torch.bfloat16)
            assert torch.equal(y[start:end].view(torch.int16), ref.view(torch.int16)), f"expert {e}: fp64 reference"
            d = F.linear(x[start:end], w[e])
            assert torch.equal(d.view(torch.int16), y[start:end].view(torch.int16)), f"expert {e}: select + linear"
        start = end


@torch.no_grad()
def test_handler_random_within_the_sum_bound_of_the_recipe():
    from ao_b200.quantization import PerRow, PerTensor
    from test_grouped_fp8_weight_only_host import per_expert_within_the_sum_bound

    torch.manual_seed(3)
    E, K, N = 8, 1536, 1000
    rows = [5, 0, 40, 1, 130, 0, 16, 9]
    ref = GroupedMMModel(E, K, N)
    x = torch.randn(sum(rows), K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), device=DEV, dtype=torch.int32)
    for gran in (PerRow(), PerTensor()):
        m = _quantized(ref, gran)
        w = m.weight
        for functional in (False, True):
            y = m(x, offs, functional)
            y_dq = torch._grouped_mm(x, w.dequantize().transpose(-2, -1), offs=offs)   # the reference's recipe
            q = w.qdata.view(torch.uint8).cpu().numpy()
            sc = w.scale.float().cpu().numpy()
            u16 = lambda t: t.view(torch.int16).cpu().numpy().view(np.uint16)   # noqa: E731
            assert per_expert_within_the_sum_bound(u16(y), u16(y_dq), x.float().cpu().numpy(), q, sc, gm_offs(rows)), gran
            assert sqnr(ref(x, offs), y) > 25.0


def test_golden_fixture():
    """The reference's CPU outputs: one-hot inputs bit for bit, random ones within the accumulation-order bound,
    through torch._grouped_mm and, for PerRow, select + F.linear; the quantized tensor equals the fixture's."""
    from ao_b200.quantization import Float8Tensor, PerRow, PerTensor
    from test_float8_weight_only_host import same_codes
    from test_grouped_fp8_weight_only_host import golden_shapes, per_expert_within_the_sum_bound

    d = np.load(os.path.join(HERE, "golden", "float8_weight_only_3d.npz"))
    b16 = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).to(DEV)   # noqa: E731
    u16 = lambda t: t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)   # noqa: E731
    for c, a in golden_shapes(d):
        w = b16(a["w"])
        offs = torch.from_numpy(a["offs"]).to(DEV)
        end = int(a["offs"][-1])
        for g, gran in (("PerRow", PerRow()), ("PerTensor", PerTensor())):
            t = Float8Tensor.from_hp(w, E4M3, gran)
            assert same_codes(t.qdata.view(torch.uint8).cpu().numpy(), a[f"{g}_q"]), (c, g)
            assert np.array_equal(t.scale.cpu().numpy(), a[f"{g}_scale"]), (c, g)
            with torch.no_grad():
                for fn in (torch._grouped_mm, F.grouped_mm):
                    ye = u16(fn(b16(a["xe"]), t.transpose(-2, -1), offs=offs)[:end])
                    y = u16(fn(b16(a["x"]), t.transpose(-2, -1), offs=offs)[:end])
                    nan_g, nan_w = np.isnan(f32(ye)), np.isnan(f32(a[f"{g}_ye"]))
                    zero = (f32(ye) == 0) & (f32(a[f"{g}_ye"]) == 0)
                    assert np.array_equal(nan_g, nan_w) and ((ye == a[f"{g}_ye"]) | nan_g | zero).all(), (c, g)
                    assert per_expert_within_the_sum_bound(y, a[f"{g}_y"], f32(a["x"]), a[f"{g}_q"], a[f"{g}_scale"],
                                                           a["offs"]), (c, g)
                if g == "PerRow":
                    start = 0
                    for e, o in enumerate(a["offs"]):
                        lin = u16(F.linear(b16(a["xe"])[start:o], t[e]))
                        assert np.array_equal(np.isnan(f32(lin)), np.isnan(f32(a["PerRow_ye_linear"][start:o])))
                        ok = ~np.isnan(f32(lin)) & (f32(lin) != 0)
                        assert (lin[ok] == a["PerRow_ye_linear"][start:o][ok]).all(), (c, e)
                        start = o


@torch.no_grad()
@pytest.mark.parametrize("fqn", [False, True])
def test_reference_grouped_mm_weight_only_case(fqn):
    """The reference's test_fp8_grouped_mm_weight_only: E, K, N = 4, 128, 256, rows [32, 64, 16, 48], quantize_ with
    Float8WeightOnlyConfig(granularity=PerRow()), output SQNR > 25 dB against the bf16 model."""
    from ao_b200.quantization import Float8Tensor, PerRow

    torch.manual_seed(0)
    E, K, N = 4, 128, 256
    ref = GroupedMMModel(E, K, N)
    m = _quantized(ref, PerRow(), fqn=fqn)
    assert isinstance(m.weight, Float8Tensor) and m.weight.act_quant_kwargs is None
    x = torch.randn(160, K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs([32, 64, 16, 48]), dtype=torch.int32, device=DEV)
    n0 = torch.ops.ao_b200.launch_count()
    y = m(x, offs)
    assert torch.ops.ao_b200.launch_count() - n0 == 1   # one kernel: no activation prologue
    assert y.shape == (160, N) and y.dtype == torch.bfloat16
    assert sqnr(ref(x, offs), y) > 25.0


# ------------------------------------------------------------------------------------------------ graph and compile
@torch.no_grad()
def test_cuda_graph_replay_with_new_routing():
    """Capture the quantized expert forward, then write new routings into the static offs and x: the replay must
    equal eager bit for bit, so the host never read offs."""
    E, K, N, M = 8, 2048, 1000, 48
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
    m = _quantized(GroupedMMModel(4, 1024, 520))
    x = torch.randn(20, 1024, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([3, 3, 12, 20], dtype=torch.int32, device=DEV)
    y = m(x, offs)
    yc = torch.compile(m, fullgraph=True, backend=backend)(x, offs)
    assert torch.equal(y[:20].view(torch.int16), yc[:20].view(torch.int16))


def test_opcheck():
    _, q, s = exact_experts(3, 136, 1024, ex.gen(9))
    x = torch.randn(10, 1024, device=DEV).to(torch.bfloat16)
    offs = torch.tensor([2, 5, 10], dtype=torch.int32, device=DEV)
    # test_schema is left out: it multiplies the inputs, and torch has no mul for float8_e4m3fn
    torch.library.opcheck(torch.ops.ao_b200.fp8_weight_grouped_mm.default, (x, q, s, offs),
                          test_utils=("test_faketensor", "test_autograd_registration"))


@torch.no_grad()
def test_save_load_then_grouped_forward():
    from ao_b200.quantization import Float8Tensor, PerTensor

    torch.manual_seed(6)
    base = GroupedMMModel(4, 512, 296)
    x = torch.randn(40, 512, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([10, 10, 25, 40], dtype=torch.int32, device=DEV)
    for gran in (None, PerTensor()):
        m = _quantized(base, gran)
        buf = io.BytesIO()
        torch.save(m.state_dict(), buf)
        buf.seek(0)
        m2 = GroupedMMModel(4, 512, 296)
        m2.load_state_dict(torch.load(buf, weights_only=True), assign=True)
        assert type(m2.weight) is Float8Tensor and m2.weight.act_quant_kwargs is None
        assert torch.equal(m2(x, offs).view(torch.int16), m(x, offs).view(torch.int16))


# ------------------------------------------------------------------------------------------------ PDL handoffs
def test_pdl_overlapped_equals_serialized():
    """offs from a torch cumsum, then grouped gate/up -> torch SiLU-mul -> grouped down, parked behind a long kernel
    (tests/test_pdl_handoffs_gpu.py's stall head), against the same launches run one at a time, and as a graph."""
    lib = _lib()
    head = Head(lib)
    M, E, H, I = 300, 4, 2048, 1024
    _, qg, sg = exact_experts(E, 2 * I, H, ex.gen(32))
    _, qd, sd = exact_experts(E, H, I, ex.gen(33))
    x = (torch.randn(M, H, device=DEV) * 0.25).to(torch.bfloat16)
    counts = torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    ws2 = torch.zeros_like(ws)
    c = Chain(lib, "cumsum offs -> grouped gate/up -> silu-mul -> grouped down")
    offs = c.out((E,), torch.int32)
    h = c.out((M, 2 * I), torch.bfloat16)
    a = c.out((M, I), torch.bfloat16)
    y = c.out((M, H), torch.bfloat16)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    c.call("ao_fp8_weight_grouped_mm", x, M, H, qg, sg, E, 2 * I, offs, h, ws, ws.numel())
    c.torch(lambda: torch.mul(F.silu(h[:, :I]), h[:, I:], out=a))
    c.call("ao_fp8_weight_grouped_mm", a, M, I, qd, sd, E, H, offs, y, ws2, ws2.numel())
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
