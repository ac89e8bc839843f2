"""torch._grouped_mm on MX expert weights (torch.ops.ao_b200.mx{fp8,fp4}_grouped_mm, mx{fp8,fp4}_fakequant and the
MXTensor handler) on the GPU:

* the GEMM bit-exact under every forced stream-K grid, with exact-product operands (bf16 activations, MX weight codes
  times chosen e8m0 bytes): empty experts, experts of one row, of width - 1, width and more rows, E = 1 and E = 64, K
  tails, rows past offs[-1], malformed offs, all experts empty; the workspace flags must be back to zero after each
  launch; owners with fewer contributors than ring stages, exactly as many and more;
* the activation prologue bit for bit against the two-launch composition it replaces (mx*_quantize with blocked
  scales, then the dense linear's dequant_act_kernel, read back from the workspace slab);
* 3-D to_mx byte for byte against the reference's CPU to_mx (tests/golden/mx_3d.npz);
* the handler through quantize_ / FqnToConfig: on exact operands equal to the fp64 result rounded once to bf16 and to
  F.linear(x[rows_e], w[e]) bit for bit; on random operands >= 80 dB against select + the dense MX linear;
* a CUDA graph replayed with new routings written into its static x and offs; a PDL chain against a serialized run.
tests/test_grouped_mx_host.py checks on the CPU that GROUPED_CASES reach every segment kind, token tile and staged
gather layout.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import exact_operands as ex
import grouped_model as gm
import streamk_model as sk
from test_grouped_int4_gpu import Chain, Head

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda"
FMTS = ("mxfp8", "mxfp4")
ELEM = {"mxfp8": torch.float8_e4m3fn, "mxfp4": torch.float4_e2m1fn_x2}
MAXC = {"mxfp8": 448.0, "mxfp4": 6.0}   # max_pos of the element format

# (rows per expert, N, K, rows past the last expert, forced grids; None = every grid up to the host bound)
GROUPED_CASES = [
    ([13], 128, 1024, 0, None),                                   # E = 1, N_MMA 16
    ([7, 9, 0, 12], 128, 1056, 3, None),                          # N_MMA 32, K tail, rows past offs[-1]
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 512, 2, None),               # E = 8, empty experts, N_MMA 64
    ([150, 0, 127, 1, 128], 256, 512, 0, (1, 2, 3, 5, 8, 13, 21, 34)),  # N_MMA 128: width - 1, width, two m-blocks
    ([20, 30], 640, 1024, 0, (3, 6, 7, 11)),                      # five n-tiles: CONTRIB, FULL and OWNER in one CTA
    ([1, 0, 2, 1, 0, 0, 3, 1] * 8, 128, 96, 5, None),             # E = 64, K = 96 (one partial chunk), N_MMA 128
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 0, (1, 2, 5, 16, 64)),  # E = 64, one expert with every row
    ([15, 16, 17], 128, 4096, 0, (1, 3, 9, 40)),                  # width - 1, width, width + 1 at N_MMA 64
]
# offs values that are not cumulative row ends: the kernel clamps each into [end[e-1], M]
MALFORMED = [([9, 4, -3, 30, 12, 500], 40), ([-5, -1, 0, 3], 8), ([100, 200], 64)]


def grids_of(fmt, rows, N, K, tail, grids, sm):
    M = sum(rows) + tail
    p = gm.plan(gm.cumulative(rows), M, N, K, grid=1, sm=sm, fmt=fmt)
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def stacked_blocked(s):
    """[E, N, K/32] scale bytes -> each expert's blocked scales, one after the other."""
    return torch.stack([ex.to_blocked(s[e]) for e in range(s.shape[0])])


def mx_weights(fmt, E, N, K, g, codes=None):
    """Stored qdata, blocked scales and fp64 values of [E, N, K] MX weights: random codes (e4m3 bytes 0x30..0x47 with
    either sign and zeros, or every e2m1 code) times scale bytes 124..127."""
    if codes is None:
        if fmt == "mxfp8":
            codes = ex.randint(0x30, 0x47, (E, N, K), g) | (ex.randint(0, 1, (E, N, K), g) << 7)
            codes[ex.randint(0, 7, (E, N, K), g) == 0] = 0
        else:
            codes = ex.randint(0, 15, (E, N, K), g)
    sb = ex.randint(124, 127, (E, N, K // 32), g)
    scale = ex.pow2(sb - 127).repeat_interleave(32, 2)
    if fmt == "mxfp8":
        W = ex.e4m3_bytes_value(codes) * scale
        wq = codes.to(torch.uint8).view(torch.float8_e4m3fn)
    else:
        W = ex.e2m1_value(codes) * scale
        wq = torch.stack([ex.pack_e2m1(codes[e]) for e in range(E)])
    return wq, stacked_blocked(sb.to(torch.uint8)), W


class GroupedCase:
    """Exact operands: X in {-3..3} / 2 (bf16) and the weights of mx_weights: every product is a multiple of 2^-8 (mxfp8)
    or 2^-5 (mxfp4) and every sum stays below 2^24 of them (exact_operands.premise), so the output must equal the
    fp64 reference rounded once to bf16."""

    def __init__(self, fmt, offs, M, N, K, seed):
        E = len(offs)
        g = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E + (fmt == "mxfp4"))
        X = ex.randint(-3, 3, (M, K), g).double() * 0.5
        self.wq, self.ws, W = mx_weights(fmt, E, N, K, g)
        ex.premise(X, W.reshape(E * N, K))
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                ref[start:end] = X[start:end] @ W[e].t()
            start = end
        ex.fp32_exact(ref, f"grouped {fmt}: the sums")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.x = X.to(torch.bfloat16)
        self.offs = torch.tensor(offs, dtype=torch.int32, device=DEV)
        self.fmt, self.M, self.N, self.K, self.E = fmt, M, N, K, E

    def run(self):
        return getattr(ex.ops(), f"{self.fmt}_grouped_mm")(self.x, self.wq, self.ws, self.offs)


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
        p = gm.plan(case.offs.tolist(), case.M, case.N, case.K, grid=G, sm=ex.sm_count(), fmt=case.fmt)
        pytest.fail(f"{what} {case.fmt} M={case.M} N={case.N} K={case.K} E={case.E} grid={G or 'default'}: {nb} wrong "
                    f"elements, {nr} flags left raised (U={p.U}, width {p.width}, device grid {p.G} of {p.G_host}); "
                    f"{len(wrong)} of {len(grids)} launches wrong")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, fmt, ci):
    rows, N, K, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(fmt, gm.cumulative(rows), sum(rows) + tail, N, K, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(fmt, rows, N, K, tail, grids, ex.sm_count()), f"case {ci} rows={rows}")


# one expert whose rows fill one tile of each staging width, K = 8192: a forced grid of G CTAs gives its owner G - 1
# contributors, so the grids below put owners below, at and above the ring's stage count S
def staging_layouts(fmt):
    out = []
    for width in sk.WIDTHS[fmt]:
        _, _, S, staging = sk.ring(fmt, width, grouped=True)
        if not staging:
            continue
        for rows in sorted({width, width - 1, max(1, width // 2 + 1)}):
            out.append((width, S, rows))
    return out


@pytest.mark.parametrize("fmt", FMTS)
def test_owner_gather_below_at_and_above_the_ring(ops, set_ctas, fmt):
    for width, S, rows in staging_layouts(fmt):
        N, K, M = 128, 8192, rows
        offs = [0, rows, rows]   # the middle expert has every row
        assert sk.n_mma(fmt, M) == width
        gb = sk.group_width(width)
        grids = sorted({2, S, S + 1, S + 2} | {S + 1 + j for j in range(gb + 1)} | {S + 34})
        seen = set()
        for G in grids:
            p = gm.plan(offs, M, N, K, grid=G, sm=ex.sm_count(), fmt=fmt)
            for c in p.contributor_counts():
                seen.add((c > S) - (c < S))
        assert seen == {-1, 0, 1}, (fmt, width, S, seen)
        case = GroupedCase(fmt, offs, M, N, K, seed=width + rows)
        _sweep(ops, set_ctas, case, grids, f"staged gather width {width} S={S} rows {rows}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, fmt, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(fmt, offs, M, 256, 512, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


@pytest.mark.parametrize("fmt", FMTS)
def test_all_experts_empty(ops, set_ctas, fmt):
    case = GroupedCase(fmt, [0, 0, 0], 20, 256, 512, seed=7)
    flags = ops.debug_workspace(case.x).view(torch.int32)[:4096]
    for G in (0, 5):
        set_ctas(G)
        out = case.run()
        torch.cuda.synchronize()
        assert out.shape == (20, 256) and not bool(flags.ne(0).any())


# ------------------------------------------------------------------------------------------------ prologue
def _composition(ops, fmt, x):
    """xhat as the dense MX linear makes it: mx*_quantize(x, blocked scales), then its dequant_act_kernel writes the
    bf16 rows into the workspace slab behind the partial slots (ao_b200/csrc/lowp_linear.cu block_scaled), read back."""
    M, K = x.shape
    q, s = getattr(ops, f"{fmt}_quantize")(x, True)
    kq = K // 2 if fmt == "mxfp4" else K
    wq = torch.zeros(128, kq, dtype=q.dtype, device=DEV)
    wsc = torch.zeros(32, 16 * -(-(K // 32) // 4), dtype=torch.uint8, device=DEV)
    getattr(ops, f"{fmt}_linear")(q, s, wq, wsc, None)
    act_off = (64 * 1024 + ex.sm_count() * 128 * 128 * 4 + (1 << 20) - 1) & ~((1 << 20) - 1)
    ws = ops.debug_workspace(x)
    assert ws.numel() - act_off >= M * K * 2, "one slab holds every row"
    return ws[act_off: act_off + M * K * 2].view(torch.bfloat16).view(M, K).clone()


def _edge_rows(K, g):
    """Rows that reach the ends of the e8m0 range and the special values: all-zero blocks, NaN and inf blocks,
    results that are bf16 subnormals, the largest bf16 (e8m0 247) and the smallest subnormal (e8m0 0)."""
    x = torch.randn(12, K, device=DEV, generator=g)
    x[0, :32] = 0.0
    x[1, 5] = float("nan")
    x[2, 40] = float("inf")
    x[3, 70] = -float("inf")
    x[4] *= 1e-38                              # codes times 2^(e - 127) below the smallest normal
    x[5] *= 2.0**-133                          # bf16 subnormals: scale byte 0
    x[6, :32] = 3.3895e38                      # the largest bf16
    x[6, 32:64] = -3.3895e38
    x[7] *= 1e30
    x[8, ::7] = 0.0
    x[9] = torch.where(x[9] > 0, x[9] * 1e-20, x[9] * 1e20)
    return x.to(torch.bfloat16)


def _check_bits(a, b, what):
    an, bn = torch.isnan(a), torch.isnan(b)
    assert torch.equal(an, bn), f"{what}: NaN positions differ"
    assert torch.equal(a.view(torch.int16)[~an], b.view(torch.int16)[~bn]), f"{what}: bits differ"


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,K", [(1, 32), (37, 96), (300, 1024), (64, 4096)])
def test_fakequant_equals_quantize_then_dequant(ops, fmt, M, K):
    g = ex.gen(M * 7 + K)
    x = (torch.randn(M, K, device=DEV, generator=g) * torch.logspace(-4, 4, M, device=DEV)[:, None]).to(torch.bfloat16)
    xhat = getattr(ops, f"{fmt}_fakequant")(x)
    _check_bits(xhat, _composition(ops, fmt, x), f"{fmt} M={M} K={K}")
    assert not bool(torch.isnan(xhat).any())


@pytest.mark.parametrize("fmt", FMTS)
def test_fakequant_edges_and_strided_rows(ops, fmt):
    g = ex.gen(41)
    x = _edge_rows(256, g)
    xhat = getattr(ops, f"{fmt}_fakequant")(x)
    want = _composition(ops, fmt, x)
    _check_bits(xhat, want, f"{fmt} edge rows")
    assert bool(torch.isnan(xhat[1, :32]).all()) and bool(torch.isnan(xhat[2, 32:64]).all())
    assert not bool(xhat[0, :32].view(torch.int16).ne(0).any()), "a zero block stays +0"
    sub = xhat[4].float()
    assert bool(((sub != 0) & (sub.abs() < 2.0**-126)).any()), "premise: row 4 has subnormal results"
    _, s = getattr(ops, f"{fmt}_quantize")(x, False)
    top = {"mxfp8": 247, "mxfp4": 253}[fmt]   # RCEIL(3.3895e38 / max_pos)
    assert int(s.min()) == 0 and int(s.masked_select(s != 255).max()) == top, "premise: the e8m0 range ends"
    wide = (torch.randn(30, 384, device=DEV, generator=g) * 3).to(torch.bfloat16)
    a = getattr(ops, f"{fmt}_fakequant")(wide[:, 64:320])     # rows with a pitch of 384
    b = getattr(ops, f"{fmt}_fakequant")(wide[:, 64:320].contiguous())
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    _check_bits(a, _composition(ops, fmt, wide[:, 64:320]), f"{fmt} strided rows")


# ------------------------------------------------------------------------------------------------ 3-D to_mx
def test_3d_to_mx_matches_reference_golden():
    """The reference's CPU MXTensor.to_mx on [3, 256, 256] and [3, 128, 96] weights, mxfp8 and mxfp4, blocked and plain
    scales, byte for byte."""
    from ao_b200.prototype.mx_formats import MXTensor

    d = np.load(os.path.join(HERE, "golden", "mx_3d.npz"))
    for tag in ("3x256x256", "3x128x96"):
        w = torch.from_numpy(d[f"x_{tag}"].view(np.int16)).view(torch.bfloat16).cuda()
        for fmt in FMTS:
            for layout, swz in (("blocked", True), ("plain", False)):
                t = MXTensor.to_mx(w, ELEM[fmt], 32, is_swizzled_scales=swz)
                assert t.shape == w.shape, (fmt, tag, layout)
                assert np.array_equal(t.qdata.view(torch.uint8).cpu().numpy(), d[f"q_{fmt}_{tag}"]), (fmt, tag, layout)
                assert np.array_equal(t.scale.view(torch.uint8).cpu().numpy(), d[f"s_{fmt}_{tag}_{layout}"]), (fmt, tag, layout)


# ------------------------------------------------------------------------------------------------ handler
class Experts(torch.nn.Module):
    """An MoE expert layer: torch._grouped_mm on a 3-D parameter [E, N, K]."""

    def __init__(self, w):
        super().__init__()
        self.w = torch.nn.Parameter(w)

    def forward(self, x, offs):
        return torch._grouped_mm(x, self.w.transpose(-2, -1), offs=offs)


def _quantized(fmt, w):
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig, MXTensor
    from ao_b200.quantization import FqnToConfig, quantize_

    m = Experts(w)
    cfg = MXDynamicActivationMXWeightConfig(activation_dtype=ELEM[fmt], weight_dtype=ELEM[fmt])
    quantize_(m, FqnToConfig({"w": cfg}), filter_fn=None)
    assert isinstance(m.w, MXTensor) and m.w.shape == w.shape and m.w.is_swizzled_scales
    return m


def _blocks_with_max(fmt, R, K, small, lead, sb_lo, sb_hi, g):
    """fp64 [R, K] values whose every 32-block holds +-max_pos at position `lead` and codes from `small` elsewhere, times
    2^(b - 127), b in [sb_lo, sb_hi] per block: to_mx gives back exactly these codes and bytes (RCEIL of max_pos * 2^j
    is 2^j)."""
    v = ex.pick(small, (R, K), g)
    v.view(R, K // 32, 32)[:, :, lead] = ex.pick([MAXC[fmt], -MAXC[fmt]], (R, K // 32), g)
    return v * ex.pow2(ex.randint(sb_lo, sb_hi, (R, K // 32), g) - 127).repeat_interleave(32, 1)


@pytest.mark.parametrize("fmt", FMTS)
@torch.no_grad()
def test_handler_exact_operands(fmt):
    """quantize_ through FqnToConfig, then torch._grouped_mm(x, w.transpose(-2, -1), offs): equal to the fp64 result
    rounded once to bf16 and to F.linear(x[rows_e], w[e]) (select + the dense MX linear) bit for bit."""
    g = ex.gen(11 + (fmt == "mxfp4"))
    E, N, K = 4, 256, 512
    rows = [3, 17, 0, 40]
    M = sum(rows)
    small = [0.0, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5]
    W = _blocks_with_max(fmt, E * N, K, small, 1, 126, 127, g).reshape(E, N, K)
    X = _blocks_with_max(fmt, M, K, small, 0, 127, 128, g)
    ex.premise(X, W.reshape(E * N, K))
    m = _quantized(fmt, W.to(torch.bfloat16))
    assert torch.equal(m.w.dequantize(torch.float32).double(), W), "premise: the weights quantize exactly"
    x = X.to(torch.bfloat16)
    assert torch.equal(x.double(), X)
    offs = gm.cumulative(rows)
    ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
    start = 0
    for e, end in enumerate(offs):
        ref[start:end] = X[start:end] @ W[e].t()
        start = end
    ex.fp32_exact(ref, "handler: the fp64 reference")
    ref = ref.float().to(torch.bfloat16)
    y = m(x, torch.tensor(offs, dtype=torch.int32, device=DEV))
    assert y.shape == (M, N) and y.dtype == torch.bfloat16
    assert torch.equal(y.view(torch.int16), ref.view(torch.int16))
    start = 0
    for e, end in enumerate(offs):
        if end > start:
            d = torch.nn.functional.linear(x[start:end], m.w[e])
            assert torch.equal(d.view(torch.int16), y[start:end].view(torch.int16)), f"expert {e}"
        start = end


def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    d = (ref - out).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


@pytest.mark.parametrize("fmt", FMTS)
@torch.no_grad()
def test_handler_matches_select_and_dense_random(fmt):
    torch.manual_seed(3)
    E, K, N = 8, 512, 384
    rows = [5, 0, 40, 1, 130, 0, 16, 9]
    w = torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16)
    w[0] *= 10.0
    w[-1] *= 1e-3
    m = _quantized(fmt, w)
    x = torch.randn(sum(rows), K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm.cumulative(rows), device=DEV, dtype=torch.int32)
    y = m(x, offs)
    assert sqnr(torch._grouped_mm(x, w.transpose(-2, -1), offs=offs), y) > {"mxfp8": 20.0, "mxfp4": 8.0}[fmt]
    start = 0
    for e, end in enumerate(gm.cumulative(rows)):
        if end > start:
            d = torch.nn.functional.linear(x[start:end], m.w[e])
            assert sqnr(d, y[start:end]) >= 80.0, f"expert {e}"
        start = end


# ------------------------------------------------------------------------------------------------ CUDA graph
@pytest.mark.parametrize("fmt", FMTS)
@torch.no_grad()
def test_cuda_graph_replay_with_new_routing(fmt):
    """Capture the quantized expert forward, then write a different routing into the static offs and x: the replay
    must match eager on the new routing, so the host never read offs."""
    E, K, N, M = 8, 512, 1024, 48
    torch.manual_seed(1)
    m = _quantized(fmt, torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16))
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm.cumulative([6] * 8), dtype=torch.int32, device=DEV)
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
        offs.copy_(torch.tensor(gm.cumulative(rows), dtype=torch.int32))
        g.replay()
        want = m(x, offs)
        torch.cuda.synchronize()
        n = gm.cumulative(rows)[-1]
        assert torch.equal(y[:n].view(torch.int16), want[:n].view(torch.int16)), f"routing {rows}"


# ------------------------------------------------------------------------------------------------ PDL handoffs
def _lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    for fmt in FMTS:
        getattr(lib, f"ao_{fmt}_fakequant").argtypes = [vp, i32, i32, i32, vp, vp]
        getattr(lib, f"ao_{fmt}_grouped_mm").argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    lib.ao_fp8_quantize_rowwise.argtypes = [vp, i32, i32, vp, vp, vp]
    return lib


@pytest.mark.parametrize("fmt", FMTS)
def test_pdl_overlapped_equals_serialized(fmt):
    """An upstream kernel writes x and offs, then fakequant -> grouped GEMM, parked behind a long kernel (the stall head
    of tests/test_pdl_handoffs_gpu.py): bit for bit the same launches run one at a time, and as a graph."""
    lib = _lib()
    head = Head(lib)
    M, E, N, K = 300, 4, 1024, 2048
    g = ex.gen(32)
    wq, ws_blocked, _ = mx_weights(fmt, E, N, K, g)
    x0 = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    counts = torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV)
    buf = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    c = Chain(lib, f"upstream x, cumsum offs -> {fmt} fakequant -> grouped {fmt}")
    offs = c.out((E,), torch.int32)
    x = c.out((M, K), torch.bfloat16)
    xhat = c.out((M, K), torch.bfloat16)
    y = c.out((M, N), torch.bfloat16)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    c.torch(lambda: torch.mul(x0, 3.0, out=x))
    c.call(f"ao_{fmt}_fakequant", x, K, M, K, xhat)
    c.call(f"ao_{fmt}_grouped_mm", xhat, M, K, wq, ws_blocked, E, N, offs, y, buf, buf.numel())
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
