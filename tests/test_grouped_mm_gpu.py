"""torch._grouped_mm on rowwise-fp8 expert weights (torch.ops.ao_b200.fp8_rowwise_grouped_mm and the Float8Tensor
handler) on the GPU.

* bit-exact under every forced stream-K grid, with exact-product operands per expert (the fp8 set of
  tests/exact_operands.py): empty experts, experts of several m-blocks, a feature tail inside an expert, rows past
  offs[-1] and a malformed offs that the kernel clamps; the workspace flags must be back to zero after each launch;
* parity with the reference's _grouped_mm tests, with torch's F.scaled_grouped_mm and with the dense fp8 GEMM run
  expert by expert;
* a CUDA graph replayed with a different routing written into its static offs and x.
tests/test_grouped_schedule.py checks on the CPU that GROUPED_CASES reach every segment kind and that the schedule
(tests/grouped_model.py) stays inside [0, M).
"""
import copy

import pytest
import torch

import exact_operands as ex
import grouped_model as gm

pytestmark = pytest.mark.gpu

# (rows per expert, N, K, rows past the last expert, forced grids; None = every grid up to the host bound)
GROUPED_CASES = [
    ([13], 256, 1024, 0, None),                                   # E = 1, N_MMA 16
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 1024, 2, None),              # E = 8, empty experts, rows past offs[-1]
    ([150, 0, 70, 1], 256, 512, 0, None),                         # experts of three and two m-blocks
    ([7, 9, 0, 12], 144, 512, 3, None),                           # N = 144: a tile tail inside every expert
    ([20, 30], 640, 1024, 0, (3, 6, 7, 11)),                      # five n-tiles: CONTRIB, FULL and OWNER in one CTA
    ([1, 0, 2, 1, 0, 0, 3, 1] * 8, 128, 256, 5, None),            # E = 64
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 0, (1, 2, 5, 16, 64)),  # E = 64, one expert with every row
    # K = 16384, one tile split over up to 128 CTAs: owners gather 32 to 127 partials (N_MMA 16, 32 and 64; at 32
    # also 4 and 5, and 25 valid token columns of the 32)
    ([0, 16, 0], 128, 16384, 0, (33, 64, 65, 127, 128)),
    ([0, 25, 0], 128, 16384, 0, (5, 6, 33, 64, 65, 127, 128)),
    ([0, 64, 0], 128, 16384, 0, (33, 64, 65, 127, 128)),
]
# offs values that are not cumulative row ends: the kernel clamps each into [end[e-1], M]
MALFORMED = [([9, 4, -3, 30, 12, 500], 40), ([-5, -1, 0, 3], 8), ([100, 200], 64)]


def grids_of(case_rows, N, K, tail, grids, sm):
    M = sum(case_rows) + tail
    p = gm.plan(gm_offs(case_rows), M, N, K, grid=1, sm=sm)
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def gm_offs(rows):
    out, s = [], 0
    for r in rows:
        s += r
        out.append(s)
    return out


class GroupedCase:
    """Exact e4m3 operands: X in {-7..7} / 4, W in {-7..7} / 8, scales with three significant bits; every expert's
    products and chunk sums stay exact in fp32 (exact_operands.premise), so the output must equal the fp64 reference
    rounded once to bf16."""

    def __init__(self, offs, M, N, K, seed):
        E = len(offs)
        g = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E)
        X = ex.randint(-7, 7, (M, K), g).double() * 2.0**-2
        W = ex.randint(-7, 7, (E, N, K), g).double() * 2.0**-3
        self.xq, self.wq = X.to(torch.float8_e4m3fn), W.to(torch.float8_e4m3fn)
        assert torch.equal(self.xq.double(), X) and torch.equal(self.wq.double(), W)
        ex.premise(X, W.reshape(E * N, K), chunk=True)
        rs = ex.pick(ex.ODD, (M,), g) * 2.0**-8
        sw = ex.pick(ex.ODD, (E, N), g) * 2.0**-9
        self.rs, self.sw = rs.float(), sw.float()
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N, dtype=torch.float64, device=ex.DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                ref[start:end] = (X[start:end] @ W[e].t()) * (rs[start:end, None] * sw[e][None, :])
            start = end
        ex.fp32_exact(rs[:, None] * sw.reshape(1, -1), "grouped fp8: x_scale * w_scale")
        ex.fp32_exact(ref, "grouped fp8: acc * scales")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.offs = torch.tensor(offs, dtype=torch.int32, device=ex.DEV)
        self.M, self.N, self.K, self.E = M, N, K, E

    def run(self):
        return torch.ops.ao_b200.fp8_rowwise_grouped_mm(self.xq, self.rs, self.wq, self.sw, self.offs)


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
    bad = torch.zeros(len(grids), dtype=torch.int64, device=ex.DEV)
    raised = torch.zeros(len(grids), dtype=torch.int64, device=ex.DEV)
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
        p = gm.plan(case.offs.tolist(), case.M, case.N, case.K, grid=G, sm=ex.sm_count())
        pytest.fail(f"{what} M={case.M} N={case.N} K={case.K} E={case.E} grid={G or 'default'}: {nb} wrong elements, "
                    f"{nr} flags left raised (U={p.U}, device grid {p.G} of {p.G_host}); "
                    f"{len(wrong)} of {len(grids)} launches wrong")


@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, ci):
    rows, N, K, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(gm_offs(rows), sum(rows) + tail, N, K, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(rows, N, K, tail, grids, ex.sm_count()), f"case {ci} rows={rows}")


@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(offs, M, 256, 512, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


def test_all_experts_empty(ops, set_ctas):
    """U = 0: every CTA leaves right after reading offs, at the default grid and at a forced one."""
    case = GroupedCase([0, 0, 0], 20, 256, 512, seed=7)
    flags = ops.debug_workspace(case.xq).view(torch.int32)[:4096]
    for G in (0, 5):
        set_ctas(G)
        out = case.run()
        torch.cuda.synchronize()
        assert out.shape == (20, 256) and not bool(flags.ne(0).any())


# ------------------------------------------------------------------------------------------------ reference parity
def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    d = (ref - out).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


class GroupedMMModel(torch.nn.Module):
    """The reference's toy model whose only op is torch._grouped_mm (test_float8_tensor.py)."""

    def __init__(self, E, K, N, device, dtype=torch.bfloat16):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(E, N, K, device=device, dtype=dtype))

    def forward(self, x, offs):
        return torch._grouped_mm(x, self.weight.transpose(-2, -1), offs=offs)


def _quantized(E, K, N, granularity):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, quantize_

    ref = GroupedMMModel(E, K, N, device="cuda")
    m = copy.deepcopy(ref)
    quantize_(m, Float8DynamicActivationFloat8WeightConfig(granularity=granularity),
              filter_fn=lambda mod, fqn: isinstance(mod, GroupedMMModel) and hasattr(mod, "weight"))
    return ref, m


@pytest.mark.parametrize("E,K,N,m_per_group", [(4, 128, 256, [32, 64, 16, 48]), (8, 256, 512, [16] * 8)])
@torch.no_grad()
def test_fp8_grouped_mm_dynamic_act_weight(E, K, N, m_per_group):
    from ao_b200.quantization import Float8Tensor, PerRow

    torch.manual_seed(0)
    ref, m = _quantized(E, K, N, PerRow())
    assert isinstance(m.weight, Float8Tensor)
    assert m.weight.qdata.shape == (E, N, K) and m.weight.scale.shape == (E, N, 1)
    x = torch.randn(sum(m_per_group), K, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor([sum(m_per_group[: i + 1]) for i in range(E)], device="cuda", dtype=torch.int32)
    assert sqnr(ref.weight, m.weight.dequantize()) > 25.0
    y = m(x, offs)
    assert y.shape == (x.shape[0], N) and y.dtype == torch.bfloat16
    assert sqnr(ref(x, offs), y) > 20.0


@torch.no_grad()
def test_fp8_grouped_mm_non_rowwise_raises():
    from ao_b200.quantization import Float8Tensor, PerTensor

    ref, m = _quantized(4, 128, 256, PerTensor())
    assert isinstance(m.weight, Float8Tensor)
    x = torch.randn(160, 128, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor([32, 96, 112, 160], device="cuda", dtype=torch.int32)
    with pytest.raises(NotImplementedError):
        m(x, offs)


@pytest.mark.parametrize("E,N,K,rows", [(8, 512, 1024, [16, 0, 48, 32, 0, 16, 64, 16]), (4, 4096, 2048, [16] * 4),
                                        (16, 768, 2048, [0, 16, 32, 0, 16, 0, 0, 48, 16, 0, 0, 16, 32, 0, 16, 16])])
def test_vs_scaled_grouped_mm_and_dense_fp8(ops, E, N, K, rows):
    """Same quantized operands: against the fp64 product of the codes (> 45 dB), torch's rowwise
    F.scaled_grouped_mm and the dense fp8 GEMM expert by expert (> 70 dB, as test_lowp_gpu.py sets for the dense
    GEMM against torch._scaled_mm)."""
    g = torch.Generator(device="cuda").manual_seed(E + N + K)
    M = sum(rows)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(E, N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    xq, sx = ops.fp8_quantize_rowwise(x)
    wq, sw = ops.fp8_quantize_rowwise(w.reshape(E * N, K))
    wq, sw = wq.reshape(E, N, K), sw.reshape(E, N)
    offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device="cuda")
    y = ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), wq, sw, offs)
    ref64 = torch.empty(M, N, dtype=torch.float64, device="cuda")
    dense = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    start = 0
    for e, end in enumerate(gm_offs(rows)):
        if end > start:
            ref64[start:end] = (xq[start:end].double() @ wq[e].double().t()) * sx[start:end].double() * sw[e].double()
            dense[start:end] = ops.fp8_rowwise_linear(xq[start:end], sx[start:end].reshape(-1), wq[e], sw[e], None)
        start = end
    assert sqnr(ref64, y) > 45.0
    assert sqnr(dense, y) > 70.0
    import torch.nn.functional as F

    try:
        y_t = F.scaled_grouped_mm(xq, wq.transpose(-2, -1), scale_a=sx.reshape(-1), scale_recipe_a=F.ScalingType.RowWise,
                                  scale_b=sw, scale_recipe_b=F.ScalingType.RowWise, offs=offs, output_dtype=torch.bfloat16)
    except (RuntimeError, NotImplementedError) as e:   # not every torch build has the sm90 grouped kernel
        pytest.skip(f"F.scaled_grouped_mm unavailable: {e}")
    assert sqnr(y_t, y) > 70.0


# ------------------------------------------------------------------------------------------------ CUDA graph
@torch.no_grad()
def test_cuda_graph_replay_with_new_routing():
    """Capture the quantized expert forward, then write a different routing into the static offs and x: the replay
    must match eager on the new routing, so the host never read offs."""
    from ao_b200.quantization import PerRow

    E, K, N, M = 8, 512, 1024, 48
    torch.manual_seed(1)
    _, m = _quantized(E, K, N, PerRow())
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs([6] * 8), dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(x, offs)   # warm-up on the capture stream: creates its workspace outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        y = m(x, offs)
    for rows in ([6] * 8, [0, 30, 0, 0, 1, 17, 0, 0], [48, 0, 0, 0, 0, 0, 0, 0], [0] * 7 + [40]):
        x.copy_(torch.randn(M, K, device="cuda", dtype=torch.bfloat16))
        offs.copy_(torch.tensor(gm_offs(rows), dtype=torch.int32))
        g.replay()
        want = m(x, offs)
        torch.cuda.synchronize()
        n = gm_offs(rows)[-1]
        assert torch.equal(y[:n], want[:n]), f"routing {rows}"


# ------------------------------------------------------------------------------------------------ activation layouts
def _grouped_ops(ops, E=4, N=256, K=1024, g=128, M=37):
    """Every grouped op as (activation dtype, call(x) -> y) on random operands, offs [10, 10, 30, 35] of M = 37 rows."""
    gen = ex.gen(11)
    offs = torch.tensor([10, 10, 30, 35], dtype=torch.int32, device=ex.DEV)
    xs = torch.rand(M, device=ex.DEV, generator=gen) + 0.5
    ws = torch.rand(E, N, device=ex.DEV, generator=gen) + 0.5
    w8 = ex.randint(-128, 127, (E, N, K), gen).to(torch.int8)
    w_e4m3 = torch.randn(E, N, K, device=ex.DEV, generator=gen).to(torch.float8_e4m3fn)
    w4 = ex.randint(-2**31, 2**31 - 1, (E, N // 8, K // 128, 32, 4), gen).to(torch.int32)
    sz = (torch.randn(E, K // g, N, 2, device=ex.DEV, generator=gen) * 0.1).to(torch.bfloat16)
    w_fp4 = ex.randint(0, 255, (E, N, K // 2), gen).to(torch.uint8)
    sf_fp4 = ex.randint(0x30, 0x3F, (E * N * K // 16,), gen).to(torch.uint8)   # e4m3 block scales 0.5 .. 0.94
    pts = torch.rand(E, device=ex.DEV, generator=gen) + 0.5
    return {
        "fp8_rowwise": (torch.float8_e4m3fn, lambda x: ops.fp8_rowwise_grouped_mm(x, xs, w_e4m3, ws, offs)),
        "fp8_weight": (torch.bfloat16, lambda x: ops.fp8_weight_grouped_mm(x, w_e4m3, ws, offs)),
        "int8_weight": (torch.bfloat16, lambda x: ops.int8_weight_grouped_mm(x, w8, ws, offs)),
        "int8_dyn": (torch.int8, lambda x: ops.int8_dyn_grouped_mm(x, xs, w8, ws, offs)),
        "nvfp4": (torch.bfloat16, lambda x: ops.nvfp4_grouped_mm(x, xs, w_fp4, sf_fp4, pts, offs)),
        "int4": (torch.bfloat16, lambda x: ops.int4_tilepacked_grouped_mm(x, w4, g, sz, offs, 0)),
    }


@pytest.mark.parametrize("layout", ["column_slice", "storage_offset"])
@pytest.mark.parametrize("op", ["fp8_rowwise", "fp8_weight", "int8_weight", "int8_dyn", "nvfp4", "int4"])
def test_misaligned_activation_views_equal_a_contiguous_copy(ops, op, layout):
    """Every grouped op takes its activations as any 2-D view: one that does not start on 16 bytes (a column slice of
    a wider buffer, rows at an odd storage offset) gives the bits of the same call on a dense, aligned copy."""
    M, K = 37, 1024
    dtype, call = _grouped_ops(ops, M=M, K=K)[op]
    wide = torch.randn(M, K + 8, device=ex.DEV, generator=ex.gen(12))
    wide = (wide * 40).clamp(-128, 127).to(torch.int8) if dtype == torch.int8 else wide.to(dtype)
    x = wide[:, 4:4 + K] if layout == "column_slice" else wide.flatten()[4:4 + M * K].view(M, K)
    dense = x.clone(memory_format=torch.contiguous_format)
    assert x.data_ptr() % 16 != 0 and dense.data_ptr() % 16 == 0
    y, want = call(x), call(dense)
    assert torch.equal(y[:35].view(torch.int16), want[:35].view(torch.int16))
