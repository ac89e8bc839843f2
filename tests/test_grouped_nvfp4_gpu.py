"""torch._grouped_mm on NVFP4 expert weights (torch.ops.ao_b200.nvfp4_grouped_mm, nvfp4_fakequant_grouped and the
NVFP4Tensor handler) on the GPU.

* the GEMM bit-exact under every forced stream-K grid, with exact-product operands per expert (bf16 xhat, odd per-token
  scales, e2m1 weight codes with scale bytes from a window, odd per-expert scales): empty experts, experts of several
  m-blocks, E = 1 and E = 64, rows past offs[-1], malformed offs, token tiles 16 / 32 / 64 / 128; the workspace flags
  must be back to zero after each launch;
* the per-expert activation quantizer bit-exact against nvfp4_quantize on each expert's rows (and the oracle);
* the reference's tests (test_grouped_mm_nvfp4, test_nvfp4_per_expert_scale) and a golden fixture of its CPU 3-D
  to_nvfp4;
* the handler against the dense NVFP4 linear expert by expert;
* a CUDA graph replayed with a different routing written into its static x and offs.
tests/test_grouped_nvfp4_host.py checks on the CPU that GROUPED_CASES reach every segment kind and token tile.
"""
import copy
import os

import numpy as np
import pytest
import torch

import exact_operands as ex
import grouped_model as gm
import grouped_nvfp4_model as gnm

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (rows per expert, N, K, rows past the last expert, forced grids; None = every grid up to the host bound)
GROUPED_CASES = [
    ([13], 128, 1024, 0, None),                                   # E = 1, N_MMA 16
    ([7, 9, 0, 12], 128, 1024, 3, None),                          # N_MMA 32, rows past offs[-1]
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 512, 2, None),               # E = 8, empty experts, N_MMA 64
    ([150, 0, 70, 1], 256, 512, 0, (1, 2, 3, 5, 8, 13, 21, 34)),  # N_MMA 128, experts of two m-blocks
    ([20, 30], 640, 1024, 0, (3, 6, 7, 11)),                      # five n-tiles: CONTRIB, FULL and OWNER in one CTA
    ([1, 0, 2, 1, 0, 0, 3, 1] * 8, 128, 256, 5, None),            # E = 64, N_MMA 128
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 0, (1, 2, 5, 16, 64)),  # E = 64, one expert with every row
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
    p = gnm.plan(gm_offs(case_rows), M, N, K, grid=1, sm=sm)
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def stacked_blocked(w_bytes):
    """[E, N, K/16] scale bytes -> each expert's blocked scales, one after the other."""
    return torch.stack([ex.to_blocked(w_bytes[e]) for e in range(w_bytes.shape[0])])


class GroupedCase:
    """Exact operands: X in {-3..3} / 2 (bf16), per-token scales odd * 2^-6, weights e2m1 codes times scale bytes
    0x30..0x37, per-expert scales odd * 2^-4: every product, sum and epilogue product is exact in fp32
    (exact_operands.premise, fp32_exact), so the output must equal the fp64 reference rounded once to bf16."""

    def __init__(self, offs, M, N, K, seed):
        E = len(offs)
        g = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E)
        X = ex.randint(-3, 3, (M, K), g).double() * 0.5
        wc = ex.randint(0, 15, (E, N, K), g)
        wb = ex.randint(0x30, 0x37, (E, N, K // 16), g)
        W = ex.e2m1_value(wc) * ex.e4m3_bytes_value(wb).repeat_interleave(16, 2)
        ex.premise(X, W.reshape(E * N, K))
        rs = ex.pick(ex.ODD, (M,), g) * 2.0**-6
        wp = ex.pick(ex.ODD, (E,), g) * 2.0**-4
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N, dtype=torch.float64, device=ex.DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                acc = (X[start:end] @ W[e].t()) * rs[start:end, None]
                ex.fp32_exact(acc, "grouped nvfp4: acc * x_scale")
                ref[start:end] = acc * wp[e]
            start = end
        ex.fp32_exact(ref, "grouped nvfp4: acc * x_scale * w_pts")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.x = X.to(torch.bfloat16)
        self.wq = torch.stack([ex.pack_e2m1(wc[e]) for e in range(E)])
        self.ws = stacked_blocked(wb.to(torch.uint8))
        self.rs, self.wp = rs.float(), wp.float()
        self.offs = torch.tensor(offs, dtype=torch.int32, device=ex.DEV)
        self.M, self.N, self.K, self.E = M, N, K, E

    def run(self):
        return torch.ops.ao_b200.nvfp4_grouped_mm(self.x, self.rs, self.wq, self.ws, self.wp, self.offs)


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
        p = gnm.plan(case.offs.tolist(), case.M, case.N, case.K, grid=G, sm=ex.sm_count())
        pytest.fail(f"{what} M={case.M} N={case.N} K={case.K} E={case.E} grid={G or 'default'}: {nb} wrong elements, "
                    f"{nr} flags left raised (U={p.U}, width {p.width}, device grid {p.G} of {p.G_host}); "
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
    case = GroupedCase([0, 0, 0], 20, 256, 512, seed=7)
    flags = ops.debug_workspace(case.x).view(torch.int32)[:4096]
    for G in (0, 5):
        set_ctas(G)
        out = case.run()
        torch.cuda.synchronize()
        assert out.shape == (20, 256) and not bool(flags.ne(0).any())


# ------------------------------------------------------------------------------------------------ quantizer
def _expert_rows(offs, M):
    ends, start, out = gm.row_ends(offs, M), 0, []
    for end in ends:
        out.append((start, end))
        start = end
    return out, (ends[-1] if ends else 0)


def _check_fakequant(ops, x, offs_list):
    """xhat / x_scale of nvfp4_fakequant_grouped against nvfp4_quantize of each expert's rows with that expert's
    scale, an exact dequant of its codes, and the oracle's quantizer."""
    from oracle import oracle as o

    from ao_b200.prototype.mx_formats import per_tensor_amax_to_scale

    M, K = x.shape
    offs = torch.tensor(offs_list, dtype=torch.int32, device="cuda")
    xhat, xs = ops.nvfp4_fakequant_grouped(x, offs)
    spans, end = _expert_rows(offs_list, M)
    torch.cuda.synchronize()
    for e, (s0, s1) in enumerate(spans):
        if s1 == s0:
            continue
        xe = x[s0:s1]
        a = per_tensor_amax_to_scale(torch.max(torch.abs(xe))).reshape(1)
        assert torch.equal(xs[s0:s1], a.expand(s1 - s0)), f"expert {e}: x_scale"
        if float(a) == 0.0:
            assert not bool(xhat[s0:s1].view(torch.int16).ne(0).any()), f"expert {e}: all-zero rows give xhat = 0"
            continue
        q, sc = ops.nvfp4_quantize(xe.contiguous(), a, False)
        codes = torch.stack([q & 15, q >> 4], -1).reshape(s1 - s0, K)
        want = ex.e2m1_value(codes) * ex.e4m3_bytes_value(sc).repeat_interleave(16, 1)
        assert torch.equal(xhat[s0:s1].double(), want), f"expert {e}: xhat values"
        assert torch.equal(xhat[s0:s1].view(torch.int16), want.to(torch.bfloat16).view(torch.int16)), f"expert {e}: bits"
        qo, so = o.nvfp4_quantize(o.bf16_bits(xe), float(a.item()))
        assert np.array_equal(q.cpu().numpy(), qo) and np.array_equal(sc.cpu().numpy(), so), f"expert {e}: oracle"
    assert not bool(xhat[end:].view(torch.int16).ne(0).any()) and not bool(xs[end:].ne(0).any()), "rows past the end"


@pytest.mark.parametrize("rows,tail,K", [([1, 3, 4, 16], 0, 128), ([40, 0, 0, 7, 300, 1, 0, 9], 5, 512),
                                         ([2] * 64, 3, 256), ([700], 0, 4096)])
def test_fakequant_per_expert_bit_exact(ops, rows, tail, K):
    g = torch.Generator(device="cuda").manual_seed(sum(rows) + K)
    M = sum(rows) + tail
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    offs = gm_offs(rows)
    x[: offs[0]] *= 10.0      # the reference's magnitudes: expert 0 x 10, the last x 1e-3
    x[offs[-2] if len(offs) > 1 else 0: offs[-1]] *= 1e-3
    _check_fakequant(ops, x, offs)


def test_fakequant_zero_expert_malformed_offs_and_strided_rows(ops):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(40, 256, device="cuda", generator=g).to(torch.bfloat16)
    x[3:9] = 0.0   # expert 1 of the first routing: every row zero
    _check_fakequant(ops, x, [3, 9, 9, 30])
    for offs, M in MALFORMED:
        xm = torch.randn(M, 256, device="cuda", generator=g).to(torch.bfloat16)
        _check_fakequant(ops, xm, offs)
    wide = torch.randn(30, 384, device="cuda", generator=g).to(torch.bfloat16)
    offs = torch.tensor([10, 30], dtype=torch.int32, device="cuda")
    a, sa = ops.nvfp4_fakequant_grouped(wide[:, :256], offs)
    b, sb = ops.nvfp4_fakequant_grouped(wide[:, :256].contiguous(), offs)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(sa, sb)


# ------------------------------------------------------------------------------------------------ reference tests
def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    d = (ref - out).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


class GroupedMMModel(torch.nn.Module):
    """The reference's toy model whose only op is torch._grouped_mm (test_inference_workflow.py)."""

    def __init__(self, E, K, N, device, dtype=torch.bfloat16):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(E, N, K, device=device, dtype=dtype))

    def forward(self, x, offs):
        return torch._grouped_mm(x, self.weight.transpose(-2, -1), offs=offs)


def _quantized(model):
    from ao_b200.prototype.mx_formats import NVFP4DynamicActivationNVFP4WeightConfig
    from ao_b200.quantization import quantize_

    m = copy.deepcopy(model)
    quantize_(m, NVFP4DynamicActivationNVFP4WeightConfig(use_triton_kernel=False),
              filter_fn=lambda mod, *args: isinstance(mod, GroupedMMModel) and hasattr(mod, "weight"))
    return m


@torch.no_grad()
def test_grouped_mm_nvfp4():
    from ao_b200.prototype.mx_formats import NVFP4Tensor

    torch.manual_seed(0)
    E, K, N = 4, 128, 256
    m_per_group = [1, 3, 4, 16]
    ref = GroupedMMModel(E, K, N, device="cuda")
    ref.weight[0, :, :] *= 10.0
    ref.weight[-1, :, :] *= 1e-3
    m = _quantized(ref)
    x = torch.randn(sum(m_per_group), K, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs(m_per_group), device="cuda", dtype=torch.int32)
    y_ref = ref(x, offs)
    assert isinstance(m.weight, NVFP4Tensor)
    assert m.weight.per_tensor_scale.shape == (E, 1, 1)
    assert sqnr(ref.weight, m.weight.dequantize()) > 18.0
    wt = m.weight.transpose(-2, -1)
    assert tuple(wt.shape) == (E, K, N)
    y = m(x, offs)
    assert y.shape == (x.shape[0], N) and y.dtype == torch.bfloat16
    assert sqnr(y_ref, y) > 15.0


def test_nvfp4_per_expert_scale():
    from ao_b200.prototype.mx_formats import NVFP4Tensor, per_tensor_amax_to_scale

    E, K, N = 2, 64, 128
    x0 = torch.randn(N, K, dtype=torch.bfloat16, device="cuda")
    x1 = torch.randn(N, K, dtype=torch.bfloat16, device="cuda") * 2
    p0, p1 = per_tensor_amax_to_scale(torch.max(torch.abs(x0))), per_tensor_amax_to_scale(torch.max(torch.abs(x1)))
    t0 = NVFP4Tensor.to_nvfp4(x0, per_tensor_scale=p0, is_swizzled_scales=False)
    t1 = NVFP4Tensor.to_nvfp4(x1, per_tensor_scale=p1, is_swizzled_scales=False)
    xc = torch.cat([x0, x1], dim=0).view(E, N, K)
    tc = NVFP4Tensor.to_nvfp4(xc, per_tensor_scale=torch.stack([p0, p1]).view(E, 1, 1), is_swizzled_scales=False)
    assert torch.equal(torch.cat([t0.qdata, t1.qdata]).view(E, N, K // 2), tc.qdata)
    assert torch.equal(torch.cat([t0.scale, t1.scale]).view(torch.uint8).view(E, N, K // 16), tc.scale.view(torch.uint8))
    assert torch.equal(torch.cat([t0.dequantize(), t1.dequantize()]).view(E, N, K), tc.dequantize())


def test_3d_to_nvfp4_matches_reference_golden():
    """The reference's CPU NVFP4Tensor.to_nvfp4 on a [3, 128, 128] weight with per-expert scales, byte for byte."""
    from ao_b200.prototype.mx_formats import NVFP4Tensor

    d = np.load(os.path.join(HERE, "golden", "nvfp4_3d.npz"))
    w = torch.from_numpy(d["x"].view(np.int16)).view(torch.bfloat16).cuda()
    pts = torch.from_numpy(d["pts"]).cuda().view(-1, 1, 1)
    for name, swz in (("blocked", True), ("plain", False)):
        t = NVFP4Tensor.to_nvfp4(w, per_tensor_scale=pts, is_swizzled_scales=swz)
        assert np.array_equal(t.qdata.cpu().numpy(), d[f"q_{name}"]), name
        assert np.array_equal(t.scale.view(torch.uint8).cpu().numpy(), d[f"s_{name}"]), name


# ------------------------------------------------------------------------------------------------ handler vs dense
def _dense_expert(w, e, x_rows):
    """The dense NVFP4 linear (F.linear on the 2-D NVFP4Tensor of expert e: nvfp4_quantize + nvfp4_linear)."""
    from ao_b200.prototype.mx_formats import NVFP4Tensor

    w2 = NVFP4Tensor(w.qdata[e], w.scale[e], 16, torch.bfloat16, w.per_tensor_scale.reshape(-1)[e], None, True,
                     False, w.act_quant_kwargs)
    return torch.nn.functional.linear(x_rows, w2)


@torch.no_grad()
def test_handler_matches_dense_random():
    torch.manual_seed(3)
    E, K, N = 8, 512, 384
    rows = [5, 0, 40, 1, 130, 0, 16, 9]
    m = _quantized(GroupedMMModel(E, K, N, device="cuda"))
    x = torch.randn(sum(rows), K, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), device="cuda", dtype=torch.int32)
    y = m(x, offs)
    start = 0
    for e, end in enumerate(gm_offs(rows)):
        if end > start:
            d = _dense_expert(m.weight, e, x[start:end])
            assert sqnr(d, y[start:end]) >= 80.0, f"expert {e}"
        start = end


@torch.no_grad()
def test_handler_matches_dense_exact():
    """Exact operands: each 16-block of x holds an e2m1 code 6 (so its block scale is exactly the chosen byte) and each
    expert's largest element is 6 * 448 * 2^-j (so a_pts = 2^-j); weights are codes {0, +-0.5, +-1} times bytes
    0x30..0x37 with a per-expert scale 2^-i.  Both the handler and the dense NVFP4 linear must give the fp64 result
    rounded once to bf16."""
    from ao_b200.prototype.mx_formats import NVFP4Tensor
    from ao_b200.prototype.mx_formats.nvfp4_tensor import QuantizeTensorToNVFP4Kwargs

    g = ex.gen(11)
    E, N, K = 4, 256, 512
    rows = [3, 17, 0, 40]
    M = sum(rows)
    wc = ex.pick([0, 1, 2, 8, 9, 10], (E, N, K), g).long()
    wb = ex.randint(0x30, 0x37, (E, N, K // 16), g)
    wp = torch.tensor([2.0**-3, 2.0**-1, 1.0, 2.0**2], dtype=torch.float64, device="cuda")
    W = ex.e2m1_value(wc) * ex.e4m3_bytes_value(wb).repeat_interleave(16, 2) * wp.view(E, 1, 1)
    kw = QuantizeTensorToNVFP4Kwargs(use_dynamic_per_tensor_scale=True, is_swizzled_scales=True)
    w = NVFP4Tensor(torch.stack([ex.pack_e2m1(wc[e]) for e in range(E)]),
                    stacked_blocked(wb.to(torch.uint8)).view(torch.float8_e4m3fn), 16, torch.bfloat16,
                    wp.float().view(E, 1, 1), None, True, False, kw)
    xc = ex.pick([0, 1, 2, 3, 8, 9, 10, 11], (M, K), g).long()
    xc.view(M, K // 16, 16)[:, :, 0] = ex.pick([7, 15], (M, K // 16), g).long()   # +-6 in every block
    xb = ex.randint(0x38, 0x3F, (M, K // 16), g)
    X = ex.e2m1_value(xc) * ex.e4m3_bytes_value(xb).repeat_interleave(16, 1)
    offs = gm_offs(rows)
    start = 0
    for e, end in enumerate(offs):
        if end > start:
            a = 2.0 ** -(e + 2)
            X[start:end] *= a
            X[start, 1:16] = 0.0   # the expert's maximum, 6 * 448 * a, alone in its block
            X[start, 0] = 6 * 448 * a
        start = end
    x = X.to(torch.bfloat16)
    assert torch.equal(x.double(), X)
    ref = torch.zeros(M, N, dtype=torch.float64, device="cuda")
    start = 0
    for e, end in enumerate(offs):
        if end > start:
            ex.premise(X[start:end], W[e])
            ref[start:end] = X[start:end] @ W[e].t()
        start = end
    ex.fp32_exact(ref, "handler: the fp64 reference")
    ref = ref.float().to(torch.bfloat16)
    y = torch._grouped_mm(x, w.transpose(-2, -1), offs=torch.tensor(offs, dtype=torch.int32, device="cuda"))
    assert torch.equal(y.view(torch.int16), ref.view(torch.int16))
    start = 0
    for e, end in enumerate(offs):
        if end > start:
            d = _dense_expert(w, e, x[start:end])
            assert torch.equal(d.view(torch.int16), y[start:end].view(torch.int16)), f"expert {e}"
        start = end


# ------------------------------------------------------------------------------------------------ CUDA graph
@torch.no_grad()
def test_cuda_graph_replay_with_new_routing():
    """Capture the quantized expert forward, then write a different routing into the static offs and x: the replay
    must match eager on the new routing, so the host never read offs."""
    E, K, N, M = 8, 512, 1024, 48
    torch.manual_seed(1)
    m = _quantized(GroupedMMModel(E, K, N, device="cuda"))
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
