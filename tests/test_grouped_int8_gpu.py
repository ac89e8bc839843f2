"""torch._grouped_mm on 3-D int8 expert weights (torch.ops.ao_b200.int8_weight_grouped_mm / int8_dyn_grouped_mm and the
Int8Tensor handler) on the GPU:

* dynamic (int8 x int8): every expert's rows equal the dense int8_dyn_linear on that expert's weights bit for bit, for
  random operands (s32 sums are exact), under every forced stream-K grid, at every token tile, with N and K tails,
  empty experts, malformed (clamped) offs and all experts empty; single-tile layouts put owners with fewer
  contributors than ring stages, exactly as many and more;
* weight-only (bf16 x int8): bit for bit on exact operands under the same grids (also at N % 8 != 0), within the fp32
  sum bound of the recipe on random ones;
* rows from offs[-1] on keep a sentinel; the handler equals select + F.linear and the reference's fixture for the
  three configs; CUDA-graph replay with new routings, torch.compile fullgraph, opcheck, save / load and a PDL chain
  against a serialized run.

Exact weight-only operands: activations -8..8 times 2^-3 and codes -127..127: every product is a multiple of 2^-3 below
2^10 of them, and K products stay below 2^24 such quanta, so fp32 sums exactly in any order.
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
import streamk_model as sk
from test_grouped_int4_gpu import Chain, Head

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda"

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
MALFORMED = [([9, 4, -3, 30, 12, 500], 40), ([-5, -1, 0, 3], 8), ([100, 200], 64)]
OPS = ("int8", "int8wo")   # streamk_model formats: Grouped<SsFmt<KIND_I8>> and Grouped<Int8WoFmt>


def grids_of(fmt, rows, N, K, tail, grids, sm):
    M = sum(rows) + tail
    p = gm.plan(gm.cumulative(rows), M, N, K, grid=1, sm=sm, fmt=fmt)
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


class GroupedCase:
    """int8 expert weights [E, N, K] with per-row scales that differ per expert.  int8: random int8 activations with
    random row scales, reference = the dense int8_dyn_linear per expert.  int8wo: exact bf16 activations, reference =
    the recipe's roundings applied to the exact fp64 sums (which the dense int8_weight_linear also gives)."""

    def __init__(self, fmt, offs, M, N, K, seed):
        E = len(offs)
        g = ex.gen(seed * 7919 + M * 31 + N * 7 + K + E + (fmt == "int8"))
        self.fmt = fmt
        self.wq = ex.randint(-127, 127, (E, N, K), g).to(torch.int8)
        self.ws = (torch.rand(E, N, device=DEV, generator=g) + 0.5) * ex.pow2(-(6 + torch.arange(E, device=DEV) % 24))[:, None].float()
        self.ends = gm.row_ends(offs, M)
        self.valid = self.ends[-1] if self.ends else 0
        self.offs = torch.tensor(offs, dtype=torch.int32, device=DEV)
        self.M, self.N, self.K, self.E = M, N, K, E
        ops = ex.ops()
        ref = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
        if fmt == "int8":
            self.xq = ex.randint(-128, 127, (M, K), g).to(torch.int8)
            self.xs = torch.rand(M, device=DEV, generator=g) * 1e-2 + 1e-3
            start = 0
            for e, end in enumerate(self.ends):
                if end > start:
                    ref[start:end] = ops.int8_dyn_linear(self.xq[start:end], self.xs[start:end].contiguous(), self.wq[e],
                                                         self.ws[e].contiguous(), None)
                start = end
        else:
            X = ex.randint(-8, 8, (M, K), g).double() * 2.0**-3
            self.x = X.to(torch.bfloat16)
            assert K * 8 * 127 < 2**24, "premise: K products stay below 2^24 quanta"
            start = 0
            for e, end in enumerate(self.ends):
                if end > start:
                    acc = X[start:end] @ self.wq[e].double().t()
                    ex.fp32_exact(acc, "grouped int8 weight-only: acc")
                    ref[start:end] = wo_epilogue(acc.float(), self.ws[e])
                start = end
        self.ref = ref[: self.valid]

    def run(self):
        ops = ex.ops()
        if self.fmt == "int8":
            return ops.int8_dyn_grouped_mm(self.xq, self.xs, self.wq, self.ws, self.offs)
        return ops.int8_weight_grouped_mm(self.x, self.wq, self.ws, self.offs)


def wo_epilogue(acc32, s):
    """The weight-only recipe's roundings on fp32 sums: bf16(bf16(bf16(acc) * bf16(s))) (a product of two bf16 is
    exact in fp32)."""
    return (acc32.to(torch.bfloat16).float() * s.to(torch.bfloat16).float()).to(torch.bfloat16)


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
    flags = ops.debug_workspace(case.ws).view(torch.int32)[:4096]
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


@pytest.mark.parametrize("fmt", OPS)
@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, fmt, ci):
    rows, N, K, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(fmt, gm.cumulative(rows), sum(rows) + tail, N, K, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(fmt, rows, N, K, tail, grids, ex.sm_count()), f"case {ci}")


# one expert whose rows fill one tile of each staging width, K = 8192: a forced grid of G CTAs gives its owner G - 1
# contributors, so the grids below put owners below, at and above the ring's stage count S
def _staging_layouts(fmt):
    out = []
    for width in sk.WIDTHS[fmt]:
        _, _, S, staging = sk.ring(fmt, width, grouped=True)
        if not staging:
            continue
        for rows in sorted({width, width - 1, max(1, width // 2 + 1)}):
            out.append((width, S, rows))
    return out


@pytest.mark.parametrize("fmt", OPS)
def test_owner_gather_below_at_and_above_the_ring(ops, set_ctas, fmt):
    for width, S, rows in _staging_layouts(fmt):
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


@pytest.mark.parametrize("fmt", OPS)
@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, fmt, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(fmt, offs, M, 200, 1040, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


def test_weight_only_n_not_a_multiple_of_8(ops, set_ctas):
    """No N rule for the weight-only op: every weight box may start on any row of the [E*N, K] map and the scales are
    read by the epilogue.  N = 77 and 333 (boxes at rows e*N + 128t), bit-exact under forced grids."""
    for N, rows in ((77, [3, 0, 20, 9]), (333, [40, 1, 0, 100])):
        case = GroupedCase("int8wo", gm.cumulative(rows), sum(rows) + 2, N, 1040, seed=N)
        _sweep(ops, set_ctas, case, [None, 1, 2, 5, 17, 64], f"N={N}")


def _lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.ao_int8_weight_grouped_mm.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    lib.ao_int8_dyn_grouped_mm.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    lib.ao_fp8_quantize_rowwise.argtypes = [vp, i32, i32, vp, vp, vp]
    return lib


def _call(lib, case, y, ws):
    st = torch.cuda.current_stream().cuda_stream
    if case.fmt == "int8":
        rc = lib.ao_int8_dyn_grouped_mm(case.xq.data_ptr(), case.xs.data_ptr(), case.M, case.K, case.wq.data_ptr(),
                                        case.ws.data_ptr(), case.E, case.N, case.offs.data_ptr(), y.data_ptr(),
                                        ws.data_ptr(), ws.numel(), st)
    else:
        rc = lib.ao_int8_weight_grouped_mm(case.x.data_ptr(), case.M, case.K, case.wq.data_ptr(), case.ws.data_ptr(),
                                           case.E, case.N, case.offs.data_ptr(), y.data_ptr(), ws.data_ptr(),
                                           ws.numel(), st)
    assert rc == 0, lib.ao_b200_last_error()


@pytest.mark.parametrize("fmt", OPS)
def test_rows_past_the_last_expert_and_all_empty_experts_are_not_written(fmt):
    """Through the C ABI into a poisoned y: the rows from offs[-1] on keep their bytes, the rest is the reference; with
    every expert empty nothing is written and no flag stays raised."""
    lib = _lib()
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    for offs, M in (([5, 5, 20], 37), ([3, 40, 90], 130), ([0, 0, 0], 20)):
        case = GroupedCase(fmt, offs, M, 200, 1040, seed=3)
        y = torch.full((case.M, case.N), ex.POISON_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        _call(lib, case, y, ws)
        torch.cuda.synchronize()
        assert torch.equal(y[: case.valid].view(torch.int16), case.ref.view(torch.int16))
        assert bool((y[case.valid:].view(torch.int16) == ex.POISON_BF16).all()), offs
        assert not bool(ws[:4096 * 4].view(torch.int32).ne(0).any())


def test_weight_only_random_within_the_sum_bound(ops, set_ctas):
    """Random bf16 activations: y lies between the recipe's roundings of the fp64 sum -/+ the fp32 accumulation bound
    (K * 2^-24 * sum |x w|; the roundings are monotonic for positive scales), under forced grids."""
    torch.manual_seed(4)
    rows = [5, 0, 40, 1, 130, 0, 16, 9]
    E, N, K = len(rows), 1000, 4096
    offs = torch.tensor(gm.cumulative(rows), dtype=torch.int32, device=DEV)
    x = torch.randn(sum(rows), K, device=DEV).to(torch.bfloat16)
    wq = torch.randint(-127, 128, (E, N, K), device=DEV, dtype=torch.int8)
    s = torch.rand(E, N, device=DEV) * 1e-2 + 1e-4
    lo, hi = [], []
    start = 0
    for e, end in enumerate(gm.cumulative(rows)):
        if end > start:
            xe, we = x[start:end].double(), wq[e].double()
            ref, mag = xe @ we.t(), xe.abs() @ we.abs().t()
            err = mag * (K * 2.0**-24)
            lo.append(wo_epilogue((ref - err).float(), s[e]))
            hi.append(wo_epilogue((ref + err).float(), s[e]))
        start = end
    lo, hi = torch.cat(lo).float(), torch.cat(hi).float()
    for G in (0, 1, 7, 33, 132):
        set_ctas(G)
        y = ops.int8_weight_grouped_mm(x, wq, s, offs).float()
        assert bool(((y >= lo) & (y <= hi)).all()), G
    set_ctas(0)


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


def _config(mode, gran=None, act_scale=None):
    from ao_b200.quantization import (Int8DynamicActivationInt8WeightConfig, Int8StaticActivationInt8WeightConfig,
                                      Int8WeightOnlyConfig, PerRow, PerTensor)

    if mode == "wo":
        return Int8WeightOnlyConfig(granularity=gran or PerRow())
    if mode == "dyn":
        return Int8DynamicActivationInt8WeightConfig(granularity=gran or PerRow())
    return Int8StaticActivationInt8WeightConfig(act_quant_scale=act_scale, granularity=[PerTensor(), PerRow()])


def _quantized(model, mode="wo", gran=None, act_scale=None, fqn=True):
    from ao_b200.quantization import FqnToConfig, quantize_

    m = copy.deepcopy(model)
    cfg = _config(mode, gran, act_scale)
    if fqn:
        quantize_(m, FqnToConfig({"weight": cfg}), filter_fn=None)
    else:
        quantize_(m, cfg, filter_fn=lambda mod, name: isinstance(mod, GroupedMMModel))
    return m


MODES = ["wo", "wo_pt", "dyn", "static"]


def _mode_model(base, mode, x):
    from ao_b200.quantization import PerTensor

    if mode == "wo_pt":
        return _quantized(base, "wo", PerTensor())
    if mode == "static":
        m = _quantized(base, "static", act_scale=(x.float().abs().amax() / 127).reshape(1, 1))
        m.weight.act_pre_scale = (torch.rand(x.shape[1], device=DEV) + 0.5).to(torch.bfloat16)
        return m
    return _quantized(base, mode)


@torch.no_grad()
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("functional", [False, True])
def test_handler_equals_select_and_linear(mode, functional):
    """Every expert's rows equal the per-expert recipe select + F.linear bit for bit (weight-only: random bf16
    activations, the same K order per output tile as the dense kernel is not guaranteed, so exact-integer ones; the
    int8 x int8 sums are exact for any operands)."""
    torch.manual_seed(5)
    E, N, K = 6, 1000, 2064
    rows = [3, 17, 0, 40, 1, 9]
    base = GroupedMMModel(E, K, N)
    if mode.startswith("wo"):
        x = (torch.randint(-8, 9, (sum(rows), K), device=DEV) * 0.125).to(torch.bfloat16)
    else:
        x = torch.randn(sum(rows), K, device=DEV).to(torch.bfloat16)
    m = _mode_model(base, mode, x)
    offs = torch.tensor(gm.cumulative(rows), dtype=torch.int32, device=DEV)
    n0 = torch.ops.ao_b200.launch_count()
    y = m(x, offs, functional)
    launches = torch.ops.ao_b200.launch_count() - n0
    assert launches == (1 if mode.startswith("wo") else 2), launches   # quantizer + GEMM for int8 activations
    assert y.shape == (sum(rows), N) and y.dtype == torch.bfloat16
    w = m.weight
    start = 0
    for e, end in enumerate(gm.cumulative(rows)):
        if end > start:
            d = F.linear(x[start:end], w[e])
            assert torch.equal(d.view(torch.int16), y[start:end].view(torch.int16)), f"{mode} expert {e}"
        start = end
    if mode != "static":   # the random pre-scale changes the function: no bf16 model to compare with
        assert sqnr(base(x, offs), y) > 25.0


@torch.no_grad()
def test_handler_reduce_range_and_fp32_pre_scale_take_the_torch_quantizer():
    """Dynamic reduce_range and a static fp32 pre-scale quantize through the same per-row / per-tensor rules the dense
    linear uses; the grouped result still equals select + F.linear bit for bit."""
    from ao_b200.quantization import Int8DynamicActivationInt8WeightConfig, FqnToConfig, quantize_

    torch.manual_seed(8)
    rows = [4, 0, 30]
    base = GroupedMMModel(3, 512, 264)
    x = torch.randn(sum(rows), 512, device=DEV).to(torch.bfloat16)
    offs = torch.tensor(gm.cumulative(rows), dtype=torch.int32, device=DEV)
    m1 = copy.deepcopy(base)
    quantize_(m1, FqnToConfig({"weight": Int8DynamicActivationInt8WeightConfig(reduce_range=True)}), filter_fn=None)
    m2 = _mode_model(base, "static", x)
    m2.weight.act_pre_scale = m2.weight.act_pre_scale.float() * 1.01
    m3 = _mode_model(base, "static", x)
    m3.weight.act_quant_scale = m3.weight.act_quant_scale.to(torch.bfloat16)   # not the fused quantizer's dtype
    for m in (m1, m2, m3):
        y = m(x, offs)
        start = 0
        for e, end in enumerate(gm.cumulative(rows)):
            if end > start:
                assert torch.equal(F.linear(x[start:end], m.weight[e]).view(torch.int16),
                                   y[start:end].view(torch.int16)), e
            start = end


def test_golden_fixture():
    """The reference's per-expert F.linear through its select: the quantized tensors equal the fixture's; dynamic and
    static outputs bit for bit; weight-only one-hot outputs bit for bit and random ones within one bf16 step of the
    sum's rounding (the fp32 sums' order differs from the CPU's)."""
    from ao_b200.quantization import Int8Tensor, PerRow, PerTensor, QuantizeTensorToInt8Kwargs
    from test_grouped_int8_host import golden_shapes

    d = np.load(os.path.join(HERE, "golden", "int8_3d.npz"))
    b16 = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).to(DEV)   # noqa: E731
    u16 = lambda t: t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)   # noqa: E731
    for c, a in golden_shapes(d):
        w = b16(a["w"])
        offs = torch.from_numpy(a["offs"]).to(DEV)
        end = int(a["offs"][-1])
        for v in ("wo_PerRow", "wo_PerTensor", "dyn_PerRow", "static_PerTensor"):
            kind, gname = v.split("_")
            kw = {}
            if kind == "dyn":
                kw = dict(act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow()))
            elif kind == "static":
                kw = dict(act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerTensor()),
                          act_quant_scale=torch.from_numpy(a["act_scale"]).to(DEV), act_pre_scale=b16(a["pre"]))
            gran = PerTensor() if v == "wo_PerTensor" else PerRow()
            t = Int8Tensor.from_hp(w, gran, **kw)
            assert np.array_equal(t.qdata.cpu().numpy(), a[f"{v}_q"]), (c, v)
            assert np.array_equal(t.scale.cpu().numpy(), a[f"{v}_scale"]), (c, v)
            if v == "wo_PerTensor":
                continue
            with torch.no_grad():
                for fn in (torch._grouped_mm, F.grouped_mm):
                    ye = u16(fn(b16(a["xe"]), t.transpose(-2, -1), offs=offs)[:end])
                    y = u16(fn(b16(a["x"]), t.transpose(-2, -1), offs=offs)[:end])
                    assert np.array_equal(ye, a[f"{v}_ye"]), (c, v)
                    if kind == "wo":
                        got, want = y.astype(np.int32), a[f"{v}_y"].astype(np.int32)
                        assert (np.abs(got - want) <= 1).all() and (got == want).mean() > 0.9, (c, v)
                    else:
                        assert np.array_equal(y, a[f"{v}_y"]), (c, v)


# ------------------------------------------------------------------------------------------------ graph and compile
@torch.no_grad()
@pytest.mark.parametrize("mode", ["wo", "dyn", "static"])
def test_cuda_graph_replay_with_new_routing(mode):
    """Capture the quantized expert forward, then write new routings into the static offs and x: the replay must equal
    eager bit for bit, so the host never read offs."""
    E, K, N, M = 8, 2048, 1000, 48
    torch.manual_seed(1)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    m = _mode_model(GroupedMMModel(E, K, N), mode, x)
    offs = torch.tensor(gm.cumulative([6] * 8), dtype=torch.int32, device=DEV)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(x, offs)
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
        assert torch.equal(y[:n].view(torch.int16), want[:n].view(torch.int16)), f"{mode} routing {rows}"


@torch.no_grad()
@pytest.mark.parametrize("mode", ["wo", "dyn", "static"])
@pytest.mark.parametrize("backend", ["inductor", "aot_eager"])
def test_compile_fullgraph_through_the_handler(mode, backend):
    torch.manual_seed(2)
    x = torch.randn(20, 1024, device=DEV, dtype=torch.bfloat16)
    m = _mode_model(GroupedMMModel(4, 1024, 520), mode, x)
    offs = torch.tensor([3, 3, 12, 20], dtype=torch.int32, device=DEV)
    y = m(x, offs)
    torch._dynamo.reset()
    yc = torch.compile(m, fullgraph=True, backend=backend)(x, offs)
    assert torch.equal(y[:20].view(torch.int16), yc[:20].view(torch.int16))


def test_opcheck():
    g = ex.gen(9)
    wq = ex.randint(-127, 127, (3, 136, 1024), g).to(torch.int8)
    s = torch.rand(3, 136, device=DEV) + 0.5
    x = torch.randn(10, 1024, device=DEV).to(torch.bfloat16)
    xq = ex.randint(-127, 127, (10, 1024), g).to(torch.int8)
    xs = torch.rand(10, device=DEV) + 0.5
    offs = torch.tensor([2, 5, 10], dtype=torch.int32, device=DEV)
    # test_schema is left out: it multiplies the inputs, and torch has no mul for the int8 codes of a real checkpoint
    for op, args in ((torch.ops.ao_b200.int8_weight_grouped_mm.default, (x, wq, s, offs)),
                     (torch.ops.ao_b200.int8_dyn_grouped_mm.default, (xq, xs, wq, s, offs))):
        torch.library.opcheck(op, args, test_utils=("test_faketensor", "test_autograd_registration"))


@torch.no_grad()
@pytest.mark.parametrize("mode", MODES)
def test_save_load_then_grouped_forward(mode):
    from ao_b200.quantization import Int8Tensor

    torch.manual_seed(6)
    base = GroupedMMModel(4, 512, 296)
    x = torch.randn(40, 512, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([10, 10, 25, 40], dtype=torch.int32, device=DEV)
    m = _mode_model(base, mode, x)
    buf = io.BytesIO()
    torch.save(m.state_dict(), buf)
    buf.seek(0)
    m2 = GroupedMMModel(4, 512, 296)
    m2.load_state_dict(torch.load(buf, weights_only=True), assign=True)
    assert type(m2.weight) is Int8Tensor
    assert torch.equal(m2(x, offs).view(torch.int16), m(x, offs).view(torch.int16))


# ------------------------------------------------------------------------------------------------ PDL handoffs
@pytest.mark.parametrize("fmt", OPS)
def test_pdl_overlapped_equals_serialized(fmt):
    """offs from a torch cumsum, then grouped gate/up -> torch SiLU-mul (and, for int8 activations, a torch per-row
    quantizer) -> grouped down, parked behind a long kernel (tests/test_pdl_handoffs_gpu.py's stall head), against
    the same launches run one at a time, and as a graph."""
    lib = _lib()
    head = Head(lib)
    M, E, H, I = 300, 4, 2048, 1024
    g = ex.gen(32)
    qg = ex.randint(-127, 127, (E, 2 * I, H), g).to(torch.int8)
    qd = ex.randint(-127, 127, (E, H, I), g).to(torch.int8)
    sg = torch.rand(E, 2 * I, device=DEV) * 1e-3 + 1e-4
    sd = torch.rand(E, H, device=DEV) * 1e-3 + 1e-4
    x = (torch.randn(M, H, device=DEV) * 0.25).to(torch.bfloat16)
    counts = torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    ws2 = torch.zeros_like(ws)
    c = Chain(lib, f"cumsum offs -> grouped {fmt} gate/up -> silu-mul -> grouped {fmt} down")
    offs = c.out((E,), torch.int32)
    h = c.out((M, 2 * I), torch.bfloat16)
    a = c.out((M, I), torch.bfloat16)
    y = c.out((M, H), torch.bfloat16)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    if fmt == "int8wo":
        c.call("ao_int8_weight_grouped_mm", x, M, H, qg, sg, E, 2 * I, offs, h, ws, ws.numel())
        c.torch(lambda: torch.mul(F.silu(h[:, :I]), h[:, I:], out=a))
        c.call("ao_int8_weight_grouped_mm", a, M, I, qd, sd, E, H, offs, y, ws2, ws2.numel())
    else:
        xq = torch.randint(-127, 128, (M, H), device=DEV, dtype=torch.int8)
        xs = torch.rand(M, device=DEV) * 1e-2
        aq = c.out((M, I), torch.int8)
        sa = c.out((M, 1), torch.float32)
        c.call("ao_int8_dyn_grouped_mm", xq, xs, M, H, qg, sg, E, 2 * I, offs, h, ws, ws.numel())
        c.torch(lambda: torch.mul(F.silu(h[:, :I]), h[:, I:], out=a))
        c.torch(lambda: torch.div(a.float().abs().amax(dim=1, keepdim=True).clamp(min=1e-6), 127, out=sa))
        c.torch(lambda: aq.copy_(torch.round(a.float() / sa).clamp(-128, 127)))
        c.call("ao_int8_dyn_grouped_mm", aq, sa, M, I, qd, sd, E, H, offs, y, ws2, ws2.numel())
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
