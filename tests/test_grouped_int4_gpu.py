"""torch._grouped_mm on 3-D int4 tile-packed expert weights (torch.ops.ao_b200.int4_tilepacked_grouped_mm and the
Int4TilePackedTo4dTensor handler) on the GPU.

* layout: 3-D from_hp against a golden fixture of the reference's CPU primitives (tinygemm and HQQ, with N and K
  padding); select(e) equals from_hp of expert e (the reference's test_select); 3-D HQQ is one solve over [E*N, K];
* the GEMM bit-exact under every forced stream-K grid, with exact operands per expert: token tiles 16 / 32 / 64 / 128,
  g 32 / 64 / 128 / 256, N tails, empty experts, E = 1, 8, 64 and 128, rows past offs[-1] left unwritten, malformed
  offs clamped, every expert empty; the workspace flags back to zero after each launch;
* the handler (torch._grouped_mm and F.grouped_mm): bit-identical to select + F.linear on exact operands, >= 60 dB
  against torch._grouped_mm on the dequantized weights, > 20 dB against the bf16 weights;
* a transformers-shaped MoE block quantized through FqnToConfig, its select loop against its grouped forward (and a
  tiny transformers Mixtral when transformers imports);
* a CUDA graph replayed with new routings; PDL handoffs behind a stall head against a serialized run; torch.compile.
tests/test_grouped_int4_host.py checks on the CPU that GROUPED_CASES reach every segment kind and token tile.
"""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import exact_operands as ex
import grouped_model as gm
import grouped_nvfp4_model as gnm

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda"

# (rows per expert, N_out, K, group size, rows past the last expert, forced grids; None = every grid up to the bound)
GROUPED_CASES = [
    ([13], 128, 1024, 32, 0, None),                                        # E = 1, N_MMA 16
    ([7, 9, 0, 12], 1001, 1024, 128, 3, (1, 2, 3, 5, 8, 13, 21, 34, 64, 132)),   # N tail 1001 -> 1008, N_MMA 32
    ([5, 0, 17, 0, 0, 3, 9, 0], 256, 2048, 256, 2, None),                 # E = 8, empty experts, N_MMA 64, g 256
    ([150, 0, 70, 1], 264, 1024, 32, 0, (1, 2, 3, 5, 8, 13, 21, 34)),     # N_MMA 128, two m-blocks, 8-row tail tile
    ([20, 30], 640, 2048, 128, 0, (3, 6, 7, 11)),                         # five n-tiles: CONTRIB, FULL and OWNER
    ([1, 0, 2, 1, 0, 0, 3, 1] * 16, 136, 1024, 64, 5, (1, 7, 50, 132)),   # E = 128, N_MMA 128
    ([0] * 30 + [16] + [0] * 33, 256, 2048, 32, 0, (1, 2, 5, 16, 64)),    # E = 64, one expert with every row
]
# offs values that are not cumulative row ends: the kernel clamps each into [end[e-1], M]
MALFORMED = [([9, 4, -3, 30, 12, 500], 40), ([-5, -1, 0, 3], 8), ([100, 200], 64)]


def gm_offs(rows):
    out, s = [], 0
    for r in rows:
        s += r
        out.append(s)
    return out


def grids_of(case_rows, N_out, K, tail, grids, sm):
    M = sum(case_rows) + tail
    p = gnm.plan(gm_offs(case_rows), M, N_out, K, grid=1, sm=sm, fmt="int4")
    top = min(p.U_bound, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


def pack_codes(q):
    """[R, K] codes -> [R, K/2] bytes, even k in the high nibble (from_hp's order)."""
    return ((q[:, 0::2] << 4) | q[:, 1::2]).to(torch.uint8).contiguous()


def int4_operands(E, N, K, g, gen):
    """Exact int4 expert weights: codes 0..15, s = odd * 2^-9, z = int * 2^-9, so bf16(fma(q - 8, s, z)) is W itself.
    Returns (W fp64 [E, N, K], qdata [E, N/8, K/128, 32, 4], scale_and_zero [E, K/g, N, 2])."""
    o = ex.ops()
    q = ex.randint(0, 15, (E, N, K), gen)
    s = ex.pick(ex.ODD, (E, N, K // g), gen) * 2.0**-9
    z = ex.randint(-24, 24, (E, N, K // g), gen).double() * 2.0**-9
    W = (q.double() - 8) * s.repeat_interleave(g, 2) + z.repeat_interleave(g, 2)
    qdata = o.int4_pack_tile4d(pack_codes(q.reshape(E * N, K)), 8).reshape(E, N // 8, K // 128, 32, 4)
    sz = torch.stack([s, z], -1).to(torch.bfloat16).transpose(1, 2).contiguous()
    return W, qdata, sz


class GroupedCase:
    """Exact operands: X in {-8..8} / 8 (bf16), int4 weights exact in bf16 (int4_operands); every product and sum is
    exact in fp32 (exact_operands.premise), so the output must equal the fp64 reference rounded once to bf16.  Weight
    rows past N_out are random too: a tail tile computes them and must not store them."""

    def __init__(self, offs, M, N_out, K, g, seed):
        E = len(offs)
        N = -(-N_out // 8) * 8
        gen = ex.gen(seed * 7919 + M * 31 + N_out * 7 + K + E + g)
        W, self.qdata, self.sz = int4_operands(E, N, K, g, gen)
        X = ex.randint(-8, 8, (M, K), gen).double() * 2.0**-3
        ex.premise(X, W.reshape(E * N, K))
        self.ends = gm.row_ends(offs, M)
        ref = torch.zeros(M, N_out, dtype=torch.float64, device=DEV)
        start = 0
        for e, end in enumerate(self.ends):
            if end > start:
                ref[start:end] = X[start:end] @ W[e, :N_out].t()
            start = end
        ex.fp32_exact(ref, "grouped int4: acc")
        self.valid = self.ends[-1] if self.ends else 0
        self.ref = ref.float().to(torch.bfloat16)[: self.valid]
        self.x = X.to(torch.bfloat16)
        self.offs = torch.tensor(offs, dtype=torch.int32, device=DEV)
        self.M, self.N, self.N_out, self.K, self.E, self.g = M, N, N_out, K, E, g

    def run(self):
        return torch.ops.ao_b200.int4_tilepacked_grouped_mm(self.x, self.qdata, self.g, self.sz, self.offs, self.N_out)


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
        p = gnm.plan(case.offs.tolist(), case.M, case.N_out, case.K, grid=G, sm=ex.sm_count(), fmt="int4")
        pytest.fail(f"{what} M={case.M} N_out={case.N_out} K={case.K} g={case.g} E={case.E} grid={G or 'default'}: "
                    f"{nb} wrong elements, {nr} flags left raised (U={p.U}, width {p.width}, device grid {p.G} of "
                    f"{p.G_host}); {len(wrong)} of {len(grids)} launches wrong")


@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)))
def test_grouped_grid_sweep_bit_exact(ops, set_ctas, ci):
    rows, N_out, K, g, tail, grids = GROUPED_CASES[ci]
    case = GroupedCase(gm_offs(rows), sum(rows) + tail, N_out, K, g, seed=ci)
    _sweep(ops, set_ctas, case, [None] + grids_of(rows, N_out, K, tail, grids, ex.sm_count()), f"case {ci}")


@pytest.mark.parametrize("mi", range(len(MALFORMED)))
def test_malformed_offs_are_clamped(ops, set_ctas, mi):
    offs, M = MALFORMED[mi]
    case = GroupedCase(offs, M, 1001, 1024, 32, seed=100 + mi)
    _sweep(ops, set_ctas, case, [None, 1, 3], f"malformed offs {offs}")


def test_all_experts_empty(ops, set_ctas):
    case = GroupedCase([0, 0, 0], 20, 256, 1024, 128, seed=7)
    flags = ops.debug_workspace(case.x).view(torch.int32)[:4096]
    for G in (0, 5):
        set_ctas(G)
        out = case.run()
        torch.cuda.synchronize()
        assert out.shape == (20, 256) and not bool(flags.ne(0).any())


def test_rows_past_the_last_expert_are_not_written():
    """Through the C ABI into a poisoned y: the rows from offs[-1] on keep their bytes, the rest is the reference."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    f = lib.ao_int4_tilepacked_grouped_mm
    f.argtypes = [vp, i32, i32, vp, vp, i32, i32, i32, i32, vp, vp, vp, ctypes.c_size_t, vp]
    case = GroupedCase([5, 5, 20], 37, 1001, 1024, 32, seed=3)
    y = torch.full((case.M, case.N_out), ex.POISON_BF16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    rc = f(case.x.data_ptr(), case.M, case.K, case.qdata.data_ptr(), case.sz.data_ptr(), case.g, case.E, case.N,
           case.N_out, case.offs.data_ptr(), y.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(y[: case.valid].view(torch.int16), case.ref.view(torch.int16))
    assert bool((y[case.valid:].view(torch.int16) == ex.POISON_BF16).all())


# ------------------------------------------------------------------------------------------------ layout
def _bf16_from_bits(a):
    return torch.from_numpy(a.view(np.int16)).view(torch.bfloat16).to(DEV)


def _golden():
    return np.load(os.path.join(HERE, "golden", "int4_3d.npz"))


@pytest.mark.parametrize("case", ["e3_n20_k768_g32", "e2_n40_k1024_g128", "e4_n13_k1000_g256"])
def test_3d_from_hp_matches_reference_golden(ops, case):
    from ao_b200.quantization import Int4TilePackedTo4dTensor

    d = _golden()
    w, g = _bf16_from_bits(d[f"{case}__w"]), int(d[f"{case}__g"])
    t = Int4TilePackedTo4dTensor.from_hp(w, [1, 1, g])
    E, Np, half = d[f"{case}__q"].shape
    assert t.shape == w.shape and t.qdata.shape == (E, Np // 8, half * 2 // 128, 32, 4)
    assert np.array_equal(t.scale_and_zero.view(torch.int16).cpu().numpy().view(np.uint16), d[f"{case}__sz"])
    q_u8 = torch.from_numpy(d[f"{case}__q"]).to(DEV).reshape(E * Np, half)
    assert torch.equal(t.qdata, ops.int4_pack_tile4d(q_u8, 8).reshape(t.qdata.shape))
    # the reference's test_select: expert e of the 3-D tensor is the 2-D tensor of w[e], bit for bit
    for e in range(E):
        a, b = t[e], Int4TilePackedTo4dTensor.from_hp(w[e].contiguous(), [1, g])
        assert a.shape == b.shape and list(a.block_size) == list(b.block_size) == [1, g]
        assert torch.equal(a.qdata, b.qdata) and torch.equal(a.scale_and_zero.view(torch.int16), b.scale_and_zero.view(torch.int16))
        assert torch.equal(a.dequantize().view(torch.int16), b.dequantize().view(torch.int16))
    assert torch.equal(t.dequantize().view(torch.int16), torch.stack([t[e].dequantize() for e in range(E)]).view(torch.int16))


def test_3d_hqq_is_one_solve_over_all_experts_and_matches_reference(ops):
    """3-D HQQ equals the 2-D HQQ of the [E*N_pad, K_pad] view bit for bit, and the reference's one 3-D call within the
    bars of the 2-D HQQ golden test (scales exact, codes at most one step apart, zeros within one step)."""
    from ao_b200.quantization import Int4TilePackedTo4dTensor
    from ao_b200.quantization.quantize_.workflows import Int4ChooseQParamsAlgorithm

    d = _golden()
    case = "hqq_e3_n20_k768_g64"
    w, g = _bf16_from_bits(d[f"{case}__w"]), int(d[f"{case}__g"])
    E, N0, K0 = w.shape
    t = Int4TilePackedTo4dTensor.from_hp(w, [1, 1, g], int4_choose_qparams_algorithm=Int4ChooseQParamsAlgorithm.HQQ)
    Np, Kp = -(-N0 // 8) * 8, 1024
    flat = F.pad(w, (0, Kp - K0, 0, Np - N0)).reshape(E * Np, Kp).contiguous()
    t2 = Int4TilePackedTo4dTensor.from_hp(flat, [1, g], int4_choose_qparams_algorithm=Int4ChooseQParamsAlgorithm.HQQ)
    assert torch.equal(t.qdata.reshape(t2.qdata.shape), t2.qdata)
    sz2 = t2.scale_and_zero.reshape(Kp // g, E, Np, 2).transpose(0, 1)
    assert torch.equal(t.scale_and_zero.view(torch.int16), sz2.contiguous().view(torch.int16))
    q, s, z = ops.int4_hqq_quantize(flat, g)
    q, s, z = q.cpu().numpy(), s.view(torch.int16).cpu().numpy().view(np.uint16), z.cpu().float().numpy()
    qr = d[f"{case}__q"].reshape(E * Np, Kp // 2)
    qr = np.stack([qr >> 4, qr & 15], -1).reshape(E * Np, Kp)
    sr = d[f"{case}__s"].reshape(E * Np, Kp // g)
    zr = torch.from_numpy(d[f"{case}__z"].reshape(E * Np, Kp // g).view(np.int16)).view(torch.bfloat16).float().numpy()
    srf = torch.from_numpy(sr.view(np.int16)).view(torch.bfloat16).float().numpy()
    assert np.array_equal(s, sr), "scale differs from the reference"
    diff = np.abs(q.astype(np.int32) - qr.astype(np.int32))
    assert diff.max() <= 1 and (diff != 0).mean() <= 1e-2, (diff.max(), (diff != 0).mean())
    steps = np.abs(z - zr) / srf
    assert (steps > 0.01).mean() <= 0.01 and steps.max() <= 1.0, steps.max()


# ------------------------------------------------------------------------------------------------ handler
def sqnr(ref, out):
    ref, out = ref.double(), out.double()
    dd = (ref - out).norm()
    return float("inf") if dd == 0 else float(20 * torch.log10(ref.norm() / dd))


def _cfg(g=32):
    from ao_b200.quantization import Int4WeightOnlyConfig

    return Int4WeightOnlyConfig(group_size=g, int4_packing_format="tile_packed_to_4d")


class GroupedMMModel(nn.Module):
    def __init__(self, E, K, N):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16) * 0.05)

    def forward(self, x, offs, functional=False):
        fn = F.grouped_mm if functional else torch._grouped_mm
        return fn(x, self.weight.transpose(-2, -1), offs=offs)


def _quantized(model, g=32):
    from ao_b200.quantization import FqnToConfig, quantize_

    m = copy.deepcopy(model)
    quantize_(m, FqnToConfig({"weight": _cfg(g)}), filter_fn=None)
    return m


@torch.no_grad()
@pytest.mark.parametrize("functional", [False, True])
def test_handler_exact_equals_select_and_linear(functional):
    from ao_b200.quantization import Int4TilePackedTo4dTensor

    gen = ex.gen(5)
    E, N0, K, g = 6, 1001, 2048, 128
    N = 1008
    rows = [3, 17, 0, 40, 1, 9]
    W, qdata, sz = int4_operands(E, N, K, g, gen)
    w = Int4TilePackedTo4dTensor(qdata, sz, [1, 1, g], torch.Size([E, N0, K]))
    X = ex.randint(-8, 8, (sum(rows), K), gen).double() * 2.0**-3
    x = X.to(torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device=DEV)
    fn = F.grouped_mm if functional else torch._grouped_mm
    y = fn(x, w.transpose(-2, -1), offs=offs)
    assert y.shape == (sum(rows), N0) and y.dtype == torch.bfloat16
    start = 0
    for e, end in enumerate(gm_offs(rows)):
        if end > start:
            ref = (X[start:end] @ W[e, :N0].t()).float().to(torch.bfloat16)
            assert torch.equal(y[start:end].view(torch.int16), ref.view(torch.int16)), f"expert {e}: fp64 reference"
            d = F.linear(x[start:end], w[e])
            assert torch.equal(d.view(torch.int16), y[start:end].view(torch.int16)), f"expert {e}: select + linear"
        start = end


@torch.no_grad()
@pytest.mark.parametrize("g", [32, 128])
def test_handler_random_against_dequantized_and_bf16(g):
    torch.manual_seed(3)
    E, K, N = 8, 768, 1000   # K and N padded by from_hp
    rows = [5, 0, 40, 1, 130, 0, 16, 9]
    ref = GroupedMMModel(E, K, N)
    m = _quantized(ref, g)
    x = torch.randn(sum(rows), K, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs(rows), device=DEV, dtype=torch.int32)
    for functional in (False, True):
        y = m(x, offs, functional)
        y_dq = torch._grouped_mm(x, m.weight.dequantize().transpose(-2, -1), offs=offs)
        y_bf = ref(x, offs)
        assert sqnr(y_dq, y) >= 60.0, sqnr(y_dq, y)
        assert sqnr(y_bf, y) > 20.0, sqnr(y_bf, y)


# ------------------------------------------------------------------------------------------------ MoE block
class MoEExperts(nn.Module):
    """The transformers layout of MoE experts: 3-D gate_up_proj [E, 2I, H] and down_proj [E, H, I]."""

    def __init__(self, E, H, I):
        super().__init__()
        self.gate_up_proj = nn.Parameter(torch.randn(E, 2 * I, H, device=DEV, dtype=torch.bfloat16) * H**-0.5)
        self.down_proj = nn.Parameter(torch.randn(E, H, I, device=DEV, dtype=torch.bfloat16) * I**-0.5)

    def forward_loop(self, x, rows):
        out, start = [], 0
        for e, r in enumerate(rows):
            if r:
                gate, up = F.linear(x[start:start + r], self.gate_up_proj[e]).chunk(2, dim=-1)
                out.append(F.linear(F.silu(gate) * up, self.down_proj[e]))
            start += r
        return torch.cat(out)

    def forward_grouped(self, x, offs):
        gate, up = torch._grouped_mm(x, self.gate_up_proj.transpose(-2, -1), offs=offs).chunk(2, dim=-1)
        return torch._grouped_mm(F.silu(gate) * up, self.down_proj.transpose(-2, -1), offs=offs)


class MoEBlock(nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.experts = MoEExperts(E, H, I)


def _quantize_moe(m):
    from ao_b200.quantization import FqnToConfig, Int4TilePackedTo4dTensor, quantize_

    quantize_(m, FqnToConfig({"experts.gate_up_proj": _cfg(), "experts.down_proj": _cfg()}), filter_fn=None)
    assert isinstance(m.experts.gate_up_proj, Int4TilePackedTo4dTensor)
    assert isinstance(m.experts.down_proj, Int4TilePackedTo4dTensor)


@torch.no_grad()
@pytest.mark.parametrize("E,H,I", [(2, 4096, 14336), (8, 2048, 768)], ids=["mixtral", "qwen3"])
def test_moe_block_loop_equals_grouped(E, H, I):
    torch.manual_seed(0)
    m = MoEBlock(E, H, I)
    q = copy.deepcopy(m)
    _quantize_moe(q)
    for rows in ([1] + [0] * (E - 1), [3] * E, [0, 37] + [11] * (E - 2)):
        x = torch.randn(sum(rows), H, device=DEV, dtype=torch.bfloat16)
        offs = torch.tensor(gm_offs(rows), dtype=torch.int32, device=DEV)
        ref = m.experts.forward_grouped(x, offs)
        a, b = q.experts.forward_loop(x, rows), q.experts.forward_grouped(x, offs)
        assert sqnr(a, b) >= 60.0, (rows, sqnr(a, b))
        assert sqnr(ref, b) > 15.0, (rows, sqnr(ref, b))


@torch.no_grad()
def test_tiny_transformers_moe_with_grouped_mm_experts():
    transformers = pytest.importorskip("transformers")
    from ao_b200.quantization import FqnToConfig, quantize_

    def model(impl):
        cfg = transformers.MixtralConfig(vocab_size=256, hidden_size=1024, intermediate_size=768, num_hidden_layers=2,
                                         num_attention_heads=8, num_key_value_heads=2, num_local_experts=8,
                                         num_experts_per_tok=2, experts_implementation=impl)
        torch.manual_seed(0)
        return transformers.MixtralForCausalLM(cfg).to(device=DEV, dtype=torch.bfloat16).eval()

    ref, ids = model("grouped_mm"), torch.randint(0, 256, (2, 24), device=DEV)
    want = ref(ids).logits
    outs = {}
    for impl in ("grouped_mm", "eager"):
        m = model(impl)
        m.load_state_dict(ref.state_dict())
        quantize_(m, FqnToConfig({r"re:.*experts\.(gate_up_proj|down_proj)": _cfg()}), filter_fn=None)
        outs[impl] = m(ids).logits
    assert sqnr(outs["eager"], outs["grouped_mm"]) >= 40.0, sqnr(outs["eager"], outs["grouped_mm"])
    assert sqnr(want, outs["grouped_mm"]) > 15.0, sqnr(want, outs["grouped_mm"])


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
def test_compile_fullgraph_through_the_handler():
    torch.manual_seed(2)
    m = _quantized(GroupedMMModel(4, 1024, 512))
    x = torch.randn(20, 1024, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor([3, 3, 12, 20], dtype=torch.int32, device=DEV)
    y = m(x, offs)
    yc = torch.compile(m, fullgraph=True, backend="aot_eager")(x, offs)
    assert torch.equal(y.view(torch.int16), yc.view(torch.int16))


def test_opcheck():
    gen = ex.gen(9)
    _, qdata, sz = int4_operands(3, 136, 1024, 32, gen)
    x = torch.randn(10, 1024, device=DEV).to(torch.bfloat16)
    offs = torch.tensor([2, 5, 10], dtype=torch.int32, device=DEV)
    torch.library.opcheck(torch.ops.ao_b200.int4_tilepacked_grouped_mm.default, (x, qdata, 32, sz, offs, 130),
                          test_utils=("test_schema", "test_faketensor"))


# ------------------------------------------------------------------------------------------------ PDL handoffs
# The stall head and chain runner of tests/test_pdl_handoffs_gpu.py: the chain's kernels park behind a long
# fp8_quantize_rowwise, outputs poisoned with 0xFF, compared byte for byte with the same launches run one at a time.
SIGS = {"ao_fp8_quantize_rowwise": "piippp", "ao_int4_tilepacked_grouped_mm": "piippiiiippzp"}
_CT = {"p": ctypes.c_void_p, "i": ctypes.c_int, "f": ctypes.c_float, "z": ctypes.c_size_t}


@pytest.fixture(scope="module")
def lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    for name, sig in SIGS.items():
        getattr(lib, name).argtypes = [_CT[c] for c in sig]
    return lib


class Head:
    """fp8_quantize_rowwise on [8, 2^25] bf16 rows: one CTA per row on 8 SMs, milliseconds long, triggers its
    dependents at entry."""

    M, K = 8, 1 << 25

    def __init__(self, lib):
        self.lib = lib
        g = torch.Generator(device=DEV).manual_seed(99)
        self.x = torch.randn(self.M, self.K, device=DEV, generator=g).to(torch.bfloat16)
        self.q = torch.empty(self.M, self.K, dtype=torch.uint8, device=DEV)
        self.s = torch.empty(self.M, dtype=torch.float32, device=DEV)

    def __call__(self):
        st = torch.cuda.current_stream().cuda_stream
        assert self.lib.ao_fp8_quantize_rowwise(self.x.data_ptr(), self.M, self.K, self.q.data_ptr(), self.s.data_ptr(), st) == 0


@pytest.fixture(scope="module")
def head(lib):
    return Head(lib)


class Chain:
    def __init__(self, lib, name):
        self.lib, self.name, self.outs, self.steps = lib, name, [], []

    def out(self, shape, dtype):
        t = torch.empty(shape, dtype=dtype, device=DEV)
        self.outs.append(t)
        return t

    def call(self, name, *args):
        self.steps.append((name, args))

    def torch(self, fn):
        self.steps.append((fn, ()))

    def run(self, head=None, sync_each=False):
        if head is not None:
            head()
        for name, args in self.steps:
            if callable(name):
                name()
            else:
                conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
                rc = getattr(self.lib, name)(*conv, torch.cuda.current_stream().cuda_stream)
                assert rc == 0, f"{self.name}: {name}: {self.lib.ao_b200_last_error()}"
            if sync_each:
                torch.cuda.synchronize()

    def result(self, head=None, sync_each=False):
        for t in self.outs:
            t.view(torch.uint8).fill_(0xFF)
        torch.cuda.synchronize()
        self.run(head, sync_each)
        torch.cuda.synchronize()
        return [t.clone() for t in self.outs]


def _gemm_args(x, M, K, qd, sz, g, E, N, N_out, offs, y, ws):
    return (x, M, K, qd, sz, g, E, N, N_out, offs, y, ws, ws.numel())


def offs_chain(lib, M=300, E=4, N=1008, N_out=1001, K=2048, g=32):
    """offs from a torch cumsum, read by the grouped int4 GEMM."""
    c = Chain(lib, "cumsum offs -> grouped int4")
    _, qd, sz = int4_operands(E, N, K, g, ex.gen(31))
    x = (torch.randn(M, K, device=DEV) * 0.5).to(torch.bfloat16)
    counts = torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    offs = c.out((E,), torch.int32)
    y = c.out((M, N_out), torch.bfloat16)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    c.call("ao_int4_tilepacked_grouped_mm", *_gemm_args(x, M, K, qd, sz, g, E, N, N_out, offs, y, ws))
    return c


def mlp_chain(lib, M=64, E=4, H=2048, I=1024, g=32):
    """grouped gate/up -> torch SiLU-mul -> grouped down."""
    c = Chain(lib, "grouped gate/up -> silu-mul -> grouped down")
    _, qg, szg = int4_operands(E, 2 * I, H, g, ex.gen(32))
    _, qdn, szd = int4_operands(E, H, I, g, ex.gen(33))
    x = (torch.randn(M, H, device=DEV) * 0.25).to(torch.bfloat16)
    offs = torch.tensor(gm_offs([10, 30, 0, 24]), dtype=torch.int32, device=DEV)
    ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)
    ws2 = torch.zeros_like(ws)
    h = c.out((M, 2 * I), torch.bfloat16)
    a = c.out((M, I), torch.bfloat16)
    y = c.out((M, H), torch.bfloat16)
    c.call("ao_int4_tilepacked_grouped_mm", *_gemm_args(x, M, H, qg, szg, g, E, 2 * I, 2 * I, offs, h, ws))
    c.torch(lambda: torch.mul(F.silu(h[:, :I]), h[:, I:], out=a))
    c.call("ao_int4_tilepacked_grouped_mm", *_gemm_args(a, M, I, qdn, szd, g, E, H, H, offs, y, ws2))
    return c


@pytest.mark.parametrize("make", [offs_chain, mlp_chain], ids=["offs", "mlp"])
def test_pdl_overlapped_equals_serialized(lib, head, make):
    c = make(lib)
    want = c.result(sync_each=True)
    got = c.result(head=head)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{c.name}: output {i} differs (eager)"
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
    for i, (a, b) in enumerate(zip(c.outs, want)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{c.name}: output {i} differs (graph replay)"


@torch.no_grad()
def test_quantize_3d_then_grouped_forward_at_once(head):
    """quantize_ on 3-D expert weights behind the stall head, followed at once by the first grouped call, against the
    same with a sync between them."""
    from ao_b200.quantization import FqnToConfig, quantize_

    torch.manual_seed(4)
    base = GroupedMMModel(8, 4096, 1024)
    x = torch.randn(64, 4096, device=DEV, dtype=torch.bfloat16)
    offs = torch.tensor(gm_offs([8] * 8), dtype=torch.int32, device=DEV)
    a, b = copy.deepcopy(base), copy.deepcopy(base)
    torch.cuda.synchronize()
    quantize_(b, FqnToConfig({"weight": _cfg()}), filter_fn=None)
    torch.cuda.synchronize()
    want = b(x, offs)
    torch.cuda.synchronize()
    head()
    quantize_(a, FqnToConfig({"weight": _cfg()}), filter_fn=None)
    got = a(x, offs)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
