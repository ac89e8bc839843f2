"""Every quantized linear checked bit for bit, element by element, under every stream-K split the kernel allows.

The operands come from tests/exact_operands.py: codes and scales for which fp32 accumulation is exact in any order,
so the kernel's bf16 output must equal the fp64 reference rounded once to bf16.  One wrong element, one wrong partial
of an owner's gather or one unwritten ragged token fails the test; an SQNR bar cannot see those.  The CTA count is
forced through torch.ops.ao_b200.debug_set_streamk_ctas, so the split patterns do not depend on the card's SM count.
tests/test_streamk_plan.py checks on the CPU that GRID_CASES reach every segment pattern and gather group.
"""
import ctypes
import os

import pytest
import torch

import exact_operands as ex
import streamk_model as sk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OPS = ("int4", "int8_dyn", "int8_mm_i32", "fp8", "mxfp8", "nvfp4", "nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts", "int8wo",
       "fp8wo", "mxfp4", "fp8_blockwise", "fp8_sparse")
OP_FORMAT = {"int4": "int4", "int8_dyn": "int8", "int8_mm_i32": "int8", "fp8": "fp8", "mxfp8": "mxfp8", "nvfp4": "nvfp4",
             "nvfp4w": "nvfp4", "nvfp4w_xs": "nvfp4", "nvfp4w_rowpts": "nvfp4", "int8wo": "int8wo", "fp8wo": "fp8wo",
             "mxfp4": "mxfp4", "fp8_blockwise": "fp8_blockwise", "fp8_sparse": "fp8_sparse"}

# (M, N, K, forced grids; None = every grid from 1 to min(units, SMs))
#   * N = 256, K = 4096: every token-tile width and two m-blocks, all grids
#   * N = 128, K = 16384: one tile per m-block split over up to 127 CTAs (owner gathers of more than 32 and 64)
#   * N = 640, K = 1024: five tiles, so that one CTA holds CONTRIB, FULL and OWNER segments
GRID_CASES = ([(M, 256, 4096, None) for M in (1, 17, 33, 65, 129)]
              + [(M, 128, 16384, (33, 64, 65, 127, 128)) for M in (1, 32, 64, 128)]
              + [(M, 640, 1024, (3, 6, 7, 11)) for M in (16, 32, 64, 128)])


def shape_supported(op, M, N, K):
    fmt = OP_FORMAT[op]
    if fmt == "int4":
        return K % 1024 == 0 and N % 8 == 0
    if fmt == "nvfp4":
        return K % (256 if op == "nvfp4" else 128) == 0 and N % 16 == 0
    if fmt in ("mxfp8", "mxfp4"):
        return K % 32 == 0
    if fmt in ("int8wo", "fp8wo"):
        return K % 16 == 0
    if fmt == "fp8":
        return K % 16 == 0 and N % 16 == 0
    if fmt == "fp8_blockwise":
        return K % 128 == 0 and N % 128 == 0
    if fmt == "fp8_sparse":
        return K % 32 == 0 and N % 16 == 0
    return K % 16 == 0 and N % 8 == 0


def grids_of(fmt, M, N, K, grids, sm=132):
    U = sk.plan(fmt, M, N, K, grid=1).U
    top = min(U, sm)
    return list(range(1, top + 1)) if grids is None else [G for G in grids if G <= top]


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    """Forces the stream-K CTA count; always restores the heuristic."""
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def _flags(ops, like):
    return ops.debug_workspace(like).view(torch.int32)[:4096]   # the 16 KiB flag area


def _explain(case, y, G, M=None):
    mm = ex.first_mismatch(case, y, M)
    p = sk.plan(case.fmt, case.M if M is None else M, case.n_plan, case.K, grid=G, sm=ex.sm_count())
    if mm is None:
        return f"{case.op}: outputs match but the workspace flags were left raised ({p.describe(0, 0)})"
    m, n, got, want, nbad = mm
    return (f"{case.op} M={case.M if M is None else M} N={case.N} K={case.K} grid={G or 'default'}: {nbad} wrong elements, "
            f"first at (m={m}, n={n}) got {got!r} want {want!r}; {p.describe(m, n)}")


def _sweep(ops, set_ctas, case, grids, Ms=None):
    """Runs `case` at every grid (or every token count at the default grid), compares bits and checks the flag area on
    the device, and synchronises once."""
    flags = _flags(ops, case.ref_full)
    runs = [(G, M) for G in grids for M in (Ms or [None])]
    bad = torch.zeros(len(runs), dtype=torch.int64, device=ex.DEV)
    raised = torch.zeros(len(runs), dtype=torch.int64, device=ex.DEV)
    for i, (G, M) in enumerate(runs):
        set_ctas(G or 0)
        y = case.run(M)
        bad[i] = (case.bits(y) != case.bits(case.ref(M))).sum()
        raised[i] = flags.ne(0).sum()
        case.scrub(y)
    set_ctas(0)
    bad, raised = bad.cpu(), raised.cpu()
    for i, (G, M) in enumerate(runs):
        if bad[i] or raised[i]:
            set_ctas(G or 0)
            y = case.run(M)
            set_ctas(0)
            pytest.fail(_explain(case, y, G, M) + f" [{int((bad != 0).sum())} of {len(runs)} launches wrong]")


@pytest.mark.parametrize("op", OPS)
def test_grid_sweep_bit_exact(ops, set_ctas, op):
    sm = ex.sm_count()
    for M, N, K, grids in GRID_CASES:
        if not shape_supported(op, M, N, K):
            continue
        case = ex.build(op, M, N, K)
        _sweep(ops, set_ctas, case, grids_of(OP_FORMAT[op], M, N, K, grids, sm))


@pytest.mark.parametrize("op", OPS)
def test_ragged_token_counts_bit_exact(ops, set_ctas, op):
    """M = 1..130, 255, 256, 257 at the default grid: every token-tile width, every masked column of a tile."""
    case = ex.build(op, 257, 256, 2048, seed=1)
    _sweep(ops, set_ctas, case, [None], Ms=list(range(1, 131)) + [255, 256, 257])


TAILS = ([("int4", 7, n, 2048, n_out) for n, n_out in ((8, 8), (128, 120), (136, 136), (272, 264))]
         + [("int4", 40, 136, 1024, 136)]
         + [(op, M, n, 1024, None) for op in ("int8_dyn", "int8_mm_i32") for n in (8, 136) for M in (5, 40)]
         + [(op, M, n, 1024, None) for op in ("fp8", "nvfp4", "nvfp4w_xs") for n in (16, 144) for M in (5, 40)]
         + [(op, M, 256, k, None) for op in ("int8_dyn", "int8_mm_i32", "fp8") for k in (16, 144, 1040) for M in (9, 70)]
         + [(op, M, n, 1024, None) for op in ("int8wo", "fp8wo", "mxfp4") for n in (77, 200) for M in (5, 40)]
         + [(op, M, 256, k, None) for op in ("int8wo", "fp8wo") for k in (16, 144, 1040) for M in (9, 70)]
         + [("mxfp4", M, 256, k, None) for k in (32, 160, 1056) for M in (9, 70)]
         + [("fp8_sparse", M, n, 1024, None) for n in (48, 80, 208) for M in (5, 40)]
         + [("fp8_sparse", M, 256, k, None) for k in (32, 160, 1056, 4128) for M in (9, 70)])


@pytest.mark.parametrize("op,M,N,K,n_out", TAILS)
def test_feature_and_k_tails_bit_exact(ops, set_ctas, op, M, N, K, n_out):
    """Output-feature tails (a partial 128-row tile, int4 n_out < N) and K tails (TMA zero fill of the last chunk);
    the mxfp8 K tails are in test_parity_holes_gpu.py::test_k_tail_is_zero_filled.  2:4-sparse e4m3: the metadata
    rows past N (up to the next 64) and the metadata words of a K-tail chunk past K are sanitized, not used.
    Blockwise e4m3 has no tails: its K and N are multiples of 128."""
    case = ex.build(op, M, N, K, seed=2, n_out=n_out)
    U = sk.plan(case.fmt, M, case.n_plan, K, grid=1).U
    _sweep(ops, set_ctas, case, sorted({None, 1, min(U, ex.sm_count())}, key=lambda g: g or 0))


def test_mixed_formats_and_grids_in_one_cuda_graph(ops, set_ctas):
    """int4, nvfp4, int8, fp8, mxfp8, the weight-only int8 and fp8, mxfp4, blockwise fp8, 2:4-sparse fp8 and int4
    again back to back in one CUDA graph, PDL on, each under its own forced grid; a large grid followed by a small one
    would expose a flag the owners did not re-arm.  Two replays."""
    M, N, K = 20, 384, 4096
    plan = [("int4", 96), ("nvfp4", 5), ("int8_dyn", 80), ("fp8", 3), ("mxfp8", 64), ("int8wo", 90), ("fp8wo", 4),
            ("mxfp4", 70), ("fp8_blockwise", 6), ("fp8_sparse", 90), ("int4", 7)]
    cases = [ex.build(op, M, N, K, seed=3 + i) for i, (op, _) in enumerate(plan)]
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for c, (_, G) in zip(cases, plan):   # warm-up on the capture stream: creates its workspace outside the capture
            set_ctas(G)
            c.run()
        flags = _flags(ops, cases[0].ref_full)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        outs = []
        for c, (_, G) in zip(cases, plan):
            set_ctas(G)
            outs.append(c.run())
    set_ctas(0)
    for replay in range(2):
        for c, y in zip(cases, outs):
            c.scrub(y)
        g.replay()
        torch.cuda.synchronize()
        for c, y, (_, G) in zip(cases, outs, plan):
            assert torch.equal(c.bits(y), c.bits(c.ref())), f"replay {replay}: " + _explain(c, y, G)
        assert not bool(flags.ne(0).any()), f"replay {replay}: flags left raised in the capture stream's workspace"


def _slab_workspace_bytes(K, rows):
    # restates the slab offset of block_scaled() in ao_b200/csrc/lowp_linear.cu: the partial slots take at most
    # SMs x 128 x 128 words behind the 64 KiB flag area, and the bf16 activation slab starts on the next MiB
    act_off = (64 * 1024 + ex.sm_count() * 128 * 128 * 4 + (1 << 20) - 1) & ~((1 << 20) - 1)
    return act_off + rows * K * 2


@pytest.mark.parametrize("rows", [37, 128])
@pytest.mark.parametrize("M", [100, 129, 300])
def test_block_scaled_activation_slabs(M, rows):
    """ao_mxfp8_linear / ao_nvfp4_linear through ctypes with a workspace that holds `rows` activation rows: slab
    boundaries at multiples of 37 or 128 tokens, not of the token-tile width."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.ao_mxfp8_linear.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, sz, vp]
    lib.ao_nvfp4_linear.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, i32, vp, vp, vp, sz, vp]
    N, K = 256, 1024
    ws_bytes = _slab_workspace_bytes(K, rows)
    stream = torch.cuda.current_stream().cuda_stream
    for op in ("mxfp8", "nvfp4"):
        case = ex.build(op, M, N, K, seed=4)
        r = case.raw
        xs = ex.to_blocked(r["x_bytes"])
        ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=ex.DEV)
        y = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=ex.DEV)
        if op == "mxfp8":
            rc = lib.ao_mxfp8_linear(r["xq"].data_ptr(), xs.data_ptr(), M, K, r["wq"].data_ptr(), r["w_blocked"].data_ptr(), N,
                                     r["bias"].data_ptr(), y.data_ptr(), ws.data_ptr(), ws_bytes, stream)
        else:
            rc = lib.ao_nvfp4_linear(r["xq"].data_ptr(), xs.data_ptr(), r["a_pts"].data_ptr(), M, K, r["wq"].data_ptr(),
                                     r["w_blocked"].data_ptr(), r["b_pts"].data_ptr(), N, r["bias"].data_ptr(), y.data_ptr(),
                                     ws.data_ptr(), ws_bytes, stream)
        assert rc == 0, lib.ao_b200_last_error()
        torch.cuda.synchronize()
        assert torch.equal(case.bits(y), case.bits(case.ref())), _explain(case, y, None) + f" (slabs of {rows} rows)"
        assert not bool(ws[:16384].ne(0).any()), "flags left raised"


def test_nvfp4_every_weight_scale_byte_bit_exact(ops):
    """Both nvfp4 kernels with weights whose blocks use byte b and its neighbour, for every byte 0x00..0x7E: the zero
    byte and the e4m3 subnormals 0x01..0x07 included.  0x7F (NaN) and the sign-bit bytes are left out: no quantizer in
    this project or in the one it follows writes them."""
    N, K, M = 256, 1024, 24
    g = ex.gen(5)
    runs = []
    for byte in range(0x7F):
        nb = byte + 1 if byte < 0x7E else byte - 1
        wb = torch.where(ex.randint(0, 1, (N, K // 16), g).bool(), byte, nb)
        for op in ("nvfp4", "nvfp4w_xs"):
            case = ex.build(op, M, N, K, seed=byte, w_bytes=wb)
            y = case.run()
            runs.append((byte, op, case, y, (case.bits(y) != case.bits(case.ref())).sum()))
    failed = [(f"0x{byte:02X}", op) for byte, op, _, _, nbad in runs if int(nbad)]
    assert not failed, f"wrong outputs for weight scale bytes {failed}; first: " + _explain(
        next(c for b, o, c, y, n in runs if int(n)), next(y for b, o, c, y, n in runs if int(n)), None)


def _e2m1_rtne(v):
    """Round to the nearest e2m1 value, ties to even; returns the 4-bit codes."""
    a = v.abs()
    idx = ((a > 0.25).int() + (a >= 0.75).int() + (a > 1.25).int() + (a >= 1.75).int() + (a > 2.5).int()
           + (a >= 3.5).int() + (a > 5.0).int())
    return idx | ((v < 0).int() << 3)


def _te_recipe_nvfp4(w):
    """The TransformerEngine NVFP4 weight recipe (1 x 16 blocks), restated with torch ops: S_enc = 448 * 6 / amax,
    block scale = e4m3(min(block_amax * (S_enc / 6), 448)) with NO lower clamp (blocks that underflow e4m3 get the
    zero byte, small blocks subnormal bytes), encode = 1 / (scale / S_enc) capped at FLT_MAX, codes = RTNE e2m1 of
    the clamped product (a zero-scale block saturates to +-6); per-tensor scale 1 / S_enc."""
    N, K = w.shape
    wf = w.float()
    amax = wf.abs().max()
    s_enc = torch.clamp(torch.full_like(amax, 448.0 * 6.0) / amax, max=torch.finfo(torch.float32).max)
    block_amax = wf.reshape(N, K // 16, 16).abs().amax(-1)
    scale = (block_amax * (s_enc * (1.0 / 6.0))).clamp(max=448.0).to(torch.float8_e4m3fn)
    enc = (1.0 / (scale.float() * (1.0 / s_enc))).clamp(max=torch.finfo(torch.float32).max)
    scaled = (wf.reshape(N, K // 16, 16) * enc.unsqueeze(-1)).reshape(N, K).clamp(-6.0, 6.0)
    return ex.pack_e2m1(_e2m1_rtne(scaled).long()), scale.view(torch.uint8), (1.0 / s_enc).reshape(())


def test_nvfp4_tensor_from_unclamped_recipe_matches_its_dequantization(ops):
    """An NVFP4Tensor built outside this project's quantizer (the TransformerEngine recipe has no lower clamp on
    the block scale): F.linear through the kernel must equal F.linear on w.dequantize() in fp32 up to summation order
    and the bf16 output rounding, >= 70 dB as in test_lowp_gpu.py::test_block_scaled_linears_vs_fp32_dequant_matmul.
    The rows span seven decades, so every output feature is normalised to unit norm first: the features whose blocks
    have subnormal scales weigh as much as the large ones.  Features whose blocks all have the zero scale must be
    exact zeros."""
    from ao_b200.prototype.mx_formats import NVFP4Tensor

    N, K, M = 256, 1024, 8
    g = ex.gen(6)
    # rows 1 .. 1e-7 of the largest: normal, subnormal and zero block scales
    w = (torch.randn(N, K, device=ex.DEV, generator=g) * torch.logspace(0, -7, N, device=ex.DEV).unsqueeze(1)).to(torch.bfloat16)
    q, sb, pts = _te_recipe_nvfp4(w)
    assert bool((sb == 0).any()) and bool(((sb > 0) & (sb < 8)).any()), "premise: the recipe wrote zero and subnormal scales"
    wt = NVFP4Tensor(q, ex.to_blocked(sb), 16, torch.bfloat16, per_tensor_scale=pts, is_swizzled_scales=True)
    x = torch.randn(M, K, device=ex.DEV, generator=g).to(torch.bfloat16)
    y = torch.nn.functional.linear(x, wt).double()
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = torch.nn.functional.linear(x.float(), wt.dequantize(torch.float32)).to(torch.bfloat16).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    norm = ref.norm(dim=0)
    zero = norm == 0
    assert bool((y[:, zero] == 0).all()), f"features {zero.nonzero().flatten().tolist()[:8]}... must be exact zeros"
    rel = (y[:, ~zero] - ref[:, ~zero]) / norm[~zero]
    db = float(20 * torch.log10(torch.sqrt(torch.tensor(float((~zero).sum()), dtype=torch.float64)) / rel.norm()))
    worst = int(rel.norm(dim=0).argmax())
    assert db >= 70.0, f"{db:.1f} dB; worst feature {int((~zero).nonzero()[worst])}, scale bytes {sorted(set(sb[int((~zero).nonzero()[worst])].tolist()))[:8]}"
