"""The HQQ int4 solver (ao_b200/csrc/int4_hqq.cu) bit for bit against its restatement (tests/hqq_model.py).

The solver is deterministic (_rn intrinsics, fixed xor-butterfly warp sums, in-order double sums per block and one
fixed-order double reduction per iteration), so the restatement, run on the same device, matches it bit for bit,
including the fp32 state that bf16 rounding hides.  Through the C ABI the caller owns the workspace; it is filled with
0xFF bytes before the call and read back afterwards: fp32 scale[G] and zero[G], partial[nblocks] (the per-block error
sums of the last executed iteration) and Ctrl {best, stop, iters}.  So the iteration at which the solver stopped and
every fp32 zero point are pinned, not only the codes and the bf16 scale and zero.

Cases: g 32 / 64 / 128 / 256 x std 0.02, std 0.02 with outliers (Tier 1: the shrinkage relu is zero whatever the
last bits of powf), std 1 and std 2 (Tier 2: thousands of shrink-active elements, powf evaluated by torch on the same
device) x a small weight, 3 x 3g (9 groups: the last block has 7 empty warps), 1032 x 4096 (more than 256 blocks: the
strided sum in decide_kernel) and the Llama-3-8B qkv (6144 x 4096) and down (4096 x 14336) projections; plus special
groups (constants, +0 / -0 / mixed zeros, a huge outlier, ranges whose 15 / range passes the 2e4 clamp or overflows).
Also: the torch op, Int4TilePackedTo4dTensor.from_hp and quantize_ with padding, a CUDA graph replayed on weights
that stop at other iterations, a side stream, and the reference's own solves on shrink-active weights.
"""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import hqq_model as hm
from oracle import oracle as o

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda"
GS = (32, 64, 128, 256)
REGIMES = tuple(hm.STD)
SHAPES = {"small": lambda g: (64, 1024), "odd": lambda g: (3, 3 * g), "wide": lambda g: (1032, 4096)}
LLAMA = {"qkv": (6144, 4096), "down": (4096, 14336)}


@pytest.fixture(scope="module")
def lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_int4_hqq_workspace_bytes.restype = ctypes.c_size_t
    lib.ao_int4_hqq_workspace_bytes.argtypes = [ctypes.c_int] * 3
    lib.ao_int4_hqq_quantize.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                         ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


def _seed(g, regime, shape):
    return 1000 * GS.index(g) + 100 * REGIMES.index(regime) + list(SHAPES).index(shape)


def case_weight(g, regime, shape):
    N, K = SHAPES[shape](g) if shape in SHAPES else LLAMA[shape]
    return hm.weight(regime, N, K, _seed(g, regime, shape) if shape in SHAPES else 7 + N + K + g)


@functools.lru_cache(maxsize=None)
def restated(g, regime, shape, extra_iters=0):
    """The restatement of one matrix case on the GPU (cached: the premise test reuses it)."""
    w = hm.special_weight(g) if regime == "special" else case_weight(g, regime, shape)
    return hm.solve(w.to(DEV), g, extra_iters=extra_iters)


# ---------------------------------------------------------------------------------------------- C ABI
def abi_solve(lib, w, g, ws=None, poison=True):
    """ao_int4_hqq_quantize on the current stream; outputs (and the workspace, unless poison=False) filled with 0xFF
    first.  Returns the outputs and the solver state read back from the workspace."""
    N, K = w.shape
    G, nb, off_p, off_c = hm.workspace_layout(N, K, g)
    nbytes = lib.ao_int4_hqq_workspace_bytes(N, K, g)
    assert off_c + 16 <= nbytes
    if ws is None:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    if poison:
        ws.fill_(0xFF)
    q = torch.full((N, K), 0xFF, dtype=torch.uint8, device=DEV)
    s = torch.full((N, K // g), -1, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    z = torch.full((N, K // g), -1, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    rc = lib.ao_int4_hqq_quantize(w.data_ptr(), N, K, g, q.data_ptr(), s.data_ptr(), z.data_ptr(), ws.data_ptr(),
                                  ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.ao_b200_last_error()
    torch.cuda.synchronize()
    b = ws.cpu().numpy()
    return {"q": q, "scale": s, "zero": z, "s": b[: 4 * G].view(np.float32), "z": b[4 * G: 8 * G].view(np.float32),
            "partial": b[off_p: off_p + 8 * nb].view(np.float64), "best": b[off_c: off_c + 8].view(np.float64)[0],
            "stop": int(b[off_c + 8: off_c + 12].view(np.int32)[0]), "iters": int(b[off_c + 12: off_c + 16].view(np.int32)[0])}


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int16).numpy() if t.dtype == torch.bfloat16 else t.numpy()


def mismatches(out, ref):
    """Names of the outputs and state where the kernel and the restatement differ in any bit."""
    bad = [k for k in ("q", "scale", "zero") if not np.array_equal(_bits(out[k]), _bits(getattr(ref, k)))]
    if "s" in out:
        for k in ("s", "z"):
            if not np.array_equal(out[k].view(np.uint32), getattr(ref, k).cpu().numpy().view(np.uint32)):
                bad.append(k)
        if not np.array_equal(out["partial"].view(np.uint64), ref.partial.cpu().numpy().view(np.uint64)):
            bad.append("partial")
        if np.float64(out["best"]).view(np.uint64) != np.float64(ref.best).view(np.uint64):
            bad.append("best")
        bad += [k for k in ("stop", "iters") if out[k] != getattr(ref, k)]
    return bad


def describe(out, ref):
    msg = f"restated: iters {ref.iters} stop {ref.stop} tier1 {ref.tier1} active {ref.active}"
    if "s" in out:
        z = out["z"]
        zr = ref.z.cpu().numpy()
        msg += (f"; kernel: iters {out['iters']} stop {out['stop']}; fp32 zeros differ in {(z != zr).mean():.2%} of "
                f"groups, at most {np.abs(z - zr).max():.3g} steps")
    return msg


CASES = [(g, r, s) for g in GS for r in REGIMES for s in SHAPES]


@pytest.mark.parametrize("g,regime,shape", CASES, ids=[f"g{g}-{r}-{s}" for g, r, s in CASES])
def test_abi_bit_exact_with_workspace_state(lib, g, regime, shape):
    ref = restated(g, regime, shape)
    if regime.startswith("s002"):
        assert ref.tier1, ref.margin
    elif shape != "odd":
        assert min(ref.active) > 0, ref.active   # premise: the shrinkage step runs
    w = case_weight(g, regime, shape).to(DEV)
    out = abi_solve(lib, w, g)
    bad = mismatches(out, ref)
    assert not bad, f"{bad} differ; {describe(out, ref)}"


LLAMA_CASES = [(g, r, s) for s in LLAMA for g in GS for r in REGIMES]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("g,regime,shape", LLAMA_CASES, ids=[f"{s}-g{g}-{r}" for g, r, s in LLAMA_CASES])
def test_abi_bit_exact_llama_projections(lib, g, regime, shape):
    w = case_weight(g, regime, shape).to(DEV)
    ref = hm.solve(w, g)
    if regime.startswith("s002"):
        assert ref.tier1, ref.margin
    else:
        assert min(ref.active) > 0
    out = abi_solve(lib, w, g)
    bad = mismatches(out, ref)
    assert not bad, f"{bad} differ; {describe(out, ref)}"


@pytest.mark.parametrize("g", GS)
def test_abi_bit_exact_special_groups(lib, g):
    ref = restated(g, "special", None)
    s = ref.s.cpu().numpy()
    # premises: every special group but the outlier one clamps its scale, and 15 / range overflows in one of them
    assert all(s[i] == np.float32(2e4) for i, n in enumerate(hm.SPECIAL_GROUPS) if n != "huge_outlier")
    assert 15.0 / 2.0 ** -133 > np.finfo(np.float32).max
    w = hm.special_weight(g).to(DEV)
    out = abi_solve(lib, w, g)
    bad = mismatches(out, ref)
    assert not bad, f"{bad} differ; {describe(out, ref)}"
    assert np.isfinite(out["z"]).all() and np.isfinite(out["s"]).all()


def test_matrix_premises():
    """The matrix reaches at least three stop iterations, 20 among them and an early one; a stop one iteration late
    changes the fp32 zero points of some early-stopping and some 20-iteration cases.  (Where a solve stops early at a
    fixed point of the zero update, one more update changes no bit: there Ctrl.iters is what pins the stop.)"""
    stops, late_early, late_full = set(), 0, 0
    for g, regime, shape in CASES + [(g, "special", None) for g in GS]:
        r, rx = restated(g, regime, shape), restated(g, regime, shape, extra_iters=1)
        stops.add(r.iters)
        moved = not torch.equal(r.z.view(torch.int32), rx.z.view(torch.int32))
        late_early += moved and r.iters < hm.ITERS
        late_full += moved and r.iters == hm.ITERS
    assert len(stops) >= 3 and hm.ITERS in stops and min(stops) < hm.ITERS, sorted(stops)
    assert late_early >= 1 and late_full >= 1, (late_early, late_full)


def test_workspace_reuse_resets_ctrl(lib):
    """An early-stopping solve leaves Ctrl.stop = 1 and a small best in the workspace; a 20-iteration solve on the same
    workspace must still run all its iterations (init_kernel resets Ctrl)."""
    g = 32
    a, b = restated(g, "s002", "small"), restated(g, "s1", "small")
    assert a.stop == 1 and a.iters < hm.ITERS and b.iters == hm.ITERS
    N, K = SHAPES["small"](g)
    ws = torch.empty(lib.ao_int4_hqq_workspace_bytes(N, K, g), dtype=torch.uint8, device=DEV)
    out_a = abi_solve(lib, case_weight(g, "s002", "small").to(DEV), g, ws=ws)
    assert not mismatches(out_a, a)
    out_b = abi_solve(lib, case_weight(g, "s1", "small").to(DEV), g, ws=ws, poison=False)
    bad = mismatches(out_b, b)
    assert not bad, f"{bad} differ; {describe(out_b, b)}"


# ---------------------------------------------------------------------------------------------- torch op
OP_CASES = [(g, r, s) for g in GS for r in REGIMES for s in ("small", "odd")] + [(g, "special", None) for g in GS]


@pytest.mark.parametrize("g,regime,shape", OP_CASES, ids=[f"g{g}-{r}-{s}" for g, r, s in OP_CASES])
def test_torch_op_bit_exact(ops, g, regime, shape):
    ref = restated(g, regime, shape)
    w = hm.special_weight(g) if regime == "special" else case_weight(g, regime, shape)
    q, s, z = ops.int4_hqq_quantize(w.to(DEV), g)
    bad = mismatches({"q": q, "scale": s, "zero": z}, ref)
    assert not bad, f"{bad} differ; {describe({}, ref)}"


def _expected_tensor(ops, w, g):
    """qdata, scale_and_zero and dequantize() bits of the HQQ Int4TilePackedTo4dTensor of bf16 w ([N0, K0] or
    [E, N0, K0]), from the restated solve of the padded [E*N, K] weight."""
    lead, (N0, K0) = tuple(w.shape[:-2]), w.shape[-2:]
    N, K = -(-N0 // 8) * 8, -(-K0 // 1024) * 1024
    wp = F.pad(w, (0, K - K0, 0, N - N0)).reshape(-1, K).to(DEV)
    ref = hm.solve(wp, g)
    q = ref.q.to(torch.int32)
    qdata = ops.int4_pack_tile4d((q[:, ::2] << 4 | q[:, 1::2]).to(torch.uint8).contiguous(), 8)
    E = w.shape[0] if lead else 1
    s, z = o.bf16_bits(ref.scale).reshape(E, N, K // g), o.bf16_bits(ref.zero).reshape(E, N, K // g)
    sz = np.stack([o.pack_scales_and_zeros(s[e], z[e]) for e in range(E)])
    deq = hm.dequant_tinygemm_bits(ref.q, ref.scale, ref.zero, g).reshape(E, N, K)[:, :N0, :K0]
    if not lead:
        sz, deq = sz[0], deq[0]
    else:
        qdata = qdata.reshape(E, N // 8, *qdata.shape[1:])
    return ref, qdata, sz, deq


@pytest.mark.parametrize("g", [64, 128, 256])
@pytest.mark.parametrize("regime", ["s002_outlier", "s1"])
@pytest.mark.parametrize("lead", [(), (3,)], ids=["2d", "3d"])
def test_from_hp_hqq_bit_exact_with_padding(ops, g, regime, lead):
    from ao_b200.quantization import Int4TilePackedTo4dTensor
    from ao_b200.quantization.quantize_.workflows import Int4ChooseQParamsAlgorithm

    N0, K0 = 20, 768   # N not a multiple of 8, K not a multiple of 1024
    w = hm.weight(regime, int(np.prod(lead, dtype=int)) * N0, K0, g).reshape(*lead, N0, K0)
    t = Int4TilePackedTo4dTensor.from_hp(w.to(DEV), [1] * len(lead) + [1, g],
                                         int4_choose_qparams_algorithm=Int4ChooseQParamsAlgorithm.HQQ)
    ref, qdata, sz, deq = _expected_tensor(ops, w, g)
    if regime == "s1":
        assert min(ref.active) > 0
    assert torch.equal(t.qdata, qdata)
    assert np.array_equal(o.bf16_bits(t.scale_and_zero), sz)
    assert np.array_equal(o.bf16_bits(t.dequantize()), deq)


@pytest.mark.parametrize("g", [64, 128, 256])
def test_quantize_hqq_bit_exact_and_sqnr(ops, g):
    """quantize_ with Int4WeightOnlyConfig(int4_choose_qparams_algorithm="hqq") on a Linear(768 -> 20) with the default
    initialisation, as the reference's tensor test builds it; SQNR > 20 dB against the bf16 linear (its bar)."""
    from ao_b200.quantization import Int4WeightOnlyConfig, quantize_

    torch.manual_seed(g)
    lin = torch.nn.Linear(768, 20, bias=False, device=DEV, dtype=torch.bfloat16)
    w = lin.weight.detach().clone()
    quantize_(lin, Int4WeightOnlyConfig(group_size=g, int4_packing_format="tile_packed_to_4d",
                                        int4_choose_qparams_algorithm="hqq"))
    _, qdata, sz, deq = _expected_tensor(ops, w.cpu(), g)
    assert torch.equal(lin.weight.qdata, qdata)
    assert np.array_equal(o.bf16_bits(lin.weight.scale_and_zero), sz)
    assert np.array_equal(o.bf16_bits(lin.weight.dequantize()), deq)
    x = torch.randn(8, 768, device=DEV, dtype=torch.bfloat16)
    ref = x.float() @ w.float().t()
    sqnr = 20 * torch.log10(ref.norm() / (ref - lin(x).float()).norm()).item()
    assert sqnr > 20.0, sqnr


# ---------------------------------------------------------------------------------------------- graph and streams
def test_cuda_graph_replay_decides_the_stop_on_the_device(ops):
    """The op captured on a weight that stops early, replayed on weights that stop at other iterations: each replay
    matches its own restatement, and for the 20-iteration weight that differs from a solve cut at the captured
    weight's stop (what a stop decided on the host during capture would give)."""
    g = 32
    names = ["s002", "s1", "s002_outlier", "s2"]
    refs = {n: restated(g, n, "small") for n in names}
    assert refs["s002"].iters < hm.ITERS and refs["s1"].iters == hm.ITERS
    assert len({r.iters for r in refs.values()}) >= 3, {n: r.iters for n, r in refs.items()}
    cut = hm.solve(case_weight(g, "s1", "small").to(DEV), g, max_iters=refs["s002"].iters)
    assert mismatches({"q": cut.q, "scale": cut.scale, "zero": cut.zero}, refs["s1"])

    static_w = case_weight(g, "s002", "small").to(DEV)
    ops.int4_hqq_quantize(static_w, g)   # warm up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q, s, z = ops.int4_hqq_quantize(static_w, g)
    for n in names[1:] + names[:1]:
        static_w.copy_(case_weight(g, n, "small").to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        bad = mismatches({"q": q, "scale": s, "zero": z}, refs[n])
        assert not bad, f"replay on {n}: {bad} differ; {describe({}, refs[n])}"


def test_side_stream(ops):
    g = 128
    ref = restated(g, "s1", "small")
    w = case_weight(g, "s1", "small").to(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        q, s, z = ops.int4_hqq_quantize(w, g)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert not mismatches({"q": q, "scale": s, "zero": z}, ref)


# ---------------------------------------------------------------------------------------------- reference parity
@pytest.mark.parametrize("case", ["s002_g256", "s1_g32", "s1_g256", "s2_g128"])
def test_against_reference_on_shrink_fixture(ops, golden_dir, case):
    """The kernel against the reference's own fp32 CPU solves on g = 256 and shrink-active weights, within the
    solver bars of tests/hqq_model.py (measured and stated in tests/test_hqq_host.py)."""
    d = np.load(os.path.join(golden_dir, "int4_hqq_shrink.npz"))
    w_bits, g = d[f"{case}__w"], int(d[f"{case}__g"])
    q, s, z = ops.int4_hqq_quantize(o.bf16_tensor(w_bits).to(DEV), g)
    rep = hm.bar_report(w_bits, g, q.cpu().numpy(), o.bf16_bits(s), o.bf16_bits(z), d[f"{case}__q"], d[f"{case}__s"],
                        d[f"{case}__z"])
    assert hm.within_bars(rep), rep
