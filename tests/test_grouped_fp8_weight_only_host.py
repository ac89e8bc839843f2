"""CPU tests of the float8 weight-only expert GEMM (torch._grouped_mm on 3-D Float8Tensor weights without
act_quant_kwargs, torch.ops.ao_b200.fp8_weight_grouped_mm):

* the Meta shape, the op schema and the C-ABI argument checks (before any CUDA call);
* the grouped schedule at this format's token tiles (16 .. 128) with N tails, and a model of the boxes
  Fp8WoFmt::issue_w_rows loads: weight rows and scales from element e*N + 128t of the stacked [E*N] maps;
* the package's 3-D quantizer and a numpy restatement of the recipe against the reference's fixture;
* select and transpose of a 3-D Float8Tensor, the handler's rejections and the config's 3-D rules;
* ts_gemm_kernel<Grouped<Fp8WoFmt>, N> exists for every token tile, has no stack and fits one CTA per SM.
"""
import ctypes
import io
import json
import logging
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import grouped_nvfp4_model as gnm
import streamk_model as sk
from test_decode_residency import LIB, RESERVED_PER_CTA, SMEM_PER_SM
from test_float8_weight_only_host import bf16_round, dequantize_ref, f32, same_bits_or_both_nan, same_codes
from test_float8_weight_only_host import within_one_step_of_the_sum
from test_grouped_schedule import _cum, _offs_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
E4M3 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
def test_meta_shape_and_schema():
    import ao_b200  # noqa: F401

    x = torch.empty(37, 160, dtype=torch.bfloat16, device="meta")
    wq = torch.empty(8, 200, 160, dtype=E4M3, device="meta")
    y = torch.ops.ao_b200.fp8_weight_grouped_mm(x, wq, torch.empty(8, 200, device="meta"),
                                                torch.empty(8, dtype=torch.int32, device="meta"))
    assert y.shape == (37, 200) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(torch.ops.ao_b200.fp8_weight_grouped_mm.default._schema).endswith(
        "(Tensor x, Tensor wq, Tensor w_scale, Tensor offs) -> Tensor")


def test_c_abi_argument_validation_without_gpu():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_fp8_weight_grouped_mm
    f.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15   # host addresses stand in for device ones: never dereferenced
    one = ctypes.c_void_p(a)

    def call(M=4, K=256, E=8, N=200, ptrs=(one,) * 6):
        x, wq, ws, offs, y, work = ptrs
        return f(x, M, K, wq, ws, E, N, offs, y, work, 1 << 20, None)

    err = lib.ao_b200_last_error
    assert call(K=200) == -1 and b"K=200" in err()
    assert call(E=0) == -1 and b"E=0" in err()
    assert call(E=1025) == -1 and b"E=1025" in err()
    assert call(E=1024, N=2**21) == -1 and b"int32" in err()
    assert call(M=-1) == -1 and b"bad sizes" in err()
    assert call(N=0) == -1 and b"bad sizes" in err()
    for i in range(6):
        ptrs = [one] * 6
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in err(), i
    assert call(ptrs=(ctypes.c_void_p(a + 8),) + (one,) * 5) == -1 and b"x must be 16-byte aligned" in err()
    assert call(ptrs=(one, one, ctypes.c_void_p(a + 4), one, one, one)) == -1 and b"w_scale must be 16-byte" in err()
    # N % 8 == 0: every scale box starts on 32 bytes; N tails past 128 are valid (the checks pass up to the null pointer)
    assert call(N=77) == -1 and b"N=77" in err()
    assert call(N=204) == -1 and b"N=204" in err()
    assert call(N=136, ptrs=(one,) * 5 + (None,)) == -1 and b"null pointer" in err()
    # no tokens: nothing to do, nothing dereferenced, no CUDA call (this process has no device)
    assert call(M=0, ptrs=(None,) * 6) == 0


# ------------------------------------------------------------------------------------------------ schedule
def plan(offs, M, N, K, grid=None, sm=132):
    """The grouped split of one launch: the nvfp4 plan, whose token tiles (16 .. 128) are this format's too, with the
    K tail of the 8-bit kinds (ceil(K / 128) chunks, zero-filled)."""
    assert sk.WIDTHS["mxfp8"] == sk.WIDTHS["nvfp4"] and sk.k_chunks("mxfp8", K) == -(-K // 128)
    return gnm.plan(offs, M, N, K, grid=grid, sm=sm, fmt="fp8wo")


def _check(offs, M, N, K, grid, sm=132):
    p = plan(offs, M, N, K, grid, sm)
    E = len(offs)
    assert p.n_tiles == -(-N // sk.ROWS)
    end = p.ends[-1]
    assert 0 <= end <= M
    assert p.G <= p.G_host and p.U <= p.U_bound and p.G <= max(p.U, 0)
    if p.U == 0:
        assert p.G == 0 and end == 0
        return p
    covered = [[0] * p.n_tiles for _ in range(end)]
    for t in range(p.U // p.KT):
        e, row0, row_end, n_tile = p.tile(t)
        assert 0 <= e < E and (p.ends[e - 1] if e > 0 else 0) <= row0 < p.ends[e] == row_end <= M
        # the weight box and the scale box start at the same element e*N + 128t, inside expert e's rows; a tail past
        # N reads the next expert's rows (or the zero fill), whose features are >= N and never stored
        row = e * N + n_tile * sk.ROWS
        assert e * N <= row < (e + 1) * N and row < 2**31
        for m in range(row0, min(row0 + p.width, row_end)):
            covered[m][n_tile] += 1
    assert all(c == [1] * p.n_tiles for c in covered), f"rows not covered once: offs={offs} M={M}"
    owned = [0] * p.U
    for b, segs in enumerate(p.ctas):
        assert segs, f"CTA {b} of the device grid {p.G} has no units"
        for s in segs:
            for u in range(s.tile * p.KT + s.kc0, s.tile * p.KT + s.kc0 + s.count):
                owned[u] += 1
    assert owned == [1] * p.U
    return p


# (N, K): N tails (N % 8 == 0), N a multiple of 128, K tails, several n-tiles
SHAPES = [(200, 160), (72, 1024), (128, 4112), (1408, 2048), (14336, 4096)]


@pytest.mark.parametrize("N,K", SHAPES)
def test_schedule_invariants_fp8wo_widths(N, K):
    widths = set()
    cases = _offs_cases()
    rng = random.Random(11)
    for _ in range(20):
        E = rng.choice([1, 8, 64, 128])
        rows = [rng.choice([0, 1, 16, 33, 64, 128, 129, 300]) for _ in range(E)]
        cases.append((list(_cum(rows)), max(1, sum(rows) + rng.choice([0, 5]))))
    for offs, M in cases:
        for G in (None, 1, 3, 64, 132):
            widths.add(_check(offs, M, N, K, G).width)
    assert widths == {16, 32, 64, 128}, widths


def test_gpu_cases_reach_every_segment_kind_and_width():
    import test_grouped_fp8_weight_only_gpu as suite

    kinds, widths = set(), set()
    for rows, N, K, tail, grids in suite.GROUPED_CASES:
        offs, M = list(_cum(rows)), sum(rows) + tail
        for G in [None] + suite.grids_of(rows, N, K, tail, grids, 132):
            p = _check(offs, M, N, K, G)
            widths.add(p.width)
            for segs in p.ctas:
                kinds.update(s.kind for s in segs)
    assert {sk.FULL, sk.CONTRIB, sk.OWNER} <= kinds, kinds
    assert widths == {16, 32, 64, 128}, widths


# ------------------------------------------------------------------------------------------------ producer hook model
def _tma_box_1d(v, start, n=128):
    """A 1-D TMA box of n elements from element `start` of v, zero past its end."""
    out = torch.zeros(n, dtype=v.dtype)
    k = min(n, max(0, v.numel() - start))
    out[:k] = v[start:start + k]
    return out


def _tma_box_2d(t, c0, r0, w, h):
    out = torch.zeros(h, w, dtype=t.dtype)
    rows, cols = t.shape
    rr, cc = min(h, max(0, rows - r0)), min(w, max(0, cols - c0))
    out[:rr, :cc] = t[r0:r0 + rr, c0:c0 + cc]
    return out


@pytest.mark.parametrize("E,N,K", [(3, 200, 160), (4, 128, 384), (2, 72, 256), (5, 8, 128), (2, 296, 1040)])
def test_issue_w_rows_loads_each_experts_rows_and_scales(E, N, K):
    """Fp8WoFmt::issue_w_rows for weight row e*N + 128t, chunk kc: the {128 k, 128 rows} box at (128 kc, e*N + 128t) of
    the [E*N, K] bytes and the 128-element box at e*N + 128t of w_scale [E*N].  Rows r < N - 128t of both are expert
    e's features 128t + r; the others belong to the next expert or are zero, and are exactly the features >= N.  With
    N % 8 == 0 every scale box starts on 32 bytes of w_scale."""
    gen = torch.Generator().manual_seed(E * N + K)
    q = torch.randint(0, 256, (E, N, K), generator=gen, dtype=torch.int32).to(torch.uint8)
    s = torch.rand(E, N, generator=gen) + 0.5
    wmap, smap = q.reshape(E * N, K), s.reshape(E * N)
    for e in range(E):
        for t in range(-(-N // 128)):
            row = e * N + 128 * t
            assert (row * 4) % 32 == 0
            sbox = _tma_box_1d(smap, row)
            own = min(128, N - 128 * t)
            assert torch.equal(sbox[:own], s[e, 128 * t:128 * t + own])
            assert torch.equal(sbox[own:], _tma_box_1d(smap, (e + 1) * N)[:128 - own])   # next expert or zero
            for kc in range(-(-K // 128)):
                wbox = _tma_box_2d(wmap, 128 * kc, row, 128, 128)
                kk = min(128, K - 128 * kc)
                assert torch.equal(wbox[:own, :kk], q[e, 128 * t:128 * t + own, 128 * kc:128 * kc + kk])
                assert not wbox[:, kk:].any()   # the K tail is zero-filled
                # a stored feature's output reads its own weight row and scale only: row r of both boxes
                if own < 128:
                    assert row + own == (e + 1) * N


# ------------------------------------------------------------------------------------------------ residency
TABLE_BYTES = 4 * (1024 + 1025)   # s_end[MAX_EXPERTS] + s_mbp[MAX_EXPERTS + 1]


def test_grouped_tables_fit_beside_the_ring_one_cta_per_sm():
    for n_mma in (16, 32, 64, 128):
        _, ctas, stages, _ = sk.ring("fp8wo", n_mma, grouped=True)
        smem = sk.ring_smem("fp8wo", n_mma, grouped=True)
        assert ctas == 1 and stages >= 2
        assert smem + TABLE_BYTES <= 227 * 1024 and smem + TABLE_BYTES + RESERVED_PER_CTA <= SMEM_PER_SM, n_mma


def test_grouped_fp8_weight_only_kernels_have_no_stack():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found = {}
    fn = None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_4lowp8Fp8WoFmtE\S*?Li(\d+)E\S*):", line)
        if m:
            fn = int(m.group(2))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            found[fn] = (int(m.group(1)), int(m.group(2)))
        fn = None
    assert sorted(found) == [16, 32, 64, 128], found
    for n_mma, (reg, stack) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<Fp8WoFmt>, {n_mma}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (n_mma, reg)   # one CTA of 384 threads per SM: 65536 / 384, rounded down to 8


# ------------------------------------------------------------------------------------------------ the fixture
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "float8_weight_only_3d.npz"))


def golden_shapes(d):
    """(case, arrays) per shape of the fixture, with each granularity's qdata, scale, block_size and outputs."""
    for c in json.loads(str(d["cases"])):
        s = c["shape"]
        a = dict(w=d[f"s{s}_w"], x=d[f"s{s}_x"], xe=d[f"s{s}_xe"], offs=d[f"s{s}_offs"])
        for g in ("PerRow", "PerTensor"):
            for f in ("q", "scale", "block_size", "y", "ye"):
                a[f"{g}_{f}"] = d[f"s{s}_{g}_{f}"]
        a["PerRow_y_linear"], a["PerRow_ye_linear"] = d[f"s{s}_PerRow_y_linear"], d[f"s{s}_PerRow_ye_linear"]
        yield c, a


def grouped_ref(x, q, scale, offs):
    """The recipe on float32 arrays: rows [offs[e-1], offs[e]) of x [M, K] times expert e's w~ = bf16(fp32(q[e]) * s),
    one fp32 sum per output rounded to bf16 (fp64 sums, exact in fp32 where the fixture's one-hot rows are used).
    Returns the rows up to offs[-1]."""
    E, N, _ = q.shape
    s = np.broadcast_to(np.asarray(scale, np.float32).reshape(-1) if scale.size > 1 else scale.reshape(1), (E * N,))
    out, start = [], 0
    for e in range(E):
        wt = dequantize_ref(q[e], s[e * N:(e + 1) * N])
        with np.errstate(invalid="ignore", over="ignore"):
            out.append(bf16_round((x[start:offs[e]].astype(np.float64) @ wt.astype(np.float64).T).astype(np.float32)))
        start = offs[e]
    return np.concatenate(out)


def per_expert_within_the_sum_bound(got_bits, ref_bits, x, q, scale, offs):
    """within_one_step_of_the_sum for the rows of each non-empty expert, with that expert's weights and scales."""
    E, N, _ = q.shape
    start = 0
    for e, o in enumerate(offs):
        if o > start:
            se = scale.reshape(-1) if scale.size == 1 else scale.reshape(E, N)[e]
            if not within_one_step_of_the_sum(got_bits[start:o], ref_bits[start:o], x[start:o], q[e], se):
                return False
        start = max(start, o)
    return True


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32).__rshift__(16).astype(np.uint16)


def test_restatement_reproduces_the_reference(golden):
    """One-hot inputs: the restatement equals the reference bit for bit; random inputs: within the accumulation-order
    bound; the reference's per-expert F.linear through select gives its grouped outputs; the zero row's NaN reaches
    every token of expert 0 under PerRow, and the fixture has the cases it claims."""
    for c, a in golden_shapes(golden):
        end = int(a["offs"][-1])
        rows = np.diff(np.concatenate([[0], a["offs"]]))
        assert (rows == 0).any() or c["shape"] == 2
        for g in ("PerRow", "PerTensor"):
            q, s = a[f"{g}_q"], a[f"{g}_scale"]
            assert same_bits_or_both_nan(_bits(grouped_ref(f32(a["xe"]), q, s, a["offs"])), a[f"{g}_ye"]), (c, g)
            ref = _bits(grouped_ref(f32(a["x"]), q, s, a["offs"]))
            assert same_bits_or_both_nan(ref, ref)
            assert per_expert_within_the_sum_bound(a[f"{g}_y"], ref, f32(a["x"]), q, s, a["offs"]), (c, g)
        assert np.array_equal(a["PerRow_ye_linear"], a["PerRow_ye"]) and a["PerRow_y_linear"].shape == (end, c["N"])
        if rows[0]:
            assert np.isnan(f32(a["PerRow_ye"])[:rows[0], 1]).all()
    assert any(c["N"] % 128 for c, _ in golden_shapes(golden)) and any(c["K"] % 128 for c, _ in golden_shapes(golden))
    assert any(c["tail"] for c, _ in golden_shapes(golden))


def test_package_quantizer_matches_the_fixture(golden):
    from ao_b200.quantization import Float8Tensor, PerRow, PerTensor

    for c, a in golden_shapes(golden):
        w = torch.from_numpy(a["w"].view(np.int16).copy()).view(torch.bfloat16)
        for g, gran in (("PerRow", PerRow()), ("PerTensor", PerTensor())):
            t = Float8Tensor.from_hp(w, E4M3, gran)
            assert t.shape == (c["E"], c["N"], c["K"]) and t.act_quant_kwargs is None and t.dtype == torch.bfloat16
            assert list(t.block_size) == a[f"{g}_block_size"].tolist()
            assert same_codes(t.qdata.view(torch.uint8).numpy(), a[f"{g}_q"]), (c, g)
            assert np.array_equal(t.scale.numpy(), a[f"{g}_scale"]), (c, g)


# ------------------------------------------------------------------------------------------------ tensor and handler
def _w3(E=4, N=200, K=160, gran=None, seed=0, dtype=torch.bfloat16):
    from ao_b200.quantization import Float8Tensor, PerRow

    g = torch.Generator().manual_seed(seed)
    return Float8Tensor.from_hp(torch.randn(E, N, K, generator=g).to(dtype), E4M3, gran or PerRow())


def test_select_and_transpose():
    """select(0, e) is expert e's 2-D tensor (qdata[e], scale[e], block_size[1:]) sharing the 3-D tensor's storage;
    the 2-D tensor of a per-tensor weight keeps the one scale.  transpose swaps shape, qdata, scale and block_size."""
    from ao_b200.quantization import Float8Tensor, PerTensor

    w = _w3()
    full = w.dequantize()
    for e in range(4):
        we = w[e]
        assert type(we) is Float8Tensor and we.shape == (200, 160) and list(we.block_size) == [1, 160]
        assert we.scale.shape == (200, 1) and we.act_quant_kwargs is None and we.dtype == torch.bfloat16
        assert we.qdata.untyped_storage().data_ptr() == w.qdata.untyped_storage().data_ptr()
        assert torch.equal(we.dequantize(), full[e])
    pt = _w3(gran=PerTensor(), seed=1)
    assert pt.scale.shape == (1, 1, 1) and list(pt.block_size) == [4, 200, 160]
    for e in range(4):
        assert pt[e].scale.shape == (1, 1) and list(pt[e].block_size) == [200, 160]
        assert torch.equal(pt[e].dequantize(), pt.dequantize()[e])
    with pytest.raises(AssertionError):
        torch.select(w, 1, 0)
    t = w.transpose(-2, -1)
    assert type(t) is Float8Tensor and t.shape == (4, 160, 200) and list(t.block_size) == [1, 160, 1]
    assert t.qdata.stride(-2) < t.qdata.stride(-1) and t.scale.shape == (4, 1, 200)
    assert torch.equal(t.dequantize(), full.transpose(-2, -1))
    tt = t.transpose(-2, -1)
    assert tt.shape == w.shape and list(tt.block_size) == [1, 1, 160] and torch.equal(tt.dequantize(), full)
    dyn = _w3(seed=2)   # the dynamic config's 3-D weights select the same way
    from ao_b200.quantization import QuantizeTensorToFloat8Kwargs

    dyn.act_quant_kwargs = QuantizeTensorToFloat8Kwargs()
    assert dyn[1].act_quant_kwargs == dyn.act_quant_kwargs and torch.equal(dyn[1].qdata.view(torch.uint8),
                                                                           dyn.qdata[1].view(torch.uint8))


def test_grouped_mm_handler_rejects_unsupported_forms():
    from ao_b200.quantization import Float8Tensor, PerGroup

    w = _w3()
    x = torch.randn(16, 160, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    for fn in (torch._grouped_mm, F.grouped_mm):
        with pytest.raises(AssertionError, match="offs is required"):
            fn(x, w.transpose(-2, -1))
        with pytest.raises(AssertionError, match="unsupported|transposed"):
            fn(x, w, offs=offs)
        with pytest.raises(NotImplementedError, match="bias"):
            torch._grouped_mm(x, w.transpose(-2, -1), offs=offs, bias=torch.zeros(200, dtype=torch.bfloat16))
        with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
            fn(x, w.transpose(-2, -1), offs=offs, out_dtype=torch.float32)
        with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
            fn(x.half(), w.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="2-D mat_a x 3-D mat_b"):
            fn(x.reshape(4, 4, 160), w.transpose(-2, -1), offs=offs)
        for dt in (torch.float16, torch.float32):
            with pytest.raises(NotImplementedError, match=f"quantized from {dt}"):
                fn(x, _w3(dtype=dt).transpose(-2, -1), offs=offs)
        # group scales arrive only from a checkpoint (the config handler rejects them)
        wg = Float8Tensor.from_hp(torch.randn(4, 200, 160).to(torch.bfloat16), E4M3, PerGroup(32))
        with pytest.raises(NotImplementedError, match="no sm_90a kernel"):
            fn(x, wg.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="N % 8 == 0"):
            fn(x, _w3(N=204).transpose(-2, -1), offs=offs)
        # a served form on CPU tensors reaches the CUDA-only op and fails in the dispatcher
        with pytest.raises(NotImplementedError, match="fp8_weight_grouped_mm"):
            fn(x, w.transpose(-2, -1), offs=offs)
    with pytest.raises(NotImplementedError, match="no sm_90a kernel"):   # the 2-D linear: one expert at a time
        F.linear(x, w)


def test_3d_serialization_round_trips():
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Float8Tensor, PerTensor

    for gran in (None, PerTensor()):
        w = _w3(3, 20, 64, gran=gran, seed=3)
        buf = io.BytesIO()
        torch.save({"experts.w": w}, buf)
        buf.seek(0)
        r = torch.load(buf, weights_only=True)["experts.w"]
        flat, meta = flatten_tensor_state_dict({"experts.w": w})
        s, left = unflatten_tensor_state_dict(flat, meta)
        assert not left
        for got in (r, s["experts.w"]):
            assert type(got) is Float8Tensor and got.shape == (3, 20, 64) and got.act_quant_kwargs is None
            assert list(got.block_size) == list(w.block_size) and got.dtype == torch.bfloat16
            assert torch.equal(got.qdata.view(torch.uint8), w.qdata.view(torch.uint8)) and torch.equal(got.scale, w.scale)


class Experts(torch.nn.Module):
    def __init__(self, E, H, I, dtype=torch.bfloat16):
        super().__init__()
        self.gate_up_proj = torch.nn.Parameter(torch.randn(E, 2 * I, H, dtype=dtype))
        self.down_proj = torch.nn.Parameter(torch.randn(E, H, I, dtype=dtype))


class Block(torch.nn.Module):
    def __init__(self, E, H, I, dtype=torch.bfloat16):
        super().__init__()
        self.experts = Experts(E, H, I, dtype)


def test_config_3d_rules(caplog):
    """Float8WeightOnlyConfig on 3-D parameters (through FqnToConfig) follows the 2-D rules: K % 16 != 0 and weights
    that are not bf16 stay unquantized with a log line, PerGroup and e5m2 raise, the rest quantizes per row / tensor."""
    from ao_b200.quantization import Float8Tensor, Float8WeightOnlyConfig, FqnToConfig, PerGroup, PerTensor, quantize_

    m = Block(2, 256, 200)   # down_proj K = 200
    with caplog.at_level(logging.INFO):
        quantize_(m, FqnToConfig({"experts.down_proj": Float8WeightOnlyConfig()}), filter_fn=None)
    assert type(m.experts.down_proj) is torch.nn.Parameter and m.experts.down_proj.dtype == torch.bfloat16
    assert "Skipping float8 weight only quantization" in caplog.text and "(2, 256, 200)" in caplog.text
    caplog.clear()
    mf = Block(2, 256, 128, dtype=torch.float16)
    with caplog.at_level(logging.INFO):
        quantize_(mf, FqnToConfig({"experts.gate_up_proj": Float8WeightOnlyConfig()}), filter_fn=None)
    assert type(mf.experts.gate_up_proj) is torch.nn.Parameter and "torch.float16" in caplog.text
    with pytest.raises(NotImplementedError, match="PerGroup"):
        quantize_(m, FqnToConfig({"experts.gate_up_proj": Float8WeightOnlyConfig(granularity=PerGroup(32))}),
                  filter_fn=None)
    with pytest.raises(NotImplementedError, match="float8_e5m2"):
        quantize_(m, FqnToConfig({"experts.gate_up_proj": Float8WeightOnlyConfig(weight_dtype=torch.float8_e5m2)}),
                  filter_fn=None)
    assert type(m.experts.gate_up_proj) is torch.nn.Parameter
    quantize_(m, FqnToConfig({"experts.gate_up_proj": Float8WeightOnlyConfig()}), filter_fn=None)
    w = m.experts.gate_up_proj
    assert isinstance(w, Float8Tensor) and w.shape == (2, 400, 256) and w.scale.shape == (2, 400, 1)
    assert w.act_quant_kwargs is None and list(w.block_size) == [1, 1, 256]
    m2 = Block(2, 256, 128)
    cfg = Float8WeightOnlyConfig(granularity=PerTensor())
    quantize_(m2, FqnToConfig({"experts.gate_up_proj": cfg, "experts.down_proj": cfg}), filter_fn=None)
    for p in (m2.experts.gate_up_proj, m2.experts.down_proj):
        assert isinstance(p, Float8Tensor) and p.scale.shape == (1, 1, 1) and list(p.block_size) == list(p.shape)
