"""CPU tests of the int4 expert GEMM (torch._grouped_mm on 3-D Int4TilePackedTo4dTensor weights):

* the Meta shape and schema of torch.ops.ao_b200.int4_tilepacked_grouped_mm and the C-ABI argument checks of
  ao_int4_tilepacked_grouped_mm (before any CUDA call);
* the grouped schedule (tests/grouped_model.py) at the int4 token-tile widths 16 .. 128, with N tails;
* a model of Int4Fmt::issue_w_rows: for every (expert, n-tile, chunk, group size) the scale box it loads from the
  grouped scale map is that expert's scale_and_zero block, zero past N, and its weight box starts at the expert's
  n8-tile 16t;
* Grouped<Int4Fmt> runs one CTA per SM without stack, its schedule tables fit beside the ring;
* transpose / select metadata, the handler's rejections, serialization and the config rules on hand-built tensors.
"""
import ctypes
import io
import logging
import os
import random
import re
import shutil
import subprocess

import pytest
import torch

import grouped_nvfp4_model as gnm
import streamk_model as sk
from test_decode_residency import LIB, RESERVED_PER_CTA, SMEM_PER_SM
from test_grouped_schedule import _cum, _offs_cases


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
def test_meta_shape_and_schema():
    import ao_b200  # noqa: F401

    op = torch.ops.ao_b200.int4_tilepacked_grouped_mm
    assert str(op.default._schema) == ("ao_b200::int4_tilepacked_grouped_mm(Tensor x, Tensor qdata, int group_size, "
                                       "Tensor scale_and_zero, Tensor offs, int n_out) -> Tensor")
    x = torch.empty(37, 2048, dtype=torch.bfloat16, device="meta")
    qdata = torch.empty(8, 1008 // 8, 16, 32, 4, dtype=torch.int32, device="meta")
    sz = torch.empty(8, 2048 // 32, 1008, 2, dtype=torch.bfloat16, device="meta")
    offs = torch.empty(8, dtype=torch.int32, device="meta")
    y = op(x, qdata, 32, sz, offs, 1001)
    assert y.shape == (37, 1001) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert op(x, qdata, 32, sz, offs, 0).shape == (37, 1008)


def _lib():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    return lib


def test_c_abi_argument_validation_without_gpu():
    lib = _lib()
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_int4_tilepacked_grouped_mm
    f.argtypes = [vp, i32, i32, vp, vp, i32, i32, i32, i32, vp, vp, vp, sz, vp]
    one = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first

    def call(M=4, K=1024, g=32, E=8, N=256, N_out=256, ptrs=(one,) * 6):
        x, qd, sc, offs, y, ws = ptrs
        return f(x, M, K, qd, sc, g, E, N, N_out, offs, y, ws, 1 << 20, None)

    err = lambda: lib.ao_b200_last_error()   # noqa: E731
    assert call(K=768) == -1 and b"K=768" in err()
    assert call(N=100, N_out=100) == -1 and b"N=100" in err()
    assert call(g=16) == -1 and b"group_size=16" in err()
    assert call(N_out=257) == -1 and b"N_out=257" in err()
    assert call(N_out=0) == -1 and b"N_out=0" in err()
    assert call(E=0) == -1 and b"E=0" in err()
    assert call(E=1025) == -1 and b"E=1025" in err()
    assert call(E=1024, N=2**21, N_out=2**21) == -1 and b"int32" in err()
    assert call(M=-1) == -1 and b"bad sizes" in err()
    for i in range(6):
        ptrs = [one] * 6
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in err(), i
    assert call(ptrs=(ctypes.c_void_p(24),) + (one,) * 5) == -1 and b"16-byte" in err()
    # no tokens: nothing to do, nothing dereferenced
    assert call(M=0, ptrs=(None,) * 6) == 0


# ------------------------------------------------------------------------------------------------ schedule
def plan(offs, M, N_out, K, grid=None, sm=132):
    """The grouped split of one int4 launch: the nvfp4 plan, whose token tiles (16 .. 128) and whole 128-k chunks are
    int4's too; the tiles cover the N_out output features."""
    assert sk.WIDTHS["int4"] == sk.WIDTHS["nvfp4"] and sk.k_chunks("int4", K) == sk.k_chunks("nvfp4", K)
    return gnm.plan(offs, M, N_out, K, grid=grid, sm=sm, fmt="int4")


# (N padded, N_out, K): N tails inside the last tile, N a multiple of 128, several n-tiles
SHAPES = [(1008, 1001, 1024), (128, 128, 2048), (264, 260, 1024), (2048, 2048, 4096), (8, 3, 1024)]


def _check(offs, M, N, N_out, K, grid, sm=132):
    p = plan(offs, M, N_out, K, grid, sm)
    E = len(offs)
    assert p.n_tiles == -(-N_out // sk.ROWS)
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
        # the weight box starts inside expert e's rows; a tail past N reads the next expert (or zero fill), and the
        # features it computes there are >= N_out, never stored
        row = e * N + n_tile * sk.ROWS
        assert e * N <= row < (e + 1) * N
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


@pytest.mark.parametrize("N,N_out,K", SHAPES)
def test_schedule_invariants_int4_widths(N, N_out, K):
    widths = set()
    cases = _offs_cases()
    rng = random.Random(7)
    for _ in range(20):
        E = rng.choice([1, 8, 64, 128])
        rows = [rng.choice([0, 1, 16, 33, 64, 128, 129, 300]) for _ in range(E)]
        cases.append((list(_cum(rows)), max(1, sum(rows) + rng.choice([0, 5]))))
    for offs, M in cases:
        for G in (None, 1, 3, 64, 132):
            widths.add(_check(offs, M, N, N_out, K, G).width)
    assert widths == {16, 32, 64, 128}, widths


def test_gpu_cases_reach_every_segment_kind_and_width():
    import test_grouped_int4_gpu as suite

    kinds, widths = set(), set()
    for rows, N_out, K, g, tail, grids in suite.GROUPED_CASES:
        N = -(-N_out // 8) * 8
        offs, M = list(_cum(rows)), sum(rows) + tail
        for G in [None] + suite.grids_of(rows, N_out, K, tail, grids, 132):
            p = _check(offs, M, N, N_out, K, G)
            widths.add(p.width)
            for segs in p.ctas:
                kinds.update(s.kind for s in segs)
    assert {sk.FULL, sk.CONTRIB, sk.OWNER} <= kinds, kinds
    assert widths == {16, 32, 64, 128}, widths


# ------------------------------------------------------------------------------------------------ producer hook model
def _tma_box_2d(t, c0, r0, w, h):
    """A TMA box {w, h} at (column c0, row r0) of the 2-D tensor t, zero past its bounds."""
    out = torch.zeros(h, w, dtype=t.dtype)
    rows, cols = t.shape
    rr, cc = min(h, max(0, rows - r0)), min(w, max(0, cols - c0))
    out[:rr, :cc] = t[r0:r0 + rr, c0:c0 + cc]
    return out


def issue_w_rows(E, N, K, g, row, kc):
    """Int4Fmt::issue_w_rows: (first n8-tile of the weight box, the scale box origin (column, row)) for weight row
    `row` = e*N + 128t and chunk kc, with the grouped scale map uint32 {N, E*K/g}."""
    e = row // N
    return row // 8, (row - e * N, e * (K // g) + (kc * 128) // g)


@pytest.mark.parametrize("E,N,K", [(3, 1008, 2048), (2, 264, 1024), (4, 128, 3072), (2, 8, 1024)])
def test_issue_w_rows_addresses_each_experts_block(E, N, K):
    gen = torch.Generator().manual_seed(E * N + K)
    for g in (32, 64, 128, 256):
        gpc = 128 // g if g <= 128 else 1
        sz = torch.randint(-2**31, 2**31 - 1, (E, K // g, N), generator=gen, dtype=torch.int64).to(torch.int32)
        scale_map = sz.reshape(E * (K // g), N)   # scale_and_zero [E, K/g, N, 2] bf16 as uint32 [E*K/g][N]
        for e in range(E):
            for t in range(-(-N // 128)):
                for kc in range(K // 128):
                    tile0, (c0, r0) = issue_w_rows(E, N, K, g, e * N + 128 * t, kc)
                    box = _tma_box_2d(scale_map, c0, r0, 128, gpc)
                    want = torch.zeros(gpc, 128, dtype=torch.int32)
                    g0 = (kc * 128) // g
                    blk = sz[e, g0:g0 + gpc, 128 * t:128 * t + 128]
                    want[:, :blk.shape[1]] = blk
                    assert torch.equal(box, want), (E, N, K, g, e, t, kc)
                    assert tile0 == e * N // 8 + 16 * t


# ------------------------------------------------------------------------------------------------ residency
TABLE_BYTES = 4 * (1024 + 1025)   # s_end[MAX_EXPERTS] + s_mbp[MAX_EXPERTS + 1]


def test_grouped_tables_fit_beside_the_ring_one_cta_per_sm():
    for n_mma in (16, 32, 64, 128):
        _, ctas, _, _ = sk.ring("int4", n_mma, grouped=True)
        smem = sk.ring_smem("int4", n_mma, grouped=True)
        assert ctas == 1
        assert smem + TABLE_BYTES <= 227 * 1024 and smem + TABLE_BYTES + RESERVED_PER_CTA <= SMEM_PER_SM, n_mma
        # two CTAs with the dense decode ring (6 stages of a 32-wide tile) and the tables would not fit
    assert 2 * (sk.ring_smem("int4", 32) + TABLE_BYTES + RESERVED_PER_CTA) > SMEM_PER_SM


def test_grouped_int4_kernels_have_no_stack():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found = {}
    fn = None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_5int4k7Int4FmtE\S*?Li(\d+)E\S*):", line)
        if m:
            fn = int(m.group(2))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            found[fn] = (int(m.group(1)), int(m.group(2)))
        fn = None
    assert sorted(found) == [16, 32, 64, 128], found
    for n_mma, (reg, stack) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<Int4Fmt>, {n_mma}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (n_mma, reg)   # one CTA of 384 threads per SM


# ------------------------------------------------------------------------------------------------ tensor and config
def _int4_3d(E, N0, K0, g):
    """A hand-built CPU tensor of the 3-D layout (random payload)."""
    from ao_b200.quantization import Int4TilePackedTo4dTensor

    N, K = -(-N0 // 8) * 8, -(-K0 // 1024) * 1024
    gen = torch.Generator().manual_seed(E + N0 + K0)
    qdata = torch.randint(-2**31, 2**31 - 1, (E, N // 8, K // 128, 32, 4), generator=gen, dtype=torch.int64).to(torch.int32)
    sz = torch.randn(E, K // g, N, 2, generator=gen).to(torch.bfloat16)
    return Int4TilePackedTo4dTensor(qdata, sz, [1, 1, g], torch.Size([E, N0, K0]))


def test_transpose_and_select_metadata():
    from ao_b200.quantization import Int4TilePackedTo4dTensor

    w = _int4_3d(4, 20, 768, 32)
    t = w.transpose(-2, -1)
    assert isinstance(t, Int4TilePackedTo4dTensor) and t.shape == (4, 768, 20) and list(t.block_size) == [1, 32, 1]
    assert t.qdata is w.qdata and t.scale_and_zero is w.scale_and_zero and t._is_transposed() and not w._is_transposed()
    tt = t.transpose(1, 2)
    assert tt.shape == w.shape and list(tt.block_size) == [1, 1, 32] and not tt._is_transposed()
    w.act_pre_scale = torch.full((768,), 0.5, dtype=torch.bfloat16)
    e = w[2]
    assert isinstance(e, Int4TilePackedTo4dTensor) and e.shape == (20, 768) and list(e.block_size) == [1, 32]
    assert torch.equal(e.qdata, w.qdata[2]) and torch.equal(e.scale_and_zero, w.scale_and_zero[2])
    assert e.act_pre_scale is w.act_pre_scale
    with pytest.raises(AssertionError):
        t[0]   # select the expert before transposing


def test_grouped_mm_handler_rejects_unsupported_forms():
    w = _int4_3d(4, 128, 1024, 32)
    x = torch.randn(16, 1024, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    with pytest.raises(NotImplementedError, match="transposed"):
        torch._grouped_mm(x, w, offs=offs)
    with pytest.raises(NotImplementedError, match="offs is required"):
        torch._grouped_mm(x, w.transpose(-2, -1))
    with pytest.raises(NotImplementedError, match="2-D mat_a x 3-D mat_b"):
        torch._grouped_mm(x.reshape(4, 4, 1024), w.transpose(-2, -1))
    with pytest.raises(NotImplementedError, match="bias"):
        torch._grouped_mm(x, w.transpose(-2, -1), offs=offs, bias=torch.zeros(128, dtype=torch.bfloat16))
    with pytest.raises(NotImplementedError, match="bf16"):
        torch._grouped_mm(x, w.transpose(-2, -1), offs=offs, out_dtype=torch.float32)
    with pytest.raises(NotImplementedError, match="select"):
        torch.nn.functional.linear(x, w)


def test_3d_serialization_round_trips():
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Int4TilePackedTo4dTensor

    w = _int4_3d(3, 20, 768, 64)
    buf = io.BytesIO()
    torch.save({"experts.w": w}, buf)
    buf.seek(0)
    r = torch.load(buf, weights_only=True)["experts.w"]
    flat, meta = flatten_tensor_state_dict({"experts.w": w})
    s, left = unflatten_tensor_state_dict(flat, meta)
    assert not left
    for got in (r, s["experts.w"]):
        assert isinstance(got, Int4TilePackedTo4dTensor) and got.shape == (3, 20, 768)
        assert list(got.block_size) == [1, 1, 64]
        assert torch.equal(got.qdata, w.qdata) and torch.equal(got.scale_and_zero.view(torch.int16), w.scale_and_zero.view(torch.int16))


class Experts(torch.nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.gate_up_proj = torch.nn.Parameter(torch.randn(E, 2 * I, H, dtype=torch.bfloat16))
        self.down_proj = torch.nn.Parameter(torch.randn(E, H, I, dtype=torch.bfloat16))


class Block(torch.nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.experts = Experts(E, H, I)


def test_config_3d_rules(caplog):
    """Int4WeightOnlyConfig reaches 3-D parameters through FqnToConfig; a weight with K % group_size != 0 is left
    unquantized with a log line (the reference's rule); a 3-D weight that passes it goes on to from_hp, which packs on
    the GPU."""
    from ao_b200.quantization import FqnToConfig, Int4WeightOnlyConfig, quantize_

    cfg = Int4WeightOnlyConfig(group_size=128, int4_packing_format="tile_packed_to_4d")
    m = Block(2, 256, 200)   # down_proj K = 200
    with caplog.at_level(logging.INFO):
        quantize_(m, FqnToConfig({"experts.down_proj": cfg}), filter_fn=None)
    assert type(m.experts.down_proj) is torch.nn.Parameter and m.experts.down_proj.dtype == torch.bfloat16
    assert "Skipping quantizing weight with int4 weight only quantization" in caplog.text
    with pytest.raises(NotImplementedError, match="CUDA"):
        quantize_(m, FqnToConfig({"experts.gate_up_proj": cfg}), filter_fn=None)
