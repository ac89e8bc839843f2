"""CPU tests of the MX expert GEMM (torch._grouped_mm on 3-D mxfp8 / mxfp4 MXTensor weights):

* the Meta shapes of torch.ops.ao_b200.mx{fp8,fp4}_grouped_mm / mx{fp8,fp4}_fakequant and their C-ABI argument checks
  (before any CUDA call);
* the grouped schedule (tests/grouped_model.py with the mxfp8 / mxfp4 rings) at the token tiles 16 .. 128, on random
  and malformed offs: row coverage, the bounds of every weight and scale-tile read, the device-side grid;
* the stacked per-expert blocked scales are to_blocked of the [E * N, K / 32] scales, tile by tile;
* Grouped<Mxfp8Fmt> and Grouped<Mxfp4Fmt> have no stack frame and their schedule tables fit beside the ring;
* the MXTensor pieces torch._grouped_mm and F.linear(x, w[e]) go through (3-D dequantize, transpose, select), the
  handler's rejections and the config's 3-D rule.
"""
import ctypes
import logging
import random

import pytest
import torch

import grouped_model as gm
import streamk_model as sk
from test_decode_residency import LIB, RESERVED_PER_CTA, SMEM_PER_SM
from test_grouped_schedule import _cum, _offs_cases

FMTS = ("mxfp8", "mxfp4")
ELEM = {"mxfp8": torch.float8_e4m3fn, "mxfp4": torch.float4_e2m1fn_x2}


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
@pytest.mark.parametrize("fmt", FMTS)
def test_meta_shapes(fmt):
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    x = torch.empty(37, 512, dtype=torch.bfloat16, device="meta")
    xhat = getattr(ops, f"{fmt}_fakequant")(x)
    assert xhat.shape == (37, 512) and xhat.dtype == torch.bfloat16 and xhat.device.type == "meta"
    kq = 512 // 2 if fmt == "mxfp4" else 512
    wq = torch.empty(8, 256, kq, dtype=torch.uint8, device="meta")
    ws = torch.empty(8, 64, 64, dtype=torch.uint8, device="meta")
    offs = torch.empty(8, dtype=torch.int32, device="meta")
    y = getattr(ops, f"{fmt}_grouped_mm")(xhat, wq, ws, offs)
    assert y.shape == (37, 256) and y.dtype == torch.bfloat16 and y.device.type == "meta"


def _lib():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    return lib


@pytest.mark.parametrize("fmt", FMTS)
def test_grouped_mm_c_abi_argument_validation_without_gpu(fmt):
    lib = _lib()
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = getattr(lib, f"ao_{fmt}_grouped_mm")
    f.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    one = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first

    def call(M=4, K=256, E=8, N=256, ptrs=(one,) * 5, ws=one):
        x, wq, wsc, offs, y = ptrs
        return f(x, M, K, wq, wsc, E, N, offs, y, ws, 1 << 20, None)

    assert call(K=48) == -1 and b"K=48" in lib.ao_b200_last_error()
    assert call(N=192) == -1 and b"N=192" in lib.ao_b200_last_error()
    assert call(N=64) == -1 and b"N=64" in lib.ao_b200_last_error()
    assert call(E=0) == -1 and b"E=0" in lib.ao_b200_last_error()
    assert call(E=1025) == -1 and b"E=1025" in lib.ao_b200_last_error()
    assert call(E=1024, N=2**21) == -1 and b"int32" in lib.ao_b200_last_error()
    assert call(M=-1) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    for i in range(5):
        ptrs = [one] * 5
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in lib.ao_b200_last_error(), i
    assert call(ws=None) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert call(ptrs=(ctypes.c_void_p(24),) + (one,) * 4) == -1 and b"16-byte" in lib.ao_b200_last_error()
    # no tokens: nothing to do, nothing dereferenced; K = 96 (a K tail of the last chunk) passes the K rule
    assert call(M=0, ptrs=(None,) * 5, ws=None) == 0
    assert call(M=0, K=96, ptrs=(None,) * 5, ws=None) == 0


@pytest.mark.parametrize("fmt", FMTS)
def test_fakequant_c_abi_argument_validation_without_gpu(fmt):
    lib = _lib()
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    f = getattr(lib, f"ao_{fmt}_fakequant")
    f.argtypes = [vp, i32, i32, i32, vp, vp]
    one = ctypes.c_void_p(16)

    def call(M=4, K=256, ldx=256, x=one, xhat=one):
        return f(x, ldx, M, K, xhat, None)

    assert call(K=48, ldx=48) == -1 and b"K=48" in lib.ao_b200_last_error()
    assert call(ldx=100) == -1 and b"ldx=100" in lib.ao_b200_last_error()
    assert call(x=ctypes.c_void_p(24)) == -1 and b"16-byte" in lib.ao_b200_last_error()
    assert call(x=None) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert call(xhat=None) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert call(M=0, x=None, xhat=None) == 0


# ------------------------------------------------------------------------------------------------ schedule
SHAPES = [(128, 1024), (256, 96), (640, 1056), (128, 16384)]


def _check(fmt, offs, M, N, K, grid, sm=132):
    p = gm.plan(offs, M, N, K, grid=grid, sm=sm, fmt=fmt)
    E = len(offs)
    assert N % sk.ROWS == 0 and p.n_tiles == N // sk.ROWS and p.KT == -(-K // 128)
    end = p.ends[-1]
    assert 0 <= end <= M
    assert p.G <= p.G_host and p.U <= p.U_bound and p.G <= max(p.U, 0)
    if p.U == 0:
        assert p.G == 0 and end == 0
        return p
    covered = [[0] * p.n_tiles for _ in range(end)]
    col_blocks = -(-(K // 32) // 4)
    for t in range(p.U // p.KT):
        e, row0, row_end, n_tile = p.tile(t)
        assert 0 <= e < E and (p.ends[e - 1] if e > 0 else 0) <= row0 < p.ends[e] == row_end <= M
        # the weight box (128 rows from e*N + 128 n_tile) lies inside expert e's rows: no tile tail for N % 128 == 0
        row = e * N + n_tile * sk.ROWS
        assert e * N <= row and row + sk.ROWS <= (e + 1) * N
        # its scale tile per chunk: row block row / 128, column block kc of the stacked blocked scales
        rb = row // sk.ROWS
        assert rb == e * (N // sk.ROWS) + n_tile
        assert rb * col_blocks + p.KT - 1 < (E * N // sk.ROWS) * col_blocks
        for m in range(row0, min(row0 + p.width, row_end)):
            covered[m][n_tile] += 1
    assert all(c == [1] * p.n_tiles for c in covered), f"rows not covered once: offs={offs} M={M}"
    owned = [0] * p.U
    for b, segs in enumerate(p.ctas):
        assert segs, f"CTA {b} of the device grid {p.G} has no units"
        for s in segs:
            for u in range(s.tile * p.KT + s.kc0, s.tile * p.KT + s.kc0 + s.count):
                owned[u] += 1
                assert sk.cta_of_unit(u, p.U, p.G) == b
    assert owned == [1] * p.U
    return p


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("N,K", SHAPES)
def test_schedule_invariants_mx_widths(fmt, N, K):
    widths = set()
    cases = _offs_cases()
    rng = random.Random(77)
    for _ in range(20):   # larger routings: the 128-token tile with several m-blocks per expert
        E = rng.choice([1, 4, 8, 64])
        rows = [rng.choice([0, 1, 15, 16, 17, 127, 128, 129, 300]) for _ in range(E)]
        cases.append((list(_cum(rows)), max(1, sum(rows) + rng.choice([0, 5]))))
    for offs, M in cases:
        for G in (None, 1, 2, 3, 7, 64, 131, 132, 500):
            widths.add(_check(fmt, offs, M, N, K, G).width)
    assert widths == {16, 32, 64, 128}, widths


def test_gpu_cases_reach_every_segment_kind_width_and_stage_count():
    import test_grouped_mx_gpu as suite

    for fmt in FMTS:
        kinds, widths = set(), set()
        for rows, N, K, tail, grids in suite.GROUPED_CASES:
            offs, M = list(_cum(rows)), sum(rows) + tail
            for G in [None] + suite.grids_of(fmt, rows, N, K, tail, grids, 132):
                p = _check(fmt, offs, M, N, K, G)
                widths.add(p.width)
                for segs in p.ctas:
                    kinds.update(s.kind for s in segs)
        assert {sk.FULL, sk.CONTRIB, sk.OWNER} <= kinds, (fmt, kinds)
        assert widths == {16, 32, 64, 128}, (fmt, widths)
        # the staged gather: every width whose ring stages partials, owners below, at and above its stage count
        staged = {w for w in sk.WIDTHS[fmt] if sk.ring(fmt, w, grouped=True)[3]}
        assert {w for w, _, _ in suite.staging_layouts(fmt)} == staged and staged, (fmt, staged)


# ------------------------------------------------------------------------------------------------ scale layout
def test_stacked_blocked_scales_are_the_reference_layout():
    """Each expert's blocked [N, K/32] scales one after the other == to_blocked of the [E*N, K/32] scales (N % 128 == 0);
    the 512-byte tile (row block e*N/128 + t, column block c) holds expert e's rows 128t .. 128t+127, scales 4c .. 4c+3
    (zero past K/32)."""
    from ao_b200.prototype.mx_formats.utils import to_blocked

    g = torch.Generator().manual_seed(0)
    for E, N, K in [(3, 128, 96), (3, 256, 256), (2, 384, 1024)]:
        s = torch.randint(0, 256, (E, N, K // 32), generator=g, dtype=torch.int32).to(torch.uint8)
        stacked = torch.cat([to_blocked(s[e]) for e in range(E)])
        assert torch.equal(stacked, to_blocked(s.reshape(E * N, K // 32)))
        cb = -(-(K // 32) // 4)
        tiles = stacked.reshape(-1, 512)
        r = torch.arange(128)
        for e in range(E):
            for t in range(N // 128):
                for c in range(cb):
                    tile = tiles[(e * N // 128 + t) * cb + c]
                    for j in range(4):   # blocked offset of (row r, scale j): (r % 32) * 16 + (r // 32) * 4 + j
                        want = s[e, 128 * t + r, 4 * c + j] if 4 * c + j < K // 32 else torch.zeros(128, dtype=torch.uint8)
                        assert torch.equal(tile[(r % 32) * 16 + (r // 32) * 4 + j], want)


# ------------------------------------------------------------------------------------------------ residency
TABLE_BYTES = 4 * (1024 + 1025)   # s_end[MAX_EXPERTS] + s_mbp[MAX_EXPERTS + 1]


@pytest.mark.parametrize("fmt", FMTS)
def test_grouped_tables_fit_beside_the_ring(fmt):
    for n_mma in (16, 32, 64, 128):
        _, ctas, stages, _ = sk.ring(fmt, n_mma, grouped=True)
        smem = sk.ring_smem(fmt, n_mma, grouped=True)
        assert ctas == 1 and stages >= 2
        assert smem + TABLE_BYTES <= 227 * 1024 and smem + TABLE_BYTES + RESERVED_PER_CTA <= SMEM_PER_SM, n_mma


def test_grouped_mx_kernels_have_no_stack():
    import os
    import re
    import shutil
    import subprocess

    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found = {}
    fn = None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_4lowp8(Mxfp[48])FmtE\S*?Li(\d+)E\S*):", line)
        if m:
            fn = (m.group(2), int(m.group(3)))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            found[fn] = (int(m.group(1)), int(m.group(2)))
        fn = None
    assert sorted(found) == [(f, w) for f in ("Mxfp4", "Mxfp8") for w in (16, 32, 64, 128)], found
    for key, (reg, stack) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<{key[0]}Fmt>, {key[1]}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (key, reg)   # one CTA of 384 threads per SM


# ------------------------------------------------------------------------------------------------ tensor and config
def _mx_3d(fmt, E, N, K, g, swizzled, kwargs=True):
    """A 3-D MXTensor of random codes and scale bytes 100..140 (and the per-expert 2-D tensors it stacks)."""
    from ao_b200.prototype.mx_formats import MXTensor
    from ao_b200.prototype.mx_formats.mx_tensor import QuantizeTensorToMXKwargs
    from ao_b200.prototype.mx_formats.utils import to_blocked

    kq = K // 2 if fmt == "mxfp4" else K
    q = torch.randint(0, 256, (E, N, kq), generator=g, dtype=torch.int32).to(torch.uint8)
    if fmt == "mxfp8":
        q[(q & 0x7F) == 0x7F] = 0   # no NaN codes
        q = q.view(torch.float8_e4m3fn)
    s = torch.randint(100, 141, (E, N, K // 32), generator=g, dtype=torch.int32).to(torch.uint8)
    if swizzled:
        s = torch.stack([to_blocked(s[e]).reshape(32 * -(-N // 128), -1) for e in range(E)])
    k = QuantizeTensorToMXKwargs(elem_dtype=ELEM[fmt], is_swizzled_scales=True) if kwargs else None
    w = MXTensor(q, s.view(torch.float8_e8m0fnu), ELEM[fmt], 32, torch.bfloat16, None, k, swizzled)
    experts = [MXTensor(q[e], s[e].view(torch.float8_e8m0fnu), ELEM[fmt], 32, torch.bfloat16, None, k, swizzled)
               for e in range(E)]
    return w, experts


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("swizzled", [False, True])
def test_3d_dequantize_transpose_and_select(fmt, swizzled):
    """A 3-D MXTensor dequantizes expert by expert as the 2-D tensor of that expert does; its transpose is a view whose
    shape (dim -2 doubled for mxfp4), qdata and dequantize are the transposes of the original's; select(0, e) of a
    blocked weight with N % 128 == 0 is expert e's 2-D tensor with its own blocked scales."""
    from ao_b200.prototype.mx_formats import MXTensor

    g = torch.Generator().manual_seed(1)
    E, N, K = 3, 256, 96
    w, experts = _mx_3d(fmt, E, N, K, g, swizzled)
    assert w.shape == (E, N, K)
    dq = w.dequantize()
    for e in range(E):
        assert torch.equal(dq[e], experts[e].dequantize()), e
    t = w.transpose(-2, -1)
    assert isinstance(t, MXTensor) and t.shape == (E, K, N) and t.qdata.stride(-2) < t.qdata.stride(-1)
    assert torch.equal(t.qdata.transpose(-2, -1).view(torch.uint8), w.qdata.view(torch.uint8))
    assert torch.equal(t.dequantize(), dq.transpose(-2, -1))
    assert t.transpose(-2, -1).shape == (E, N, K)
    for e in range(E):
        we = w[e]
        assert isinstance(we, MXTensor) and we.shape == (N, K) and we.is_swizzled_scales == swizzled
        assert we.act_quant_kwargs is w.act_quant_kwargs
        assert torch.equal(we.scale.view(torch.uint8), experts[e].scale.view(torch.uint8))
        assert torch.equal(we.dequantize(), experts[e].dequantize())


def test_select_keeps_rejecting_other_blocked_layouts():
    g = torch.Generator().manual_seed(2)
    w, experts = _mx_3d("mxfp8", 2, 192, 64, g, swizzled=True)   # N % 128 != 0: the experts share row blocks
    with pytest.raises(AssertionError):
        w[0]
    with pytest.raises(AssertionError):
        experts[0][0]   # a row of a 2-D blocked weight


@pytest.mark.parametrize("fmt", FMTS)
def test_grouped_mm_handler_rejects_unsupported_forms(fmt):
    g = torch.Generator().manual_seed(3)
    E, N, K = 4, 128, 128
    w, _ = _mx_3d(fmt, E, N, K, g, swizzled=True)
    x = torch.randn(16, K, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    wt = w.transpose(-2, -1)
    with pytest.raises(NotImplementedError, match="bias"):
        torch._grouped_mm(x, wt, offs=offs, bias=torch.zeros(E, N, dtype=torch.bfloat16))
    with pytest.raises(NotImplementedError, match="2-D mat_a x 3-D mat_b"):
        torch._grouped_mm(x.reshape(2, 8, K), wt, offs=offs)
    with pytest.raises(NotImplementedError, match="transposed"):
        torch._grouped_mm(x, w, offs=offs)
    with pytest.raises(NotImplementedError, match="offs is required"):
        torch._grouped_mm(x, wt)
    with pytest.raises(ValueError, match="K="):
        torch._grouped_mm(x[:, :64], wt, offs=offs)
    plain, _ = _mx_3d(fmt, E, N, K, g, swizzled=False)
    with pytest.raises(NotImplementedError, match="blocked"):
        torch._grouped_mm(x, plain.transpose(-2, -1), offs=offs)
    wo, _ = _mx_3d(fmt, E, N, K, g, swizzled=True, kwargs=False)
    with pytest.raises(NotImplementedError, match="weight-only"):
        torch._grouped_mm(x, wo.transpose(-2, -1), offs=offs)
    other = "mxfp4" if fmt == "mxfp8" else "mxfp8"
    w.act_quant_kwargs = type(w.act_quant_kwargs)(elem_dtype=ELEM[other], is_swizzled_scales=True)
    with pytest.raises(NotImplementedError, match="element dtype"):
        torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)
    with pytest.raises(NotImplementedError, match="torch._grouped_mm"):   # the linear handler is 2-D only
        torch.nn.functional.linear(x, w)


class Experts(torch.nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.gate_up_proj = torch.nn.Parameter(torch.randn(E, 2 * I, H, dtype=torch.bfloat16))
        self.down_proj = torch.nn.Parameter(torch.randn(E, H, I, dtype=torch.bfloat16))


@pytest.mark.parametrize("fmt", FMTS)
def test_config_leaves_expert_rows_not_a_multiple_of_128_unquantized(fmt, caplog):
    """MXDynamicActivationMXWeightConfig on a 3-D parameter (through FqnToConfig) with N % 128 != 0 keeps it bf16 and
    says so; quantizing it would need expert tiles that straddle two experts' scale blocks."""
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig
    from ao_b200.quantization import FqnToConfig, quantize_

    cfg = MXDynamicActivationMXWeightConfig(activation_dtype=ELEM[fmt], weight_dtype=ELEM[fmt])
    m = Experts(2, 192, 96)   # gate_up_proj [2, 192, 192], down_proj [2, 192, 96]: N = 192 both
    with caplog.at_level(logging.INFO):
        quantize_(m, FqnToConfig({"gate_up_proj": cfg, "down_proj": cfg}), filter_fn=None)
    for p in (m.gate_up_proj, m.down_proj):
        assert type(p) is torch.nn.Parameter and p.dtype == torch.bfloat16
    assert caplog.text.count("Skipping MX quantization") == 2
