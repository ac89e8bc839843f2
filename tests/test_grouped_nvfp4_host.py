"""CPU tests of the NVFP4 expert GEMM (torch._grouped_mm on 3-D NVFP4Tensor weights):

* the Meta shapes of torch.ops.ao_b200.nvfp4_grouped_mm / nvfp4_fakequant_grouped and their C-ABI argument checks
  (before any CUDA call);
* the grouped schedule (tests/grouped_nvfp4_model.py) at the nvfp4 token-tile widths 16 .. 128, on random and malformed offs:
  row coverage, the bounds of every weight and scale-tile read, the device-side grid;
* the arithmetic of the per-expert blocked scales: the tile the kernel loads for expert e's n-tile t is row block
  e * N / 128 + t of the stacked scales, and that is the reference's to_blocked of the [E * N, K / 16] scales;
* Grouped<Nvfp4Fmt> has no stack frame and its static schedule tables fit beside the ring;
* the NVFP4Tensor pieces torch._grouped_mm goes through (3-D dequantize, transpose) and the config's 3-D rules.
"""
import ctypes
import os
import random

import pytest
import torch

import grouped_model as gm
import grouped_nvfp4_model as gnm
import streamk_model as sk
from test_decode_residency import LIB, RESERVED_PER_CTA, SMEM_PER_SM
from test_grouped_schedule import _cum, _offs_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
def test_meta_shapes():
    import ao_b200  # noqa: F401

    x = torch.empty(37, 512, dtype=torch.bfloat16, device="meta")
    offs = torch.empty(8, dtype=torch.int32, device="meta")
    xhat, xs = torch.ops.ao_b200.nvfp4_fakequant_grouped(x, offs)
    assert xhat.shape == (37, 512) and xhat.dtype == torch.bfloat16 and xs.shape == (37,) and xs.dtype == torch.float32
    wq = torch.empty(8, 256, 256, dtype=torch.uint8, device="meta")
    ws = torch.empty(8, 64, 128, dtype=torch.uint8, device="meta")
    y = torch.ops.ao_b200.nvfp4_grouped_mm(x, xs, wq, ws, torch.empty(8, device="meta"), offs)
    assert y.shape == (37, 256) and y.dtype == torch.bfloat16 and y.device.type == "meta"


def _lib():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    return lib


def test_grouped_mm_c_abi_argument_validation_without_gpu():
    lib = _lib()
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    f = lib.ao_nvfp4_grouped_mm
    f.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    one = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first

    def call(M=4, K=256, E=8, N=256, ptrs=(one,) * 6, ws=one, xs=one):
        x, wq, wsc, pts, offs, y = ptrs
        return f(x, xs, M, K, wq, wsc, pts, E, N, offs, y, ws, 1 << 20, None)

    assert call(K=192) == -1 and b"K=192" in lib.ao_b200_last_error()
    assert call(N=144) == -1 and b"N=144" in lib.ao_b200_last_error()
    assert call(E=0) == -1 and b"E=0" in lib.ao_b200_last_error()
    assert call(E=1025) == -1 and b"E=1025" in lib.ao_b200_last_error()
    assert call(E=1024, N=2**21) == -1 and b"int32" in lib.ao_b200_last_error()
    assert call(M=-1) == -1 and b"bad sizes" in lib.ao_b200_last_error()
    for i in range(6):
        ptrs = [one] * 6
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in lib.ao_b200_last_error(), i
    assert call(ws=None) == -1 and b"null pointer" in lib.ao_b200_last_error()
    assert call(ptrs=(ctypes.c_void_p(24),) + (one,) * 5) == -1 and b"16-byte" in lib.ao_b200_last_error()
    # no tokens: nothing to do, nothing dereferenced
    assert call(M=0, ptrs=(None,) * 6, ws=None, xs=None) == 0


def test_fakequant_c_abi_argument_validation_without_gpu():
    lib = _lib()
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    f = lib.ao_nvfp4_fakequant_grouped
    f.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, vp, vp]
    one = ctypes.c_void_p(16)

    def call(M=4, K=256, ldx=256, E=8, ptrs=(one,) * 5):
        x, offs, xhat, xs, amax = ptrs
        return f(x, ldx, M, K, offs, E, xhat, xs, amax, None)

    assert call(K=200, ldx=200) == -1 and b"K=200" in lib.ao_b200_last_error()
    assert call(E=0) == -1 and b"E=0" in lib.ao_b200_last_error()
    assert call(ldx=100) == -1 and b"ldx=100" in lib.ao_b200_last_error()
    for i in range(5):
        ptrs = [one] * 5
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in lib.ao_b200_last_error(), i
    assert call(M=0, ptrs=(None,) * 5) == 0


# ------------------------------------------------------------------------------------------------ schedule
SHAPES = [(128, 1024), (256, 512), (640, 1024), (128, 16384)]


def _check(offs, M, N, K, grid, sm=132):
    p = gnm.plan(offs, M, N, K, grid=grid, sm=sm)
    E = len(offs)
    assert N % sk.ROWS == 0 and p.n_tiles == N // sk.ROWS
    end = p.ends[-1]
    assert 0 <= end <= M
    assert p.G <= p.G_host and p.U <= p.U_bound and p.G <= max(p.U, 0)
    if p.U == 0:
        assert p.G == 0 and end == 0
        return p
    covered = [[0] * p.n_tiles for _ in range(end)]
    col_blocks = -(-(K // 16) // 4)
    for t in range(p.U // p.KT):
        e, row0, row_end, n_tile = p.tile(t)
        assert 0 <= e < E and 0 <= row0 < row_end <= M
        assert (p.ends[e - 1] if e > 0 else 0) <= row0 < p.ends[e] == row_end
        # the weight box (128 rows from e*N + 128*n_tile) lies inside expert e's rows: no tile tail when N % 128 == 0
        row = e * N + n_tile * sk.ROWS
        assert e * N <= row and row + sk.ROWS <= (e + 1) * N
        # its two scale tiles per chunk: row block row / 128, column blocks 2kc, 2kc + 1 of the stacked scales
        rb = row // sk.ROWS
        assert rb == e * (N // sk.ROWS) + n_tile < E * N // sk.ROWS
        assert rb * col_blocks + 2 * (p.KT - 1) + 1 < (E * N // sk.ROWS) * col_blocks
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
    for t, (owner, contribs) in p.owners.items():
        for c in contribs:
            assert c < p.G and p.ctas[c] and p.ctas[c][0].tile == t and p.ctas[c][0].kind == sk.CONTRIB
    return p


@pytest.mark.parametrize("N,K", SHAPES)
def test_schedule_invariants_nvfp4_widths(N, K):
    widths = set()
    cases = _offs_cases()
    rng = random.Random(99)
    for _ in range(20):   # larger routings: the 128-token tile with several m-blocks per expert
        E = rng.choice([1, 4, 8, 64])
        rows = [rng.choice([0, 1, 63, 64, 127, 128, 129, 300]) for _ in range(E)]
        cases.append((list(_cum(rows)), max(1, sum(rows) + rng.choice([0, 5]))))
    for offs, M in cases:
        for G in (None, 1, 2, 3, 7, 64, 131, 132, 500):
            widths.add(_check(offs, M, N, K, G).width)
    assert widths == {16, 32, 64, 128}, widths


def test_gpu_cases_reach_every_segment_kind_and_width():
    import test_grouped_nvfp4_gpu as suite

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


# ------------------------------------------------------------------------------------------------ scale layout
def test_stacked_blocked_scales_are_the_reference_layout():
    """Each expert's blocked [N, K/16] scales one after the other == to_blocked of the [E*N, K/16] scales (N % 128 == 0);
    the 512-byte tile (row block e*N/128 + t, column block c) holds expert e's rows 128t .. 128t+127, scales 4c .. 4c+3."""
    from ao_b200.prototype.mx_formats.utils import to_blocked

    g = torch.Generator().manual_seed(0)
    for E, N, K in [(3, 128, 128), (4, 256, 512), (2, 384, 1024)]:
        s = torch.randint(0, 256, (E, N, K // 16), generator=g, dtype=torch.int32).to(torch.uint8)
        stacked = torch.cat([to_blocked(s[e]) for e in range(E)])
        assert torch.equal(stacked, to_blocked(s.reshape(E * N, K // 16)))
        cb = K // 64
        tiles = stacked.reshape(-1, 512)
        for e in range(E):
            for t in range(N // 128):
                for c in range(cb):
                    tile = tiles[(e * N // 128 + t) * cb + c]
                    r = torch.arange(128)
                    for j in range(4):   # blocked offset of (row r, scale j): (r % 32) * 16 + (r // 32) * 4 + j
                        assert torch.equal(tile[(r % 32) * 16 + (r // 32) * 4 + j], s[e, 128 * t + r, 4 * c + j])


# ------------------------------------------------------------------------------------------------ residency
TABLE_BYTES = 4 * (1024 + 1025)   # s_end[MAX_EXPERTS] + s_mbp[MAX_EXPERTS + 1]


def test_grouped_tables_fit_beside_the_ring():
    for n_mma in (16, 32, 64, 128):
        _, ctas, _, _ = sk.ring("nvfp4", n_mma, grouped=True)
        smem = sk.ring_smem("nvfp4", n_mma, grouped=True)
        assert ctas == 1
        assert smem + TABLE_BYTES <= 227 * 1024 and smem + TABLE_BYTES + RESERVED_PER_CTA <= SMEM_PER_SM, n_mma


def test_grouped_nvfp4_kernels_have_no_stack():
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
        m = re.search(r"Function (\S*GroupedINS_5nvf4w8Nvfp4Fmt\S*?Li(\d+)E\S*):", line)
        if m:
            fn = int(m.group(2))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            found[fn] = (int(m.group(1)), int(m.group(2)))
        fn = None
    assert sorted(found) == [16, 32, 64, 128], found
    for n_mma, (reg, stack) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<Nvfp4Fmt>, {n_mma}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (n_mma, reg)   # one CTA of 384 threads per SM


# ------------------------------------------------------------------------------------------------ tensor and config
def _nvfp4_3d(E, N, K, pts, g, swizzled=False):
    from ao_b200.prototype.mx_formats import NVFP4Tensor
    from ao_b200.prototype.mx_formats.utils import to_blocked

    q = torch.randint(0, 256, (E, N, K // 2), generator=g, dtype=torch.int32).to(torch.uint8)
    s = torch.randint(0x20, 0x50, (E, N, K // 16), generator=g, dtype=torch.int32).to(torch.uint8)
    if swizzled:
        s = torch.stack([to_blocked(s[e]).reshape(32 * (N // 128), -1) for e in range(E)])
    return NVFP4Tensor(q, s.view(torch.float8_e4m3fn), 16, torch.bfloat16, pts, None, swizzled)


@pytest.mark.parametrize("swizzled", [False, True])
def test_3d_dequantize_and_transpose(swizzled):
    """A 3-D NVFP4Tensor dequantizes expert by expert as the 2-D tensor of that expert does, with its own scale; the
    transpose is a view whose shape, dequantize and qdata are the transposes of the original's."""
    from ao_b200.prototype.mx_formats import NVFP4Tensor

    g = torch.Generator().manual_seed(1)
    E, N, K = 3, 128, 128
    pts = torch.tensor([0.5, 3.0, 1e-3]).view(E, 1, 1)
    w = _nvfp4_3d(E, N, K, pts, g, swizzled)
    assert w.shape == (E, N, K)
    dq = w.dequantize()
    for e in range(E):
        w2 = NVFP4Tensor(w.qdata[e], w.scale[e], 16, torch.bfloat16, pts.reshape(-1)[e], None, swizzled)
        assert torch.equal(dq[e], w2.dequantize())
    t = w.transpose(-2, -1)
    assert isinstance(t, NVFP4Tensor) and t.shape == (E, K, N) and t.qdata.stride(-2) < t.qdata.stride(-1)
    assert torch.equal(t.qdata.transpose(-2, -1), w.qdata) and t.per_tensor_scale is w.per_tensor_scale
    assert torch.equal(t.dequantize(), dq.transpose(-2, -1))
    with pytest.raises(AssertionError):
        NVFP4Tensor(w.qdata, w.scale, 16, torch.bfloat16, torch.ones(E), None, swizzled)   # [E] is not [E, 1, 1]


def test_grouped_mm_handler_rejects_unsupported_forms():
    from ao_b200.prototype.mx_formats.nvfp4_tensor import QuantizeTensorToNVFP4Kwargs

    g = torch.Generator().manual_seed(2)
    E, N, K = 4, 128, 128
    w = _nvfp4_3d(E, N, K, torch.ones(E, 1, 1), g, swizzled=True)
    x = torch.randn(16, K, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    with pytest.raises(NotImplementedError):   # weight-only: out of scope
        torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)
    w.act_quant_kwargs = QuantizeTensorToNVFP4Kwargs(use_dynamic_per_tensor_scale=False, is_swizzled_scales=True)
    with pytest.raises(NotImplementedError):   # static activation scales: out of scope
        torch._grouped_mm(x, w.transpose(-2, -1), offs=offs)
    w.act_quant_kwargs = QuantizeTensorToNVFP4Kwargs(use_dynamic_per_tensor_scale=True, is_swizzled_scales=True)
    with pytest.raises(NotImplementedError):   # mat_b must be the transposed view of the stored weight
        torch._grouped_mm(x, w, offs=offs)
    with pytest.raises(NotImplementedError):   # the linear handler is 2-D only
        torch.nn.functional.linear(x, w)


class Experts(torch.nn.Module):
    def __init__(self, E, K, N):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(E, N, K, dtype=torch.bfloat16))


def test_config_3d_rules(caplog):
    """3-D weights need the dynamic per-tensor (per-expert) scale, and N % 128 == 0 and K % 128 == 0; other shapes stay
    unquantized with a log line."""
    import logging

    from ao_b200.prototype.mx_formats import NVFP4DynamicActivationNVFP4WeightConfig
    from ao_b200.quantization import quantize_

    flt = lambda mod, fqn: isinstance(mod, Experts)   # noqa: E731
    with pytest.raises(NotImplementedError):
        quantize_(Experts(2, 128, 128), NVFP4DynamicActivationNVFP4WeightConfig(use_dynamic_per_tensor_scale=False),
                  filter_fn=flt)
    for K, N in [(128, 144), (192, 128)]:
        m = Experts(2, K, N)
        with caplog.at_level(logging.INFO):
            quantize_(m, NVFP4DynamicActivationNVFP4WeightConfig(), filter_fn=flt)
        assert type(m.weight) is torch.nn.Parameter and m.weight.dtype == torch.bfloat16
        assert "Skipping NVFP4 quantization" in caplog.text
