"""CPU tests of the int8 expert GEMMs (torch._grouped_mm on 3-D Int8Tensor weights: torch.ops.ao_b200.int8_weight_grouped_mm
for Int8WeightOnlyConfig, int8_dyn_grouped_mm for Int8DynamicActivationInt8WeightConfig and
Int8StaticActivationInt8WeightConfig):

* the Meta shapes, the op schemas and the C-ABI argument checks (before any CUDA call);
* the grouped schedule at both formats' token tiles (16 .. 128) with N tails;
* the package's 3-D quantizer and a numpy restatement of the per-expert recipe against the reference's fixture;
* transpose and select of a 3-D Int8Tensor, the handler's rejections, the configs' 3-D rules, serialization;
* ts_gemm_kernel<Grouped<Int8WoFmt>, N> and <Grouped<SsFmt<KIND_I8>>, N> exist for every token tile and have no stack.
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

import grouped_model as gm
import streamk_model as sk
from test_decode_residency import LIB
from test_grouped_schedule import _cum, _offs_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FMTS = ("int8wo", "int8")


# ------------------------------------------------------------------------------------------------ ops: Meta and C ABI
def test_meta_shapes_and_schemas():
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    wq = torch.empty(8, 77, 160, dtype=torch.int8, device="meta")
    ws = torch.empty(8, 77, device="meta")
    offs = torch.empty(8, dtype=torch.int32, device="meta")
    y = ops.int8_weight_grouped_mm(torch.empty(37, 160, dtype=torch.bfloat16, device="meta"), wq, ws, offs)
    assert y.shape == (37, 77) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    y = ops.int8_dyn_grouped_mm(torch.empty(37, 160, dtype=torch.int8, device="meta"), torch.empty(37, device="meta"),
                                wq, ws, offs)
    assert y.shape == (37, 77) and y.dtype == torch.bfloat16 and y.device.type == "meta"
    assert str(ops.int8_weight_grouped_mm.default._schema).endswith(
        "(Tensor x, Tensor wq, Tensor w_scale, Tensor offs) -> Tensor")
    assert str(ops.int8_dyn_grouped_mm.default._schema).endswith(
        "(Tensor xq, Tensor x_scale, Tensor wq, Tensor w_scale, Tensor offs) -> Tensor")


def _abi():
    lib = ctypes.CDLL(LIB)
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    vp, i32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.ao_int8_weight_grouped_mm.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    lib.ao_int8_dyn_grouped_mm.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    return lib


def test_c_abi_argument_validation_without_gpu():
    lib = _abi()
    buf = np.zeros(64, np.uint8)
    a = (buf.ctypes.data + 15) & ~15   # host addresses stand in for device ones: never dereferenced
    one = ctypes.c_void_p(a)
    err = lib.ao_b200_last_error

    def wo(M=4, K=256, E=8, N=200, ptrs=(one,) * 6):
        x, wq, ws, offs, y, work = ptrs
        return lib.ao_int8_weight_grouped_mm(x, M, K, wq, ws, E, N, offs, y, work, 1 << 20, None)

    def dyn(M=4, K=256, E=8, N=200, ptrs=(one,) * 7):
        xq, xs, wq, ws, offs, y, work = ptrs
        return lib.ao_int8_dyn_grouped_mm(xq, xs, M, K, wq, ws, E, N, offs, y, work, 1 << 20, None)

    for f, n in ((wo, 6), (dyn, 7)):
        assert f(K=200) == -1 and b"K=200" in err()
        assert f(E=0) == -1 and b"E=0" in err()
        assert f(E=1025) == -1 and b"E=1025" in err()
        assert f(E=1024, N=2**21) == -1 and b"int32" in err()
        assert f(M=-1) == -1 and b"bad sizes" in err()
        assert f(N=0) == -1 and b"bad sizes" in err()
        assert f(K=0) == -1 and b"bad sizes" in err()
        for i in range(n):
            ptrs = [one] * n
            ptrs[i] = None
            assert f(ptrs=ptrs) == -1 and b"null pointer" in err(), (f, i)
        assert f(ptrs=(ctypes.c_void_p(a + 8),) + (one,) * (n - 1)) == -1 and b"16-byte aligned" in err()
        # no tokens: nothing to do, nothing dereferenced, no CUDA call (this process has no device)
        assert f(M=0, ptrs=(None,) * n) == 0
    # the weight-only op has no N rule (no TMA scale box): N = 77 passes the checks up to the null pointer
    assert wo(N=77, ptrs=(one,) * 5 + (None,)) == -1 and b"null pointer" in err()
    # int8 x int8: N % 8 == 0, the dense int8 rule
    assert dyn(N=77) == -1 and b"N=77" in err()
    assert dyn(N=204) == -1 and b"N=204" in err()
    assert dyn(N=136, ptrs=(one,) * 6 + (None,)) == -1 and b"null pointer" in err()


# ------------------------------------------------------------------------------------------------ schedule
def _check(fmt, offs, M, N, K, grid, sm=132):
    p = gm.plan(offs, M, N, K, grid=grid, sm=sm, fmt=fmt)
    E = len(offs)
    assert p.n_tiles == -(-N // sk.ROWS) and p.KT == -(-K // 128)
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
        # the weight box starts at row e*N + 128t of the [E*N, K] map, inside expert e's rows (any row: no N rule for
        # the weight-only format, which has no scale box)
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


SHAPES = [(200, 160), (77, 1024), (128, 4112), (1408, 2048), (14336, 4096)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("N,K", SHAPES)
def test_schedule_invariants_at_every_width(fmt, N, K):
    widths = set()
    cases = _offs_cases()
    rng = random.Random(13)
    for _ in range(20):
        E = rng.choice([1, 8, 64, 128])
        rows = [rng.choice([0, 1, 16, 33, 64, 128, 129, 300]) for _ in range(E)]
        cases.append((list(_cum(rows)), max(1, sum(rows) + rng.choice([0, 5]))))
    for offs, M in cases:
        for G in (None, 1, 3, 64, 132):
            widths.add(_check(fmt, offs, M, N, K, G).width)
    assert widths == {16, 32, 64, 128}, widths


def test_gpu_cases_reach_every_segment_kind_width_and_gather_boundary():
    import test_grouped_int8_gpu as suite

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
        # the staged-gather layouts: every staging width, owners below, at and above the ring's stage count
        staged = {w for w in sk.WIDTHS[fmt] if sk.ring(fmt, w, grouped=True)[3]}
        assert {w for w, _, _ in suite._staging_layouts(fmt)} == staged
        assert staged == ({16, 32, 64} if fmt == "int8wo" else {16, 32}), staged


def test_rings_one_cta_per_sm():
    for fmt in FMTS:
        for n_mma in (16, 32, 64, 128):
            _, ctas, stages, _ = sk.ring(fmt, n_mma, grouped=True)
            assert ctas == 1 and stages >= 2
            assert sk.ring_smem(fmt, n_mma, grouped=True) + 4 * (1024 + 1025) <= 227 * 1024


def test_grouped_int8_kernels_have_no_stack():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    found = {}
    fn = None
    for line in out.splitlines():
        m = re.search(r"Function (\S*GroupedINS_4lowp(9Int8WoFmt|5SsFmtILi0EEE)\S*?Li(\d+)E\S*):", line)
        if m:
            fn = (m.group(2), int(m.group(3)))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            found[fn] = (int(m.group(1)), int(m.group(2)))
        fn = None
    assert len(found) == 8 and {n for _, n in found} == {16, 32, 64, 128}, found
    for key, (reg, stack) in found.items():
        assert stack == 0, f"ts_gemm_kernel<Grouped<{key[0]}>, {key[1]}>: {stack} bytes of stack (register spills)"
        assert reg <= 168, (key, reg)   # one CTA of 384 threads per SM: 65536 / 384, rounded down to 8


# ------------------------------------------------------------------------------------------------ the fixture
VARIANTS = ("wo_PerRow", "wo_PerTensor", "dyn_PerRow", "static_PerTensor")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "int8_3d.npz"))


def golden_shapes(d):
    """(case, arrays) per shape of the fixture: weight, inputs, offs, static scale and pre-scale, and each variant's
    qdata, scale, block_size (stored once per weight granularity) and (per-row weights) outputs."""
    for c in json.loads(str(d["cases"])):
        s = c["shape"]
        a = {f: d[f"s{s}_{f}"] for f in ("w", "x", "xe", "offs", "pre", "act_scale")}
        for v in VARIANTS:
            wname = "PerTensor" if v == "wo_PerTensor" else "PerRow"
            for f in ("q", "scale", "block_size"):
                a[f"{v}_{f}"] = d[f"s{s}_{wname}_{f}"]
            for f in ("y", "ye"):
                if f"s{s}_{v}_{f}" in d:
                    a[f"{v}_{f}"] = d[f"s{s}_{v}_{f}"]
        yield c, a


def _bf16(bits):
    return torch.from_numpy(np.asarray(bits).view(np.int16).copy()).view(torch.bfloat16)


def _bits(t):
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def recipe(v, a, x):
    """The per-expert recipe restated: weight-only bf16(bf16(bf16(x q^T) * bf16(s))) from exact fp64 sums (the
    fixture's one-hot inputs make them exact in fp32); int8 activations (the package's CPU quantizer: PerRow, or the
    static [1, 1] scale on bf16(x * pre)) with exact integer sums and bf16(bf16(acc * s_x) * s_w).  Rows up to
    offs[-1]."""
    from ao_b200.quantization import Int8Tensor, PerRow, PerTensor

    q, s, offs = a[f"{v}_q"], a[f"{v}_scale"], a["offs"]
    E, N, _ = q.shape
    sw = torch.from_numpy(np.broadcast_to(s.reshape(-1) if s.size > 1 else s.reshape(1), (E * N,)).reshape(E, N).copy())
    xb = _bf16(x)
    if v.startswith("dyn"):
        xt = Int8Tensor.from_hp(xb, PerRow())
    elif v.startswith("static"):
        xt = Int8Tensor.from_hp(xb * _bf16(a["pre"]), PerTensor(), scale=torch.from_numpy(a["act_scale"]))
    out, start = [], 0
    for e in range(E):
        end = int(offs[e])
        if end > start:
            if v.startswith("wo"):
                acc = (xb[start:end].double() @ torch.from_numpy(q[e]).double().t()).float()
                y = (acc.to(torch.bfloat16).float() * sw[e].to(torch.bfloat16).float()).to(torch.bfloat16)
            else:
                acc = xt.qdata[start:end].long() @ torch.from_numpy(q[e]).long().t()
                sx = xt.scale.reshape(-1).float().expand(xb.shape[0])[start:end, None]
                y = ((acc.float() * sx).to(torch.bfloat16).float() * sw[e]).to(torch.bfloat16)
            out.append(y)
        start = max(start, end)
    return torch.cat(out)


def test_restatement_reproduces_the_reference(golden):
    """Bit for bit: the one-hot outputs of every variant and the random outputs of the int8-activation variants; the
    fixture has the cases it claims (an empty expert, rows after offs[-1], N and K tails)."""
    for c, a in golden_shapes(golden):
        for v in ("wo_PerRow", "dyn_PerRow", "static_PerTensor"):
            assert np.array_equal(_bits(recipe(v, a, a["xe"])), a[f"{v}_ye"]), (c, v)
            if not v.startswith("wo"):
                assert np.array_equal(_bits(recipe(v, a, a["x"])), a[f"{v}_y"]), (c, v)
            else:   # random bf16 inputs: the fp32 sum's order may move the first rounding by one step
                d = np.abs(_bits(recipe(v, a, a["x"])).astype(np.int32) - a[f"{v}_y"].astype(np.int32))
                assert d.max() <= 1, (c, v)
        assert "wo_PerTensor_y" not in a
    cases = [c for c, _ in golden_shapes(golden)]
    assert any(0 in c["rows"] for c in cases) and any(c["tail"] for c in cases)
    assert any(c["N"] % 128 for c in cases) and any(c["K"] % 128 for c in cases)


def test_package_quantizer_matches_the_fixture(golden):
    from ao_b200.quantization import Int8Tensor, PerRow, PerTensor

    for c, a in golden_shapes(golden):
        w = _bf16(a["w"])
        for v in VARIANTS:
            t = Int8Tensor.from_hp(w, PerTensor() if v == "wo_PerTensor" else PerRow())
            assert t.shape == (c["E"], c["N"], c["K"]) and t.dtype == torch.bfloat16
            assert list(t.block_size) == a[f"{v}_block_size"].tolist(), (c, v)
            assert np.array_equal(t.qdata.numpy(), a[f"{v}_q"]), (c, v)
            assert np.array_equal(t.scale.numpy(), a[f"{v}_scale"]), (c, v)


# ------------------------------------------------------------------------------------------------ tensor and handler
def _w3(E=4, N=200, K=160, gran=None, seed=0, **kw):
    from ao_b200.quantization import Int8Tensor, PerRow

    g = torch.Generator().manual_seed(seed)
    return Int8Tensor.from_hp(torch.randn(E, N, K, generator=g).to(torch.bfloat16), gran or PerRow(), **kw)


def _kw(granularity=None, **k):
    from ao_b200.quantization import PerRow, QuantizeTensorToInt8Kwargs

    return QuantizeTensorToInt8Kwargs(granularity=granularity or PerRow(), **k)


def test_transpose_and_select_views():
    """transpose swaps shape, qdata, scale, zero_point and block_size; twice gives back the stored form.  select(0, e)
    is expert e's 2-D tensor sharing the 3-D tensor's storage, with its scale and zero point; the activation fields
    travel with both views."""
    from ao_b200.quantization import Int8Tensor, PerTensor

    w = _w3(act_quant_kwargs=_kw(), act_pre_scale=torch.rand(160).to(torch.bfloat16))
    full = w.dequantize()
    t = w.transpose(-2, -1)
    assert type(t) is Int8Tensor and t.shape == (4, 160, 200) and list(t.block_size) == [1, 160, 1]
    assert t.qdata.stride(-2) < t.qdata.stride(-1) and t.scale.shape == (4, 1, 200) and t.zero_point.shape == (4, 1, 200)
    assert t.qdata.untyped_storage().data_ptr() == w.qdata.untyped_storage().data_ptr()
    assert t.act_quant_kwargs == w.act_quant_kwargs and t.act_pre_scale is w.act_pre_scale
    assert torch.equal(t.dequantize(), full.transpose(-2, -1))
    tt = t.transpose(-2, -1)
    assert tt.shape == w.shape and list(tt.block_size) == [1, 1, 160] and tt.qdata.stride() == w.qdata.stride()
    assert tt.scale.shape == w.scale.shape and torch.equal(tt.dequantize(), full)
    for e in range(4):
        we = w[e]
        assert type(we) is Int8Tensor and we.shape == (200, 160) and list(we.block_size) == [1, 160]
        assert we.scale.shape == (200, 1) and we.zero_point.shape == (200, 1) and torch.equal(we.dequantize(), full[e])
        assert we.act_pre_scale is w.act_pre_scale
    pt = _w3(gran=PerTensor(), seed=1)
    ptt = pt.transpose(-2, -1)
    assert ptt.scale.shape == (1, 1, 1) and list(ptt.block_size) == [4, 160, 200]
    assert torch.equal(ptt.dequantize(), pt.dequantize().transpose(-2, -1))
    nz = Int8Tensor(w.qdata, w.scale, w.block_size, w.dtype)   # no zero point: stays None
    assert nz.transpose(-2, -1).zero_point is None


def test_grouped_mm_handler_rejects_unsupported_forms():
    from ao_b200.quantization import Int8Tensor, MappingType, PerGroup, PerTensor

    x = torch.randn(16, 160, dtype=torch.bfloat16)
    offs = torch.tensor([4, 8, 12, 16], dtype=torch.int32)
    w = _w3()
    dyn = _w3(act_quant_kwargs=_kw())
    s11 = torch.full((1, 1), 0.02)
    for fn in (torch._grouped_mm, F.grouped_mm):
        with pytest.raises(AssertionError, match="offs is required"):
            fn(x, w.transpose(-2, -1))
        with pytest.raises(NotImplementedError, match="transposed"):
            fn(x, _w3(N=160), offs=offs)
        with pytest.raises(NotImplementedError, match="bias"):
            torch._grouped_mm(x, w.transpose(-2, -1), offs=offs, bias=torch.zeros(200, dtype=torch.bfloat16))
        for bad in (dict(out_dtype=torch.float32),):
            with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
                fn(x, w.transpose(-2, -1), offs=offs, **bad)
        with pytest.raises(NotImplementedError, match="bf16 mat_a and output"):
            fn(x.half(), w.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="2-D mat_a x 3-D mat_b"):
            fn(x.reshape(4, 4, 160), w.transpose(-2, -1), offs=offs)
        wg = Int8Tensor.from_hp(torch.randn(4, 200, 160).to(torch.bfloat16), PerGroup(32))
        with pytest.raises(NotImplementedError, match="PerGroup"):
            fn(x, wg.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="rowsum"):
            fn(x, _w3(act_quant_kwargs=_kw(mapping_type=MappingType.ASYMMETRIC)).transpose(-2, -1), offs=offs)
        static_zp = _w3(act_quant_kwargs=_kw(PerTensor()), act_quant_scale=s11,
                        act_quant_zero_point=torch.zeros(1, 1, dtype=torch.int8))   # decided by presence, not values
        with pytest.raises(NotImplementedError, match="rowsum"):
            fn(x, static_zp.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="each expert's own rows"):
            fn(x, _w3(act_quant_kwargs=_kw(PerTensor())).transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="calibration batch"):
            fn(x, _w3(act_quant_kwargs=_kw(), act_quant_scale=torch.full((16, 1), 0.02)).transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="N % 8 == 0"):
            fn(x, _w3(N=204, act_quant_kwargs=_kw()).transpose(-2, -1), offs=offs)
        # served forms on CPU tensors reach the CUDA-only ops and fail in the dispatcher
        with pytest.raises(NotImplementedError, match="int8_weight_grouped_mm"):
            fn(x, w.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="int8_weight_grouped_mm"):   # no N rule for weight-only
            fn(x, _w3(N=77).transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="int8_dyn_grouped_mm"):
            fn(x, dyn.transpose(-2, -1), offs=offs)
        with pytest.raises(NotImplementedError, match="int8_dyn_grouped_mm"):
            fn(x, _w3(act_quant_kwargs=_kw(PerTensor()), act_quant_scale=s11).transpose(-2, -1), offs=offs)
    # no rows: an empty output, no kernel
    y = torch._grouped_mm(x[:0], w.transpose(-2, -1), offs=offs)
    assert y.shape == (0, 200) and y.dtype == torch.bfloat16


def test_3d_serialization_round_trips():
    from ao_b200.prototype.safetensors.safetensors_support import flatten_tensor_state_dict, unflatten_tensor_state_dict
    from ao_b200.quantization import Int8Tensor, PerTensor

    cases = [_w3(3, 24, 64, seed=3), _w3(3, 24, 64, gran=PerTensor(), seed=4),
             _w3(3, 24, 64, seed=5, act_quant_kwargs=_kw())]
    for w in cases:
        buf = io.BytesIO()
        torch.save({"experts.w": w}, buf)
        buf.seek(0)
        r = torch.load(buf, weights_only=True)["experts.w"]
        flat, meta = flatten_tensor_state_dict({"experts.w": w})
        s, left = unflatten_tensor_state_dict(flat, meta)
        assert not left
        for g in (r, s["experts.w"]):
            assert type(g) is Int8Tensor and g.shape == (3, 24, 64) and g.act_quant_kwargs == w.act_quant_kwargs
            assert list(g.block_size) == list(w.block_size) and g.dtype == torch.bfloat16
            assert torch.equal(g.qdata, w.qdata) and torch.equal(g.scale, w.scale)
            assert torch.equal(g.transpose(-2, -1).dequantize(), w.dequantize().transpose(-2, -1))


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
    """The three int8 configs on 3-D parameters through FqnToConfig: K % 16 != 0 stays unquantized with a log line
    (and N % 8 != 0 for the int8-activation configs); the rest quantizes per row / tensor."""
    from ao_b200.quantization import (FqnToConfig, Int8DynamicActivationInt8WeightConfig, Int8StaticActivationInt8WeightConfig,
                                      Int8Tensor, Int8WeightOnlyConfig, PerRow, PerTensor, quantize_)

    s11 = torch.full((1, 1), 0.02)
    configs = [("weight only", Int8WeightOnlyConfig()), ("dynamic", Int8DynamicActivationInt8WeightConfig()),
               ("static", Int8StaticActivationInt8WeightConfig(act_quant_scale=s11, granularity=[PerTensor(), PerRow()]))]
    for what, cfg in configs:
        m = Block(2, 256, 200)   # down_proj K = 200
        caplog.clear()
        with caplog.at_level(logging.INFO):
            quantize_(m, FqnToConfig({"experts.down_proj": cfg}), filter_fn=None)
        assert type(m.experts.down_proj) is torch.nn.Parameter
        assert f"Skipping int8 {what}" in caplog.text and "(2, 256, 200)" in caplog.text
        quantize_(m, FqnToConfig({"experts.gate_up_proj": cfg}), filter_fn=None)
        w = m.experts.gate_up_proj
        assert isinstance(w, Int8Tensor) and w.shape == (2, 400, 256) and w.scale.shape == (2, 400, 1)
        assert list(w.block_size) == [1, 1, 256] and (w.act_quant_kwargs is None) == (what == "weight only")
        if what == "static":
            assert w.act_quant_scale.shape == (1, 1)
        if what != "weight only":   # N % 8 != 0: the int8 x int8 kernels' rule
            m2 = Block(2, 260, 128)   # down_proj N = 260 passes, gate_up_proj N = 256; an N = 100 expert skips
            m2.experts.down_proj = torch.nn.Parameter(torch.randn(2, 100, 128, dtype=torch.bfloat16))
            caplog.clear()
            with caplog.at_level(logging.INFO):
                quantize_(m2, FqnToConfig({"experts.down_proj": cfg}), filter_fn=None)
            assert type(m2.experts.down_proj) is torch.nn.Parameter and "(2, 100, 128)" in caplog.text
    m3 = Block(2, 256, 128)
    m3.experts.down_proj = torch.nn.Parameter(torch.randn(2, 100, 128, dtype=torch.bfloat16))
    cfg = Int8WeightOnlyConfig(granularity=PerTensor())
    quantize_(m3, FqnToConfig({"experts.gate_up_proj": cfg, "experts.down_proj": cfg}), filter_fn=None)
    for p in (m3.experts.gate_up_proj, m3.experts.down_proj):   # weight-only: any N
        assert isinstance(p, Int8Tensor) and p.scale.shape == (1, 1, 1) and list(p.block_size) == list(p.shape)
