"""Static int8 activations on the GPU: the quantizer bit for bit against the reference's torch ops run on the same GPU
(every bf16 value, scales from subnormal to huge, zero points at both ends, reduce_range, each pre-scale dtype, row-strided
x) and against the reference's codes in tests/golden/int8_static.npz; the linear bit for bit against the reference's CUDA
recipe restated with torch, under forced stream-K grids, and within one bf16 step of the reference's CPU outputs; the
quantize handler end to end (the reference's own test case), launch count, CUDA-graph replay with the scale changed in
place, a PDL chain, and F.linear on a selected expert of a 3-D weight."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


def bits(t):
    return t.contiguous().view(torch.int16)


def sqnr(ref, got):
    ref, got = ref.float(), got.float()
    d = (ref - got).norm()
    return float("inf") if d == 0 else float(20 * torch.log10(ref.norm() / d))


def ref_codes(x, scale, zp, pre, qmin, qmax):
    """The reference's ops (int8_tensor.py:280-294, :212-230; quant_primitives.py:480-485) as they run on CUDA."""
    if pre is not None:
        x = x * pre
    s = scale.reshape(-1, 1)
    z = torch.zeros_like(s, dtype=torch.int8) if zp is None else zp.reshape(-1, 1)
    return torch.clamp(torch.round(x * (1.0 / s)) + z, qmin, qmax).to(torch.int8)


def ref_linear(xq, xs, xzp, wq, ws, bias, asym):
    """The reference's CUDA recipe (int8_tensor.py:305-359, kernels.py:114-144) restated with torch: the int32 sums of
    torch._int_mm (computed exactly in fp64 here, so any M is allowed), * the fp32 x scale, rounded to bf16, the
    zero-point correction, * the fp32 w scale in fp32, + bias, one rounding."""
    acc = (xq.double() @ wq.double().t()).to(torch.int32)
    y = (acc * xs.reshape(-1, 1)).to(torch.bfloat16)
    if asym:
        corr = (xzp.reshape(-1, 1).float() * xs.reshape(-1, 1)) * wq.sum(dim=-1).float()
        y = y - corr.to(torch.bfloat16)
    y = y * ws.reshape(-1)
    if bias is not None:
        y = y + bias
    return y.to(torch.bfloat16)


# ---------------------------------------------------------------- the quantizer
SCALES = [1e-30, 2.0**-3, 1.0, 3.0e38, 1.5 * 2.0**127, 1e-40, 0.0173]   # tiny, tie-making, 1, huge, 1/s subnormal, subnormal s


def every_bf16(M=64):
    return torch.arange(65536, dtype=torch.int32, device=DEV).to(torch.int16).view(torch.bfloat16).reshape(M, -1)


def pre_scales(K, g):
    p = torch.rand(K, generator=g, device=DEV) * 4 - 2
    p[::7] = 2.0 ** torch.randint(-3, 4, (len(p[::7]),), generator=g, device=DEV).float()
    p[3::97] = 0.0
    return {"none": None, "bf16": p.to(torch.bfloat16), "f32": p}


@pytest.mark.parametrize("pname", ["none", "bf16", "f32"])
def test_quantizer_every_bf16_value_against_the_reference_ops(ops, pname):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = every_bf16()
    M, K = x.shape
    pre = pre_scales(K, g)[pname]
    wide = torch.zeros(M, K + 64, dtype=torch.bfloat16, device=DEV)
    wide[:, 8:8 + K] = x
    views = {"dense": x, "strided": wide[:, 8:8 + K]}
    per_row_s = torch.tensor([SCALES[m % len(SCALES)] for m in range(M)], device=DEV)
    per_row_z = torch.tensor([(-128, 0, 5, 127)[m % 4] for m in range(M)], dtype=torch.int8, device=DEV)
    n = 0
    for rr in (False, True):
        qmin, qmax = (-64, 63) if rr else (-128, 127)
        for zp_v in (None, -128, 0, 5, 127):
            zp = None if zp_v is None else torch.tensor([[zp_v]], dtype=torch.int8, device=DEV)
            for s_v in SCALES:
                s = torch.tensor([[s_v]], dtype=torch.float32, device=DEV)
                want = ref_codes(x, s, zp, pre, qmin, qmax)
                for name, xv in views.items():
                    q, xs, xz = ops.int8_quantize_static(xv, s, zp, pre, qmin, qmax)
                    assert torch.equal(q, want), (rr, zp_v, s_v, name)
                    z = torch.zeros(1, dtype=torch.int8, device=DEV) if zp is None else zp
                    assert torch.equal(xs, s.reshape(1).expand(M)) and torch.equal(xz, z.reshape(1).expand(M))
                    n += 1
        # per-row scale and zero point
        want = ref_codes(x, per_row_s[:, None], per_row_z[:, None], pre, qmin, qmax)
        for xv in views.values():
            q, xs, xz = ops.int8_quantize_static(xv, per_row_s[:, None], per_row_z[:, None], pre, qmin, qmax)
            assert torch.equal(q, want) and torch.equal(xs, per_row_s) and torch.equal(xz, per_row_z)
    assert n == 2 * 5 * len(SCALES) * 2


def test_quantizer_reproduces_the_fixture_codes(ops):
    d = np.load(os.path.join(GOLDEN, "int8_static.npz"))
    for c, case in enumerate(json.loads(str(d["cases"]))):
        x = torch.from_numpy(d[f"s{case['shape']}_x"].view(np.int16)).view(torch.bfloat16).to(DEV)
        s = torch.from_numpy(d[f"c{c}_scale"]).to(DEV)
        zp = torch.from_numpy(d[f"c{c}_zp"]).to(DEV) if f"c{c}_zp" in d else None
        pre = None
        if f"c{c}_pre" in d:
            p = d[f"c{c}_pre"]
            pre = (torch.from_numpy(p.view(np.int16)).view(torch.bfloat16) if p.dtype == np.uint16 else torch.from_numpy(p)).to(DEV)
        qmin, qmax = (-64, 63) if case["reduce_range"] else (-128, 127)
        q, _, _ = ops.int8_quantize_static(x, s, zp, pre, qmin, qmax)
        assert np.array_equal(q.cpu().numpy(), d[f"c{c}_q"]), case


# ---------------------------------------------------------------- the linear
def _static_linear(K, N, act_gran, mapping, scale, zp=None, pre=None, bias=True, reduce_range=False, seed=0, weight=None,
                   w_gran=None):
    from ao_b200.quantization import Int8StaticActivationInt8WeightConfig, PerRow, quantize_

    torch.manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    if weight is not None:
        with torch.no_grad():
            lin.weight.copy_(weight)
    quantize_(lin, Int8StaticActivationInt8WeightConfig(act_quant_scale=scale, act_quant_zero_point=zp,
                                                        granularity=[act_gran, w_gran or PerRow()],
                                                        act_mapping_type=mapping,
                                                        reduce_range=reduce_range))
    lin.weight.act_pre_scale = pre
    return lin


@pytest.mark.parametrize("ctas", [0, 1, 3, 7, 132])
def test_linear_bit_exact_against_the_reference_recipe(ops, ctas):
    from ao_b200.quantization import MappingType, PerRow, PerTensor

    g = torch.Generator(device=DEV).manual_seed(2)
    M, K, N = 37, 1040, 328
    x = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16) * 3
    pre = (torch.rand(K, generator=g, device=DEV) + 0.5)
    try:
        ops.debug_set_streamk_ctas(ctas)
        for mapping in (MappingType.SYMMETRIC, MappingType.ASYMMETRIC):
            asym = mapping == MappingType.ASYMMETRIC
            for gran, scale, zp in ((PerTensor(), torch.tensor([[0.021]], device=DEV), torch.tensor([[-3]], dtype=torch.int8, device=DEV)),
                                    (PerRow(), torch.rand(M, 1, generator=g, device=DEV) * 0.05 + 0.01,
                                     torch.randint(-20, 20, (M, 1), generator=g, device=DEV).to(torch.int8))):
                for p in (None, pre.to(torch.bfloat16), pre):
                    for bias in (True, False):
                        lin = _static_linear(K, N, gran, mapping, scale, zp if asym else None, p, bias, seed=3)
                        w = lin.weight
                        with torch.no_grad():
                            y = lin(x)
                        xq = ref_codes(x, scale, zp if asym else None, p, -128, 127)
                        xs = scale.reshape(-1).expand(M).float()
                        xz = (zp if asym else torch.zeros(1, dtype=torch.int8, device=DEV)).reshape(-1).expand(M)
                        want = ref_linear(xq, xs, xz, w.qdata, w.scale.float(), lin.bias, asym)
                        assert torch.equal(bits(y), bits(want)), (mapping, gran, None if p is None else p.dtype, bias)
    finally:
        ops.debug_set_streamk_ctas(0)


def test_linear_within_one_bf16_step_of_the_fixture():
    from ao_b200.quantization import MappingType, PerRow, PerTensor

    d = np.load(os.path.join(GOLDEN, "int8_static.npz"))
    t = lambda a: torch.from_numpy(a.view(np.int16)).view(torch.bfloat16).to(DEV)
    for c, case in enumerate(json.loads(str(d["cases"]))):
        si = case["shape"]
        pre = None
        if f"c{c}_pre" in d:
            p = d[f"c{c}_pre"]
            pre = t(p) if p.dtype == np.uint16 else torch.from_numpy(p).to(DEV)
        zp = torch.from_numpy(d[f"c{c}_zp"]).to(DEV) if f"c{c}_zp" in d else None
        gran = PerTensor() if case["granularity"] == "PerTensor" else PerRow()
        lin = _static_linear(case["K"], case["N"], gran, MappingType[case["mapping"]],
                             torch.from_numpy(d[f"c{c}_scale"]).to(DEV), zp, pre, case["bias"], case["reduce_range"],
                             weight=t(d[f"s{si}_w"]), w_gran=gran)
        if case["bias"]:
            with torch.no_grad():
                lin.bias.copy_(t(d[f"s{si}_b"]))
        with torch.no_grad():
            y = lin(t(d[f"s{si}_x"])).float()
        want = t(d[f"c{c}_y"]).float()
        step = torch.maximum(want.abs(), torch.full_like(want, 2.0**-126)) * 2.0**-7
        assert bool(((y - want).abs() <= step).all()), case


# ---------------------------------------------------------------- handler end to end
@pytest.mark.parametrize("gran", ["PerRow", "PerTensor"])
@pytest.mark.parametrize("mapping", ["SYMMETRIC", "ASYMMETRIC"])
def test_static_with_dynamic_scales_equals_dynamic(gran, mapping):
    """The reference's TestInt8StaticQuant.test_static_activation_per_row_int8_weight, restated: scales taken from the
    dynamic quantizer make the static linear compute the dynamic linear exactly, eagerly and, for a symmetric mapping
    (custom ops only), under torch.compile(fullgraph=True).  Where inductor compiles torch ops (the dynamic per-tensor
    scale, the asymmetric epilogue) it may round intermediates differently; there, as in the reference, the compiled
    static and dynamic linears must be as accurate as each other."""
    import copy

    from ao_b200.quantization import (Int8DynamicActivationInt8WeightConfig, Int8StaticActivationInt8WeightConfig,
                                      Int8Tensor, MappingType, PerRow, PerTensor, quantize_)

    torch.compiler.reset()
    g = PerRow() if gran == "PerRow" else PerTensor()
    mt = MappingType[mapping]
    torch.manual_seed(4)
    x = torch.randn(128, 128, dtype=torch.bfloat16, device=DEV)
    model = nn.Linear(128, 128, bias=False).eval().to(device=DEV, dtype=torch.bfloat16)
    dyn, sta = copy.deepcopy(model), copy.deepcopy(model)
    quantize_(dyn, Int8DynamicActivationInt8WeightConfig(granularity=g, act_mapping_type=mt))
    kw = dyn.weight.act_quant_kwargs
    xt = Int8Tensor.from_hp(x, kw.granularity, mapping_type=kw.mapping_type, reduce_range=kw.reduce_range)
    zp = xt.zero_point.detach().clone() if xt.zero_point is not None else None
    quantize_(sta, Int8StaticActivationInt8WeightConfig(act_quant_scale=xt.scale.detach().clone(), act_quant_zero_point=zp,
                                                        granularity=g, act_mapping_type=mt))
    with torch.no_grad():
        d_eager, s_eager = dyn(x), sta(x)
        d_comp, s_comp = torch.compile(dyn, fullgraph=True)(x), torch.compile(sta, fullgraph=True)(x)
        base = model(x)
    assert torch.equal(bits(s_eager), bits(d_eager))
    if mt == MappingType.SYMMETRIC:
        assert torch.equal(bits(s_comp), bits(s_eager))
    assert abs(sqnr(base, s_comp) - sqnr(base, d_comp)) < 1 and sqnr(base, s_comp) > 30


def test_handler_moves_a_host_scale_to_the_device_and_empty_input():
    from ao_b200.quantization import MappingType, PerTensor

    lin = _static_linear(256, 64, PerTensor(), MappingType.ASYMMETRIC, torch.tensor([[0.05]]),
                         torch.tensor([[2]], dtype=torch.int8))
    assert lin.weight.act_quant_scale.is_cuda and lin.weight.act_quant_zero_point.is_cuda
    y = lin(torch.empty(0, 256, dtype=torch.bfloat16, device=DEV))
    assert y.shape == (0, 64) and y.dtype == torch.bfloat16
    y3 = lin(torch.randn(2, 3, 256, dtype=torch.bfloat16, device=DEV))   # a [1, 1] scale serves a 3-D input
    assert y3.shape == (2, 3, 64)


LAUNCHES = """
import sys, torch
sys.path.insert(0, {root!r})
from torch.profiler import ProfilerActivity, profile
from ao_b200.quantization import Int8StaticActivationInt8WeightConfig, PerRow, PerTensor, quantize_
K = 1024
lins = []
for pre_dtype in (None, torch.bfloat16, torch.float32):
    lin = torch.nn.Linear(K, 512, bias=True, device="cuda", dtype=torch.bfloat16)
    quantize_(lin, Int8StaticActivationInt8WeightConfig(act_quant_scale=torch.tensor([[0.02]], device="cuda"),
                                                        granularity=[PerTensor(), PerRow()]))
    if pre_dtype is not None:
        lin.weight.act_pre_scale = (torch.rand(K, device="cuda") + 0.5).to(pre_dtype)
    lins.append(lin)
x = torch.randn(8, K, dtype=torch.bfloat16, device="cuda")
with torch.no_grad():
    for lin in lins:
        lin(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # the first kernels of a session can go unrecorded: spin kernels go first, and only they are left out below
        for _ in range(2):
            torch.cuda._sleep(10000)
            torch.cuda.synchronize()
        for lin in lins:
            lin(x)
            torch.cuda.synchronize()
spans = sorted((e.time_range.start, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memcpy" not in e.name.lower() and "memset" not in e.name.lower() and "spin_kernel" not in e.name)
names = [n for _, n in spans]
assert len(names) == 6, names
assert all("int8_static_quant_kernel" in names[i] and "ts_gemm_kernel" in names[i + 1] for i in (0, 2, 4)), names
print("ok")
"""


def test_symmetric_static_linear_is_two_kernels():
    """Without, with a bf16 and with an fp32 pre-scale, one symmetric static linear is the quantizer and the GEMM:
    six kernels for the three, in one torch.profiler session.  The profiler runs in a process of its own, so that
    it attaches to nothing else the suite runs."""
    r = subprocess.run([sys.executable, "-c", LAUNCHES.format(root=ROOT)], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-3000:]


def test_cuda_graph_reads_the_scale_on_the_device():
    from ao_b200.quantization import MappingType, PerRow

    M, K = 16, 512
    scale = torch.full((M, 1), 0.03, device=DEV)
    lin = _static_linear(K, 256, PerRow(), MappingType.SYMMETRIC, scale, pre=torch.rand(K, device=DEV) + 0.5)
    x = torch.randn(M, K, dtype=torch.bfloat16, device=DEV)
    with torch.no_grad():
        lin(x)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = lin(x)
        graph.replay()
        torch.cuda.synchronize()
        first = y.clone()
        assert torch.equal(bits(first), bits(lin(x)))
        lin.weight.act_quant_scale.copy_(torch.linspace(0.01, 0.05, M, device=DEV)[:, None])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(y), bits(lin(x))) and not torch.equal(bits(y), bits(first))


def test_pdl_chain_matches_serialized():
    from ao_b200.quantization import MappingType, PerTensor

    ls = [_static_linear(2048, 2048, PerTensor(), MappingType.SYMMETRIC, torch.tensor([[0.05 * (i + 1)]], device=DEV),
                         pre=(torch.rand(2048, device=DEV) + 0.5).to(torch.bfloat16), seed=10 + i) for i in range(3)]
    with torch.no_grad():
        for M in (1, 32, 300):
            x = torch.randn(M, 2048, device=DEV, dtype=torch.bfloat16)
            chained = ls[2](ls[1](ls[0](x)))
            a = ls[0](x)
            torch.cuda.synchronize()
            b = ls[1](a)
            torch.cuda.synchronize()
            serial = ls[2](b)
            torch.cuda.synchronize()
            assert torch.equal(bits(chained), bits(serial)), f"M={M}"


def test_selected_expert_of_a_3d_static_weight():
    from ao_b200.quantization import Int8Tensor, MappingType, PerRow, PerTensor, QuantizeTensorToInt8Kwargs

    E, N, K = 3, 256, 512
    torch.manual_seed(5)
    W = torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16)
    kw = QuantizeTensorToInt8Kwargs(granularity=PerTensor(), mapping_type=MappingType.SYMMETRIC)
    attrs = dict(act_quant_kwargs=kw, act_quant_scale=torch.tensor([[0.02]], device=DEV),
                 act_pre_scale=(torch.rand(K, device=DEV) + 0.5).to(torch.bfloat16))
    w3 = Int8Tensor.from_hp(W, PerRow(), **attrs)
    x = torch.randn(9, K, device=DEV, dtype=torch.bfloat16)
    for e in range(E):
        w2 = Int8Tensor.from_hp(W[e], PerRow(), **attrs)
        assert torch.equal(bits(F.linear(x, w3[e])), bits(F.linear(x, w2))), e
