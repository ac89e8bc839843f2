"""Static e4m3 activations on the GPU: the quantizer bit for bit against the reference's torch ops run on the same GPU
(every bf16 value, scales from zero and subnormal to huge, per-tensor and per-row, row-strided x) and against the
reference's codes in tests/golden/fp8_static.npz; the linear bit for bit on exact operands against an fp64 restatement
and torch._scaled_mm under forced stream-K grids, with the output fake-quant bit for bit against the reference's ops
applied to the plain linear's output, and within one bf16 step of the reference's CPU outputs; the static config with
the dynamic config's own scale giving the dynamic config's bits (eager and compiled); launch count, CUDA-graph replay
with the scales changed in place, a PDL chain, and F.linear on a selected expert of a 3-D weight."""
import copy
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
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


def bits(t):
    return t.contiguous().view(torch.int16)


def codes(t):
    return t.contiguous().view(torch.uint8)


def ref_codes(x, scale):
    """The reference's _quantize_affine_float8 (quant_primitives.py:2271-2287) as it runs on CUDA tensors."""
    return (x.to(torch.float32) / scale.reshape(-1, 1)).clamp(min=-448.0, max=448.0).to(E4M3)


def ref_qdq(y, so):
    """The reference's output fake-quant (prototype_float8_tensor.py:461-472): from_hp(y, scale=so).dequantize()."""
    return (ref_codes(y, so).to(torch.float32) * so.reshape(-1, 1)).to(y.dtype)


# ---------------------------------------------------------------- the quantizer
SCALES = [2.0 ** -4, 0.0173, 1.0, 0.0, 1e-40, 1e-30, 3e38, 1.5 * 2.0 ** 127]   # zero, subnormal, tiny, huge


def every_bf16(M=64):
    return torch.arange(65536, dtype=torch.int32, device=DEV).to(torch.int16).view(torch.bfloat16).reshape(M, -1)


def test_quantizer_every_bf16_value_against_the_reference_ops(ops):
    x = every_bf16()
    M, K = x.shape
    wide = torch.zeros(M, K + 64, dtype=torch.bfloat16, device=DEV)
    wide[:, 8:8 + K] = x
    views = {"dense": x, "strided": wide[:, 8:8 + K]}
    for s_v in SCALES:
        s = torch.tensor([[s_v]], dtype=torch.float32, device=DEV)
        want = codes(ref_codes(x, s))
        for name, xv in views.items():
            q, xs = ops.fp8_quantize_static(xv, s)
            assert torch.equal(codes(q), want), (s_v, name)
            assert torch.equal(xs, s.reshape(1).expand(M))
    per_row = torch.tensor([SCALES[m % len(SCALES)] for m in range(M)], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    per_row[::3] = torch.rand(len(per_row[::3]), generator=g, device=DEV) * 0.1
    want = codes(ref_codes(x, per_row[:, None]))
    for xv in views.values():
        q, xs = ops.fp8_quantize_static(xv, per_row[:, None])
        assert torch.equal(codes(q), want) and torch.equal(xs, per_row)


def test_quantizer_reproduces_the_fixture_codes(ops):
    d = np.load(os.path.join(GOLDEN, "fp8_static.npz"))
    for q, case in enumerate(json.loads(str(d["qcases"]))):
        x = torch.from_numpy(d[f"q{q}_x"].view(np.int16)).view(torch.bfloat16).to(DEV)
        s = torch.from_numpy(d[f"q{q}_scale"]).to(DEV)
        got = codes(ops.fp8_quantize_static(x, s)[0]).cpu().numpy()
        want = d[f"q{q}_q"]
        nan_g, nan_w = (got & 0x7F) == 0x7F, (want & 0x7F) == 0x7F   # the CPU gives 0/0 a negative NaN
        assert np.array_equal(nan_g, nan_w) and np.array_equal(got[~nan_g], want[~nan_w]), case


# ---------------------------------------------------------------- the linear
def _weight(wq, ws, gran, act_scale, out_scale=None):
    """A PrototypeFloat8Tensor on given codes and scales, as the config's handler builds it."""
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import QuantizeTensorToFloat8Kwargs
    from ao_b200.quantization.utils import get_block_size

    kw = QuantizeTensorToFloat8Kwargs(granularity=gran)
    return PrototypeFloat8Tensor(wq, ws, act_quant_scale=act_scale, output_act_quant_scale=out_scale,
                                 block_size=list(get_block_size(wq.shape, gran)), act_quant_kwargs=kw,
                                 dtype=torch.bfloat16, output_act_quant_kwargs=None if out_scale is None else kw)


def _exact_operands(M, K, N, gran, g):
    """Integer e4m3 codes in [-8, 8] and power-of-two scales: every product and partial sum is exact in fp32, so the
    result does not depend on the summation order (any stream-K split), and x = code * s quantizes back to the code."""
    from ao_b200.quantization import PerTensor

    def ints(*shape):
        return torch.randint(-8, 9, shape, generator=g, device=DEV).float()

    rows_x, rows_w = (1, 1) if isinstance(gran, PerTensor) else (M, N)
    sx = 2.0 ** torch.randint(-6, -1, (rows_x, 1), generator=g, device=DEV).float()
    sw = 2.0 ** torch.randint(-9, -4, (rows_w, 1), generator=g, device=DEV).float()
    xc, wc = ints(M, K), ints(N, K)
    x = (xc * sx).to(torch.bfloat16)
    bias = (torch.randn(N, generator=g, device=DEV) * 4).to(torch.bfloat16)
    return x, xc, sx, wc.to(E4M3), sw, bias


def _fp64_linear(xc, sx, wc, sw, bias):
    acc = xc.double() @ wc.double().t()
    y = acc * sx.double().reshape(-1, 1) * sw.double().reshape(1, -1)
    if bias is not None:
        y = y + bias.double()
    return y.float().to(torch.bfloat16)


@pytest.mark.parametrize("ctas", [0, 1, 3, 7, 132])
def test_linear_bit_exact_on_exact_operands(ops, ctas):
    from ao_b200.quantization import PerRow, PerTensor

    g = torch.Generator(device=DEV).manual_seed(2)
    try:
        ops.debug_set_streamk_ctas(ctas)
        for M, K, N in ((37, 1040, 336), (5, 4096, 128), (130, 272, 48)):
            for gran in (PerTensor(), PerRow()):
                x, xc, sx, wq, sw, b = _exact_operands(M, K, N, gran, g)
                w = _weight(wq, sw, gran, sx)
                for bias in (b, None):
                    with torch.no_grad():
                        y = F.linear(x, w, bias)
                    what = (M, K, N, type(gran).__name__, bias is not None)
                    assert torch.equal(bits(y), bits(_fp64_linear(xc, sx, wq.float(), sw, bias))), what
                    sa = sx.reshape(()) if sx.numel() == 1 else sx
                    sb = sw.reshape(()) if sw.numel() == 1 else sw.reshape(1, -1)
                    want = torch._scaled_mm(xc.to(E4M3), wq.t(), sa, sb, bias=bias, out_dtype=torch.bfloat16,
                                            use_fast_accum=True)
                    assert torch.equal(bits(y), bits(want)), what
                    # the output fake-quant: the reference's ops on the plain output; scales that saturate a quarter of
                    # the outputs, and per token
                    amax = y.float().abs().amax()
                    for so in ((amax / 448 * 0.75).reshape(1, 1),
                               torch.rand(M, 1, generator=g, device=DEV) * amax / 448 + amax / 2000):
                        wo = _weight(wq, sw, gran, sx, so)
                        with torch.no_grad():
                            yo = F.linear(x, wo, bias)
                        assert torch.equal(bits(yo), bits(ref_qdq(y, so))), (*what, so.numel())
    finally:
        ops.debug_set_streamk_ctas(0)


def test_output_fake_quant_edges(ops):
    """A zero output scale (0/0 = NaN, y/0 = +-448 * 0 ... as the reference computes it), a subnormal and a huge one."""
    from ao_b200.quantization import PerTensor

    g = torch.Generator(device=DEV).manual_seed(3)
    x, xc, sx, wq, sw, b = _exact_operands(16, 512, 64, PerTensor(), g)
    y = F.linear(x, _weight(wq, sw, PerTensor(), sx), b)
    for s_v in (0.0, 1e-40, 3e38, 2.0 ** -10):
        so = torch.tensor([[s_v]], device=DEV)
        got = F.linear(x, _weight(wq, sw, PerTensor(), sx, so), b)
        want = ref_qdq(y, so)
        assert torch.equal(torch.isnan(got), torch.isnan(want)), s_v
        assert torch.equal(bits(got)[~torch.isnan(got)], bits(want)[~torch.isnan(want)]), s_v


def test_linear_within_one_bf16_step_of_the_fixture():
    from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig, PerTensor, quantize_

    d = np.load(os.path.join(GOLDEN, "fp8_static.npz"))
    t = lambda a: torch.from_numpy(a.view(np.int16)).view(torch.bfloat16).to(DEV)
    for c, case in enumerate(json.loads(str(d["cases"]))):
        si = case["shape"]
        lin = nn.Linear(case["K"], case["N"], bias=case["bias"], device=DEV, dtype=torch.bfloat16)
        with torch.no_grad():
            lin.weight.copy_(t(d[f"s{si}_w"]))
            if case["bias"]:
                lin.bias.copy_(t(d[f"s{si}_b"]))
        so = torch.from_numpy(d[f"c{c}_oscale"]) if case["qdq"] else None
        quantize_(lin, Float8StaticActivationFloat8WeightConfig(act_quant_scale=torch.from_numpy(d[f"c{c}_scale"]),
                                                                granularity=PerTensor(), output_act_quant_scale=so))
        assert np.array_equal(codes(lin.weight.qdata).cpu().numpy(), d[f"s{si}_PerTensor_wq"])
        with torch.no_grad():
            y = lin(t(d[f"s{si}_x"])).float()
        want = t(d[f"c{c}_y"]).float()
        # one bf16 step, plus what the tensor core's fast accumulation within a 128-k chunk may lose against the CPU's
        # exact sums where the bias cancels them: 2^-13 of the sum of |products| (bound)
        xq = (t(d[f"s{si}_x"]).float() / lin.weight.act_quant_scale).clamp(-448, 448).to(E4M3).float()
        bound = (xq.abs() @ lin.weight.qdata.float().abs().t()) * lin.weight.act_quant_scale * lin.weight.scale
        step = torch.maximum(want.abs(), torch.full_like(want, 2.0 ** -126)) * 2.0 ** -7 + bound * 2.0 ** -13
        if case["qdq"]:   # a moved output can cross an e4m3 rounding boundary: one e4m3 step
            step = step + want.abs() * 2.0 ** -3 + so.item() * 2.0 ** -9
        assert bool(((y - want).abs() <= step).all()), case


# ---------------------------------------------------------------- handler end to end
@pytest.mark.parametrize("gran", ["PerTensor", "PerRow"])
def test_static_with_dynamic_scales_equals_dynamic(gran):
    """The reference's static-vs-dynamic SQNR test made exact: the static config given the dynamic quantizer's own scale
    computes the dynamic config's bits, eagerly and under torch.compile(fullgraph=True)."""
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Float8StaticActivationFloat8WeightConfig,
                                      Float8Tensor, PerRow, PerTensor, quantize_)

    torch.compiler.reset()
    g = PerRow() if gran == "PerRow" else PerTensor()
    torch.manual_seed(4)
    x = torch.randn(128, 256, dtype=torch.bfloat16, device=DEV)
    model = nn.Linear(256, 128, bias=True).eval().to(device=DEV, dtype=torch.bfloat16)
    dyn, sta = copy.deepcopy(model), copy.deepcopy(model)
    quantize_(dyn, Float8DynamicActivationFloat8WeightConfig(granularity=g))
    s = Float8Tensor.from_hp(x, E4M3, g).scale.detach().clone()
    quantize_(sta, Float8StaticActivationFloat8WeightConfig(act_quant_scale=s, granularity=g))
    assert torch.equal(codes(sta.weight.qdata), codes(dyn.weight.qdata)) and torch.equal(sta.weight.scale, dyn.weight.scale)
    with torch.no_grad():
        d_eager, s_eager = dyn(x), sta(x)
        s_comp = torch.compile(sta, fullgraph=True)(x)
    assert torch.equal(bits(s_eager), bits(d_eager))
    assert torch.equal(bits(s_comp), bits(s_eager))


def test_handler_moves_host_scales_to_the_device_empty_and_3d_input():
    from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig, quantize_

    lin = nn.Linear(256, 64, device=DEV, dtype=torch.bfloat16)
    quantize_(lin, Float8StaticActivationFloat8WeightConfig(act_quant_scale=torch.tensor([[0.05]]),
                                                            output_act_quant_scale=torch.tensor([[0.01]])))
    assert lin.weight.act_quant_scale.is_cuda and lin.weight.output_act_quant_scale.is_cuda
    y = lin(torch.empty(0, 256, dtype=torch.bfloat16, device=DEV))
    assert y.shape == (0, 64) and y.dtype == torch.bfloat16
    x3 = torch.randn(2, 3, 256, dtype=torch.bfloat16, device=DEV)
    y3 = lin(x3)   # a [1, 1] scale serves a 3-D input
    assert y3.shape == (2, 3, 64) and torch.equal(bits(y3.reshape(6, 64)), bits(lin(x3.reshape(6, 256))))


LAUNCHES = """
import sys, torch
sys.path.insert(0, {root!r})
from torch.profiler import ProfilerActivity, profile
from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig, PerRow, PerTensor, quantize_
M, K = 8, 1024
lins = []
for gran in (PerTensor(), PerRow()):
    for qdq in (False, True):
        s = torch.full((1, 1) if isinstance(gran, PerTensor) else (M, 1), 0.02, device="cuda")
        lin = torch.nn.Linear(K, 512, bias=True, device="cuda", dtype=torch.bfloat16)
        quantize_(lin, Float8StaticActivationFloat8WeightConfig(act_quant_scale=s, granularity=gran,
                                                                output_act_quant_scale=s * 10 if qdq else None))
        lins.append(lin)
x = torch.randn(M, K, dtype=torch.bfloat16, device="cuda")
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
assert len(names) == 8, names
assert all("fp8_static_quant_kernel" in names[i] and "ts_gemm_kernel<ao::lowp::F8StaticFmt" in names[i + 1]
           for i in (0, 2, 4, 6)), names
print("ok")
"""


def test_static_linear_is_two_kernels():
    """PerTensor and PerRow, with and without the output fake-quant: each linear is the quantizer and the GEMM, eight
    kernels for the four, in one torch.profiler session of a process of its own."""
    r = subprocess.run([sys.executable, "-c", LAUNCHES.format(root=ROOT)], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-3000:]


def test_cuda_graph_reads_the_scales_on_the_device():
    from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig, PerRow, quantize_

    M, K = 16, 512
    lin = nn.Linear(K, 256, device=DEV, dtype=torch.bfloat16)
    quantize_(lin, Float8StaticActivationFloat8WeightConfig(act_quant_scale=torch.full((M, 1), 0.03, device=DEV),
                                                            granularity=PerRow(),
                                                            output_act_quant_scale=torch.full((M, 1), 0.01, device=DEV)))
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
        for attr in ("act_quant_scale", "output_act_quant_scale"):
            getattr(lin.weight, attr).copy_(torch.linspace(0.005, 0.05, M, device=DEV)[:, None])
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(bits(y), bits(lin(x))) and not torch.equal(bits(y), bits(first)), attr
            first = y.clone()


def test_pdl_chain_matches_serialized():
    from ao_b200.quantization import Float8StaticActivationFloat8WeightConfig, quantize_

    ls = []
    for i in range(3):
        torch.manual_seed(10 + i)
        lin = nn.Linear(2048, 2048, device=DEV, dtype=torch.bfloat16)
        quantize_(lin, Float8StaticActivationFloat8WeightConfig(
            act_quant_scale=torch.tensor([[0.002 * (i + 1)]], device=DEV),
            output_act_quant_scale=torch.tensor([[0.001]], device=DEV) if i == 1 else None))
        ls.append(lin)
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
    from ao_b200.prototype.quantization import PrototypeFloat8Tensor
    from ao_b200.quantization import PerRow, QuantizeTensorToFloat8Kwargs

    E, N, K = 3, 256, 512
    torch.manual_seed(5)
    W = torch.randn(E, N, K, device=DEV, dtype=torch.bfloat16)
    kw = QuantizeTensorToFloat8Kwargs(granularity=PerRow())
    attrs = dict(act_quant_kwargs=kw, act_quant_scale=torch.full((9, 1), 0.02, device=DEV),
                 output_act_quant_scale=torch.full((9, 1), 0.01, device=DEV), output_act_quant_kwargs=kw)
    w3 = PrototypeFloat8Tensor.from_hp(W, E4M3, PerRow(), **attrs)
    x = torch.randn(9, K, device=DEV, dtype=torch.bfloat16)
    for e in range(E):
        w2 = PrototypeFloat8Tensor.from_hp(W[e], E4M3, PerRow(), **attrs)
        assert torch.equal(bits(F.linear(x, w3[e])), bits(F.linear(x, w2))), e
