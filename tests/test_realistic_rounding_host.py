"""The helpers of the realistic-operand rounding tests (tests/realistic_operands.py) on the CPU: the exact roundings,
the envelope, the census and its binomial bound, and the fp32 model.  A correct fp32 matmul must pass every check; the
same matmul with a scale rounded to bf16, one output negated or one 128-k chunk dropped must each fail one."""
import math

import numpy as np
import pytest
import torch

import realistic_operands as ro

M, N, K = 64, 256, 2048


def test_rne_matches_the_hardware_conversions():
    g = torch.Generator().manual_seed(0)
    v = torch.randn(200000, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-140, 40, (200000,), generator=g).double())
    assert torch.equal(ro.r32(v), v.float().double())
    f = v.float()   # fp32 -> bf16 rounds once: the reference for r16 on fp32 values
    assert torch.equal(ro.r16(f.double()), f.to(torch.bfloat16).double())
    e = (f.clamp(-448, 448) * 0 + v.clamp(-448, 448)).float()
    assert torch.equal(ro.e4m3(e.double()), e.to(torch.float8_e4m3fn).double())
    b = torch.arange(0, 2**16, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).double()
    b = b[torch.isfinite(b) & (b != 0)]
    nxt = (b.float().view(torch.int32) + 2**16).view(torch.float32).double()   # the next bf16 away from zero
    assert torch.equal(ro.ulp16(b)[b.abs() < 2.0**127], (nxt - b).abs()[b.abs() < 2.0**127])


def operands(seed=0):
    g = torch.Generator().manual_seed(seed)
    x = ro.realistic(M, K, g).double()
    w = ro.realistic(N, K, g, scale=0.02, outlier_rows=8).double()
    xs = torch.rand(M, 1, generator=g, dtype=torch.float64).float().double() + 0.5
    ws = torch.rand(1, N, generator=g, dtype=torch.float64).float().double() * 1e-2
    b = torch.randn(1, N, generator=g).to(torch.bfloat16).double()
    return x, w, xs, ws, b


def kernel_like(x, w, xs, ws, b, scale_bf16=False, drop_chunk=None):
    """An fp32 GEMM in the kernel's order: 128-k chunk sums, the chunks added in fp32, EPI_F8."""
    parts = ro.chunk_sums_f32(x, w)
    if drop_chunk is not None:
        parts[drop_chunk] = 0
    acc = ro.add_chunks_f32(parts)
    sc = ro.r16(ro.r32(xs * ws)) if scale_bf16 else ro.r32(xs * ws)
    return ro.r16(ro.r32(acc * sc + b))


def run_checks(y, x, w, xs, ws, b):
    epi = lambda a: ro.epi_f8(a, xs, ws, b)
    acc = x @ w.t()
    S = x.abs() @ w.abs().t()
    ratio, bad = ro.envelope(y, epi, acc, S, ro.tau_for("f32", K, 1))
    ok, rep = ro.check_census(y, epi(acc), epi(ro.add_chunks_f32(ro.chunk_sums_f32(x, w))))
    return ratio, int(bad.sum()), ok, rep


def test_a_correct_fp32_gemm_passes():
    x, w, xs, ws, b = operands()
    # another fp32 order than the model's: one fp32 matmul over the whole K
    y = ro.r16(ro.r32((x.float() @ w.float().t()).double() * ro.r32(xs * ws) + b))
    ratio, nbad, ok, rep = run_checks(y, x, w, xs, ws, b)
    assert nbad == 0 and ratio <= 1.0, ratio
    assert ok, rep
    ratio, nbad, ok, rep = run_checks(kernel_like(x, w, xs, ws, b), x, w, xs, ws, b)
    assert nbad == 0 and ok, rep


def test_a_bf16_scale_product_fails_the_census():
    x, w, xs, ws, b = operands(1)
    _, _, ok, rep = run_checks(kernel_like(x, w, xs, ws, b, scale_bf16=True), x, w, xs, ws, b)
    assert not ok, rep


def test_one_negated_output_fails_the_envelope():
    x, w, xs, ws, b = operands(2)
    y = kernel_like(x, w, xs, ws, b)
    i, j = 5, 77
    assert y[i, j] != 0
    y[i, j] = -y[i, j]
    ratio, nbad, _, _ = run_checks(y, x, w, xs, ws, b)
    assert nbad == 1 and math.isinf(ratio)


def test_a_dropped_chunk_fails_the_envelope():
    x, w, xs, ws, b = operands(3)
    _, nbad, _, _ = run_checks(kernel_like(x, w, xs, ws, b, drop_chunk=7), x, w, xs, ws, b)
    assert nbad > M * N // 8   # a sixteenth of each sum missing: most outputs leave the envelope


def test_envelope_is_the_rounded_interval():
    acc = torch.tensor([[1.0, -3.0, 0.0]], dtype=torch.float64)
    S = torch.tensor([[2.0, 8.0, 1.0]], dtype=torch.float64)
    epi = lambda a: ro.r16(a)
    y = torch.tensor([[1.0 + 2.0**-7, -3.0, 0.0]], dtype=torch.float64)
    ratio, bad = ro.envelope(y, epi, acc, S, 2.0**-8)   # 1 +- 2^-7: one bf16 ulp either side
    assert not bad.any() and ratio == pytest.approx(1.0)
    y[0, 0] = 1.0 + 2.0**-6
    _, bad = ro.envelope(y, epi, acc, S, 2.0**-8)
    assert bad.tolist() == [[True, False, False]]


def test_census_and_binomial_bound():
    r = torch.ones(10000, dtype=torch.float64)
    y = r.clone()
    y[:100] = 1.0 + 2.0**-7                      # one ulp up in 1 % of the outputs
    p, bias, sq = ro.census(y, r)
    assert p == pytest.approx(0.01) and bias == pytest.approx(0.01) and sq == pytest.approx(0.01)
    p, bias, _ = ro.census(-y, -r)               # along r's sign: the same magnitude bias
    assert bias == pytest.approx(0.01)
    n = 10000
    assert ro.sigma6(0.01, n) == pytest.approx(6 * math.sqrt(0.01 * 0.99 / n + 1 / n**2))
    assert ro.census_bound(0.0, n) < 15 / n       # p = 0: a handful of flips at most
    # a binomial draw at the bound's own rate stays under it (one seeded draw per rate)
    rng = np.random.default_rng(0)
    for p0 in (1e-4, 1e-3, 1e-2):
        hits = rng.binomial(n, p0) / n
        assert hits <= ro.census_bound(p0, n)


def test_tau_follows_the_documented_arithmetic():
    assert ro.tau_for("s32", 4096, 9) == 0.0
    assert ro.tau_for("f32", 4096, 1) == (16 + 256 + 1 + 3) * 2.0**-23       # the k16 chain of one accumulator
    assert ro.tau_for("e4m3", 4096, 1) == 4 * 2.0**-13 + (32 + 1 + 3) * 2.0**-23
    assert ro.tau_for("e4m3_chain", 4096, 1) == 64 * 2.0**-13 + (1 + 3) * 2.0**-23


def test_the_truncating_chain_model_stays_in_the_envelope():
    x, w, xs, ws, b = operands(4)
    acc = ro.chain_f32(x, w)
    y = ro.epi_f8(acc, xs, ws, b)
    ratio, nbad, _, _ = run_checks(y, x, w, xs, ws, b)
    assert nbad == 0 and ratio <= 1.0


# ------------------------------------------------------------------------------------------------ the chain model
# The formats without promotion are compared with chain_f32, a truncating k16 chain that misses the correctly rounded
# output far more often than a round-to-nearest chunk model.  These cases show that it still rejects the bugs it is
# there to catch: an int4 dequantization rounded twice and a scale product carried in bf16.
GS = 128


def int4_case(seed):
    """bf16 activations x, int4 weights with full-mantissa bf16 s and z; W = bf16(fma(q - 8, s, z))"""
    g = torch.Generator().manual_seed(seed)
    x = ro.realistic(M, K, g).double()
    q = torch.randint(0, 16, (N, K), generator=g).double()
    s = (torch.rand(N, K // GS, generator=g, dtype=torch.float64) * 2e-3 + 1e-3).to(torch.bfloat16).double()
    z = (torch.randn(N, K // GS, generator=g, dtype=torch.float64) * 1e-2).to(torch.bfloat16).double()
    s, z = s.repeat_interleave(GS, 1), z.repeat_interleave(GS, 1)
    return x, q, s, z


def chain_census(y, x, w, epi):
    acc = x @ w.t()
    ratio, bad = ro.envelope(y, epi, acc, x.abs() @ w.abs().t(), ro.tau_for("f32", K, 1))
    ok, rep = ro.check_census(y, epi(acc), epi(ro.chain_f32(x, w)))
    return int(bad.sum()), ok, rep


def test_the_chain_model_passes_a_correct_int4_gemm():
    x, q, s, z = int4_case(5)
    w = ro.r16((q - 8) * s + z)
    epi = lambda a: ro.epi_float(a)
    y = epi(ro.chain_f32(x, w, step=32))   # another truncating chain: 32 products per step
    nbad, ok, rep = chain_census(y, x, w, epi)
    assert nbad == 0 and ok, rep


def test_the_chain_model_rejects_an_int4_double_rounding():
    x, q, s, z = int4_case(6)
    w = ro.r16((q - 8) * s + z)
    w_bad = ro.r16(ro.r16((q - 8) * s) + z)   # q * s rounded before z is added
    assert (w_bad != w).double().mean() > 0.05
    epi = lambda a: ro.epi_float(a)
    _, ok, rep = chain_census(epi(ro.chain_f32(x, w_bad)), x, w, epi)
    assert not ok, rep


def test_the_chain_model_rejects_a_bf16_scale():
    x, q, s, z = int4_case(7)
    w = ro.r16((q - 8) * s + z)
    osc = torch.tensor(0.7312345, dtype=torch.float64).float().double()
    epi = lambda a: ro.epi_float(a, out_scale=osc)
    _, ok, rep = chain_census(ro.epi_float(ro.chain_f32(x, w), out_scale=ro.r16(osc)), x, w, epi)
    assert not ok, rep
