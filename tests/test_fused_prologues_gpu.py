"""SURVEY 8f-1: producer-fused activation quantizers (RMSNorm -> quant, SiLU * up -> quant) against the unfused
composition: the producer restated with torch ops at the HF rounding points (LlamaRMSNorm: fp32 statistics, cast to bf16,
times the bf16 weight; LlamaMLP: bf16(silu) * up in bf16) followed by this engine's per-token quantizer, which is itself
bit-exact against the oracle (tests/test_lowp_gpu.py).

SiLU-mul is elementwise: bit-exact.  RMSNorm reduces a row in fp32; a different summation order than torch's moves the
variance by ~1e-7 relative, which flips a bf16 rounding of the normalized value about once per 1e4 elements: codes may
differ by one step there, scales by one bf16 ulp (tolerance stated below)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rmsnorm_ref(x, w, eps):
    h = x.float()
    var = h.double().pow(2).mean(-1, keepdim=True).float()   # exact mean, then the reference's fp32 arithmetic
    return w * (h * torch.rsqrt(var + eps)).to(torch.bfloat16)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("M,K", [(1, 4096), (32, 4096), (5, 14336), (64, 1024)])
def test_silu_mul_quant_bit_exact(fmt, M, K):
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    gen = torch.Generator(device="cuda").manual_seed(M + K)
    gu = (torch.randn(M, 2 * K, device="cuda", generator=gen) * 2).to(torch.bfloat16)
    gate, up = gu[:, :K], gu[:, K:]          # column slices of one fused gate|up output: row pitch 2K
    if M > 1:                                # -0.0, NaN and inf in y, each in a row of its own; the others stay finite
        up[0, 1::7] = -0.0
        up[M // 2, 5] = float("nan")
        up[M - 1, 9] = float("inf")
    y = torch.nn.functional.silu(gate) * up
    q_ref, s_ref = (ops.int8_quantize_rowwise if fmt == 0 else ops.fp8_quantize_rowwise)(y)
    q, s = ops.silu_mul_quantize_rowwise(gate, up, fmt)
    assert torch.equal(s, s_ref)
    assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8))


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("M,K", [(1, 4096), (32, 4096), (7, 8192)])
def test_rmsnorm_quant_matches_composition(fmt, M, K):
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    gen = torch.Generator(device="cuda").manual_seed(7 * M + K)
    x = (torch.randn(M, K, device="cuda", generator=gen) * 3).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(K, device="cuda", generator=gen)).to(torch.bfloat16)
    y = _rmsnorm_ref(x, w, 1e-5)
    q_ref, s_ref = (ops.int8_quantize_rowwise if fmt == 0 else ops.fp8_quantize_rowwise)(y)
    q, s = ops.rmsnorm_quantize_rowwise(x, w, 1e-5, fmt)
    # scales: equal, or one bf16 ulp apart when the row maximum sits on a rounding boundary
    assert torch.allclose(s, s_ref, rtol=2 ** -7, atol=0)
    assert (s == s_ref).float().mean() >= 0.9
    same_rows = (s == s_ref).reshape(-1)
    if fmt == 0:
        d = (q.int() - q_ref.int()).abs()[same_rows]
        assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 2e-3
    else:
        a, b = q.float()[same_rows], q_ref.float()[same_rows]
        assert float((a != b).float().mean()) < 2e-3
        assert torch.allclose(a, b, rtol=0.13, atol=2 ** -9)   # at most one e4m3 step


def test_fused_prologue_feeds_the_linear():
    """RMSNorm -> fp8 quant -> fp8 rowwise linear in two launches equals the three-launch composition."""
    import ao_b200  # noqa: F401

    ops = torch.ops.ao_b200
    torch.manual_seed(0)
    M, K, N = 16, 4096, 1024
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    g = torch.ones(K, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    wq, ws = ops.fp8_quantize_rowwise(w)
    xq, xs = ops.rmsnorm_quantize_rowwise(x, g, 1e-5, 1)
    y = ops.fp8_rowwise_linear(xq, xs.reshape(-1), wq, ws.reshape(-1), None)
    ref = _rmsnorm_ref(x, g, 1e-5).float() @ w.float().t()
    sq = 20 * torch.log10(ref.norm() / (ref - y.float()).norm())
    assert sq > 24.0
