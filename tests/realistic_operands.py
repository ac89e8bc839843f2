"""Realistic operands for the quantized GEMMs, their fp64 references, an element-wise error envelope and a rounding
census against a model of each kernel's summation order.

The exact-operand tests (exact_operands.py) choose codes and scales so that nothing rounds; they cannot see scale
arithmetic done at too low a precision, the accumulation precision, or a wrong dequantization rounding.  Here the
operands come from Gaussian bf16 data (some rows with outliers 30-100x the row RMS) through the package's own
quantizers, so every scale has a full mantissa, and each output is checked three ways:

* reference r: the fp64 sum of the stored codes times their scales (the dequantization restated here, never through a
  package dequant kernel), then the epilogue of the format's recipe with every fp32 and bf16 rounding emulated exactly
  in fp64 (rne());
* envelope: every output lies between the epilogue applied to acc - tau S and to acc + tau S, S = sum_k |x_k||w_k|
  (dequantized, fp64).  The epilogues are monotone in acc, so this is |y - r| <= ulp_bf16(r) + tau S carried through
  every rounding of the recipe; tau comes from the format's documented arithmetic (tau_for()), not from GPU output;
* census: the fraction of outputs that differ from r (correctly rounded) and their mean signed error in ulps, against
  a model of the kernel's order computed in the same test, then the format's EPI_* steps.  e4m3 formats promote each
  128-k chunk: the tensor core's chunk partials added in fp32 in k order (add_chunks_f32).  The other formats keep
  one wgmma accumulator per segment: a truncating fp32 chain of k16 steps (chain_f32).  Integer sums are exact: there
  r must match bit for bit.

All helpers take fp64 tensors on any device, so the host test checks them on the CPU.
"""
import math

import torch

KCHUNK = 128


# ------------------------------------------------------------------------------------------------ exact rounding
def pow2(e):
    """2^e for an integer tensor, exactly (a table: torch.pow on CUDA rounds)."""
    table = torch.tensor([2.0**i for i in range(-200, 201)], dtype=torch.float64, device=e.device)
    return table[e.long().clamp(-200, 200) + 200]


def rne(x, bits, emin):
    """x (fp64) rounded to nearest-even with `bits` significant bits and no exponent below emin (frexp convention:
    quantum 2^(max(e, emin) - bits)); bf16: rne(x, 8, -125), fp32: rne(x, 24, -125), e4m3: rne(x, 4, -5).  No
    overflow handling: the values here stay in range."""
    _, e = torch.frexp(x)
    q = pow2(torch.clamp(e, min=emin) - bits)
    return torch.round(x / q) * q   # torch.round: half to even; x / q and the product are exact (powers of two)


def rtz32(x):
    """x (fp64) truncated toward zero to fp32's 24 significant bits."""
    _, e = torch.frexp(x)
    q = pow2(torch.clamp(e, min=-125) - 24)
    return torch.trunc(x / q) * q


def r16(x):
    return rne(x, 8, -125)


def r32(x):
    return rne(x, 24, -125)


def ulp16(x):
    """The spacing of bf16 numbers at |x| (x fp64)."""
    _, e = torch.frexp(x)
    return pow2(torch.clamp(torch.where(x == 0, torch.full_like(e, -125), e), min=-125) - 8)


def e4m3(x):
    """fp64 -> e4m3 (RNE, saturating at 448, the quantizers' clamp)."""
    return rne(x, 4, -5).clamp(-448.0, 448.0)


# ------------------------------------------------------------------------------------------------ epilogues
# Each takes the fp32 (or exact) sums acc [M, n] as fp64 and returns the bf16 outputs as fp64, with the kernel's
# roundings (ts_gemm.cuh, epilogue); bias is fp64 of the bf16 bias [n] or None.  rows: [M, 1], cols: [1, n].
def epi_f8(acc, x_scale, w_scale, bias):
    """EPI_F8: bf16(fma(acc, fp32(x_scale[m] * w_scale[n]), bias[n]))"""
    v = r32(acc) * r32(x_scale * w_scale) + (0.0 if bias is None else bias)
    return r16(r32(v))


def epi_float(acc, row_scale=None, out_scale=None, out_scale2=None, bias=None):
    """EPI_FLOAT: x = acc (* row_scale[m]); bf16(fma(x, fp32(out_scale * out_scale2), bias))"""
    x = r32(acc)
    if row_scale is not None:
        x = r32(x * row_scale)
    osc = torch.as_tensor(1.0 if out_scale is None else out_scale, dtype=torch.float64, device=acc.device)
    if out_scale2 is not None:
        osc = r32(osc * out_scale2)
    return r16(r32(x * osc + (0.0 if bias is None else bias)))


def epi_i8(acc, x_scale, w_scale, bias):
    """EPI_I8: bf16(fma(bf16(acc * x_scale[m]), w_scale[n], bias[n])) on exact int32 sums"""
    t = r16(r32(acc * x_scale))
    return r16(r32(t * w_scale + (0.0 if bias is None else bias)))


def epi_bf16_wscale(acc, w_scale, bias):
    """EPI_BF16_WSCALE (int8 weight-only): bf16(bf16(bf16(acc) * bf16(w_scale[n])) + bias[n])"""
    o = r16(r16(r32(acc)) * r16(w_scale))
    return o if bias is None else r16(o + bias)


def epi_bf16(acc, bias):
    """EPI_BF16 (fp8 weight-only, NF4, blockwise fp8): bf16(bf16(acc) + bias[n])"""
    o = r16(r32(acc))
    return o if bias is None else r16(o + bias)


def epi_f8_sparse(acc, x_scale, w_scale, bias):
    """EPI_F8_SPARSE: bf16(fma(fp32(acc * w_scale[n]), x_scale[m], bias[n]))"""
    t = r32(r32(acc) * w_scale)
    return r16(r32(t * x_scale + (0.0 if bias is None else bias)))


# ------------------------------------------------------------------------------------------------ tau
TAU_F32 = 2.0**-23   # one fp32 add: the tensor core's adder is not documented to round to nearest, so a truncating
                     # adder's unit error (2^-23, twice round-to-nearest's) bounds each add
TAU_E4M3 = 2.0**-13  # one e4m3 wgmma accumulation: the width of the tensor core's reduced-precision adder that the
                     # exact-operand premise assumes (exact_operands.premise)


def tau_for(kind, K, contributors):
    """Relative bound of |acc - exact| / S for a sum over K, split over `contributors` stream-K partials, each add an
    error of at most its unit times S (every partial sum is at most S):
    's32': exact.
    'f32' (no promotion): one wgmma accumulator per segment, a chain of K/16 k16 steps (chain_f32), each adding 16
    products; counted as 16 adds within a step and one per step, then one fp32 add per contributor and the
    epilogue's fp32 steps (3), each TAU_F32.
    'e4m3': each 128-k chunk's four k32 wgmmas chained in the reduced adder (TAU_E4M3 each, DESIGN §1), then the
    chunk's promotion, one fp32 add per chunk and per contributor and the epilogue's 3, each TAU_F32.
    'e4m3_chain' (2:4-sparse, no promotion): two k64 wgmma.sp per chunk over the whole K in the reduced adder, then
    the contributors and the epilogue in fp32."""
    KT = -(-K // KCHUNK)
    if kind == "s32":
        return 0.0
    if kind == "f32":
        return (16 + -(-K // 16) + contributors + 3) * TAU_F32
    if kind == "e4m3":
        return 4 * TAU_E4M3 + (KT + contributors + 3) * TAU_F32
    if kind == "e4m3_chain":
        return 2 * KT * TAU_E4M3 + (contributors + 3) * TAU_F32
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------ checks
def envelope(y, epi, acc, S, tau):
    """y (fp64 of the kernel's bf16 output) against [epi(acc - tau S), epi(acc + tau S)] (either order: a negative
    scale reverses it).  Returns (ratio, bad): ratio = max |y - r| / (distance from r to the bound on y's side), <= 1
    inside the envelope, with r = epi(acc); bad = the mask of outputs outside."""
    r = epi(acc)
    a, b = epi(acc - tau * S), epi(acc + tau * S)
    lo, hi = torch.minimum(a, b), torch.maximum(a, b)
    bad = (y < lo) | (y > hi) | torch.isnan(y)
    up = torch.where(y > r, (y - r) / (hi - r).clamp_min(1e-300), torch.zeros_like(y))
    dn = torch.where(y < r, (r - y) / (r - lo).clamp_min(1e-300), torch.zeros_like(y))
    ratio = float(torch.where(bad, torch.full_like(y, math.inf), torch.maximum(up, dn)).max()) if y.numel() else 0.0
    return ratio, bad


def census(y, r):
    """(miss rate, mean signed error in ulps) of y against the correctly rounded r (both fp64 of bf16 values): the
    signed error is taken along r's sign, so a scale that is too large or too small in magnitude moves it whatever the
    sign of each output."""
    miss = (y != r).double()
    err = (y - r) / ulp16(r) * torch.sign(r)
    return float(miss.mean()), float(err.mean()), float((err * err).mean())


def sigma6(p, n):
    """Six binomial standard deviations of a rate p over n outputs (p floored at 1/n)."""
    p = min(max(p, 1.0 / n), 1.0)
    return 6.0 * math.sqrt(p * (1.0 - p) / n + 1.0 / (n * n))


def census_bound(p_model, n):
    """The miss rate a kernel of the model's order may reach: the model's, plus six standard deviations of the
    difference of two binomial rates over the same n outputs (sqrt(2) times one rate's)."""
    return p_model + math.sqrt(2.0) * sigma6(p_model, n)


def bias_bound(sq_kernel, sq_model, n):
    """How far the kernel's mean signed error may sit from the model's: six standard deviations of the difference of
    the two means over n outputs (each output's squared error in ulps estimates its variance)."""
    return 6.0 * math.sqrt((sq_kernel + sq_model) / n + 1.0 / (n * n))


def check_census(y, r, model, n=None):
    """Asserts the census of y against the model's; returns a one-line report."""
    n = n or y.numel()
    pk, bk, sk = census(y, r)
    pm, bm, sm = census(model, r)
    lim = census_bound(pm, n)
    blim = bias_bound(sk, sm, n)
    rep = f"miss {pk:.5f} (model {pm:.5f}, bar {lim:.5f}) bias {bk:+.5f} (model {bm:+.5f}, bar +-{blim:.5f})"
    return pk <= lim and abs(bk - bm) <= blim, rep


# ------------------------------------------------------------------------------------------------ fp32 model
def chunk_sums_f32(X, W):
    """Per-128-k chunk sums of X [M, K] @ W [N, K]^T (values exact in fp32), each a fp32 matmul with TF32 off:
    [KT, M, N] fp32."""
    M, K = X.shape
    KT = -(-K // KCHUNK)
    pad = KT * KCHUNK - K
    Xc = torch.nn.functional.pad(X.float(), (0, pad)).reshape(M, KT, KCHUNK).transpose(0, 1)
    Wc = torch.nn.functional.pad(W.float(), (0, pad)).reshape(W.shape[0], KT, KCHUNK).permute(1, 2, 0)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return torch.bmm(Xc.contiguous(), Wc.contiguous())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32


def chain_f32(X, W, step=16):
    """One wgmma accumulator over the whole K, the order of the formats without promotion: each k16 step's products
    (exact in fp64) added to the fp32 accumulator by an adder that truncates (TAU_F32: the tensor core's adder is not
    documented to round to nearest, and truncation is the least accurate such adder).  Returns fp64 of the sums."""
    acc = torch.zeros(X.shape[0], W.shape[0], dtype=torch.float64, device=X.device)
    for k in range(0, X.shape[1], step):
        acc = rtz32(acc + X[:, k:k + step] @ W[:, k:k + step].t())
    return acc


def add_chunks_f32(parts, combine=None):
    """The chunks added in fp32 in k order (combine(acc, part, kc) -> new acc, fp32, for formats that scale each chunk
    as it is promoted); returns fp64 of the fp32 sums."""
    acc = None
    for kc in range(parts.shape[0]):
        if combine is not None:
            acc = combine(acc, parts[kc], kc)
        else:
            acc = parts[kc].clone() if acc is None else acc + parts[kc]
    return acc.double()


# ------------------------------------------------------------------------------------------------ operands
def realistic(rows, K, g, scale=1.0, outlier_rows=4):
    """Gaussian bf16 [rows, K] (std `scale`) with `outlier_rows` heavy-tailed rows: 8 entries each at 30-100x the row
    RMS, random signs."""
    dev = g.device
    x = torch.randn(rows, K, device=dev, generator=g) * scale
    for i in range(min(outlier_rows, rows)):
        r = int(torch.randint(0, rows, (1,), device=dev, generator=g))
        cols = torch.randint(0, K, (8,), device=dev, generator=g)
        mag = 30.0 + 70.0 * torch.rand(8, device=dev, generator=g)
        sign = torch.randint(0, 2, (8,), device=dev, generator=g) * 2 - 1
        x[r, cols] = mag * sign * x[r].pow(2).mean().sqrt()
    return x.to(torch.bfloat16)
