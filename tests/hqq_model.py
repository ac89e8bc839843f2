"""A torch restatement of the HQQ int4 solver of ao_b200/csrc/int4_hqq.cu, for tests.

It follows the kernels operation by operation, with every fp32 operation a separate torch op (so nothing can be
contracted into an FMA) and every reduction in the kernels' order: the per-lane sums over j, the xor butterfly over
the 32 lanes, the in-order double sum of a block's 8 warps, the strided-then-tree double sum of decide_kernel.  Element
(group gi, j, lane) is w[gi*g + j*32 + lane].  It runs on whatever device the weight is on and returns, besides the
outputs, the fp32 state the kernels leave in their workspace (scale, zero, partial, Ctrl), so a test can pin the
iteration count and every zero point, not only what survives bf16 rounding.

Two things the kernel computes are not IEEE-specified: powf, and the sign of zero in fminf / fmaxf.  The signed-zero
order of the init min / max is restated explicitly (-0 < +0, as min.f32 / max.f32 do).  powf only matters where the
shrinkage is active: a solve is TIER 1 when at every executed iteration every |d| > 0 has inv_beta * |d|^-0.3 >=
|d| * (1 + 2^-16) in float64, so the relu is zero whatever the last bits of powf are and the restatement is exact on
any device.  Anything else (TIER 2) is exact only where `pow_fn` is the kernel's powf: torch.pow on the CUDA tensor
with an fp32 exponent is (neither build uses fast math), and it matches the kernel bit for bit on every shrink-active
case of test_hqq_exact_gpu.py (H100).  On the CPU, Tier 2 is a solve that differs in the last bits.

Mutation switches (tests use them to show the data can tell a fault apart): no_shrink (shr = 0), flip_sign
(we = -sign(d) * shr), extra_iters (that many zero updates after the iteration that stops, or after the 20th).
"""
import math
from dataclasses import dataclass, field

import numpy as np
import torch

WARPS = 8             # groups (warps) per block
ITERS = 20
BETA0, KAPPA = 10.0, 1.01
EXPONENT = -0.3       # lp_norm - 1, as an fp32 constant in the kernel
SCALE_CLAMP = 2e4
TIER1_SLACK = 1.0 + 2.0 ** -16


def default_pow(a):
    """powf(a, -0.3f) elementwise on a's device."""
    return torch.pow(a, torch.tensor(EXPONENT, dtype=torch.float32, device=a.device))


@dataclass
class Solve:
    q: torch.Tensor          # uint8 [N, K] codes
    scale: torch.Tensor      # bf16 [N, K/g]  1 / s
    zero: torch.Tensor       # bf16 [N, K/g]  (8 - z) / s
    s: torch.Tensor          # fp32 [G] workspace scale
    z: torch.Tensor          # fp32 [G] workspace zero
    partial: torch.Tensor    # float64 [nblocks] per-block error sums of the last executed iteration
    best: float
    stop: int
    iters: int
    active: list = field(default_factory=list)   # shrink-active elements (shr > 0) per executed iteration
    margin: float = math.inf  # min over executed iterations and |d| > 0 of inv_beta * |d|^-0.3 / |d| (float64)

    @property
    def tier1(self):
        return self.margin >= TIER1_SLACK


def nblocks_of(groups):
    return (groups + WARPS - 1) // WARPS


def workspace_layout(N, K, g):
    """(groups, nblocks, byte offset of partial, byte offset of Ctrl) of the kernel's workspace."""
    G = N * K // g
    nb = nblocks_of(G)
    off_partial = (2 * G * 4 + 15) // 16 * 16
    return G, nb, off_partial, off_partial + 8 * nb


def _signed_min_max(W):
    """fminf / fmaxf over each group with -0 < +0: a zero minimum is -0 when the group holds a -0, a zero maximum
    +0 when it holds a +0."""
    G = W.shape[0]
    flat = W.reshape(G, -1)
    mn, mx = flat.amin(dim=1), flat.amax(dim=1)
    negzero = ((flat == 0) & torch.signbit(flat)).any(dim=1)
    poszero = ((flat == 0) & ~torch.signbit(flat)).any(dim=1)
    zero = torch.zeros_like(mn)
    mn = torch.where(mn == 0, torch.where(negzero, -zero, zero), mn)
    mx = torch.where(mx == 0, torch.where(poszero, zero, -zero), mx)
    return mn, mx


def _butterfly(v):
    """warp_sum: v[l] = v[l] + v[l ^ o] for o = 16 .. 1; every lane ends with the same value."""
    lanes = torch.arange(32, device=v.device)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lanes ^ o]
    return v[:, 0]


def _quantize(W, s, z):
    """clamp(rint(W * s + z), 0, 15), each operation rounded on its own."""
    return torch.clamp(torch.round((W * s[:, None, None]) + z[:, None, None]), 0.0, 15.0)


def _block_partials(err, nb):
    """Per-block double sum of the 8 warp errors in warp order, from 0.0; missing warps of the last block add 0."""
    e = torch.zeros(nb * WARPS, dtype=torch.float32, device=err.device)
    e[: err.numel()] = err
    e = e.reshape(nb, WARPS).double()
    t = torch.zeros(nb, dtype=torch.float64, device=err.device)
    for i in range(WARPS):
        t = t + e[:, i]
    return t


def _decide_total(partial):
    """decide_kernel's sum: thread t adds partial[t], partial[t + 256], ... in double, then a tree fold o = 128 .. 1."""
    nb = partial.numel()
    rows = max(1, -(-nb // 256))
    p = torch.zeros(rows * 256, dtype=torch.float64, device=partial.device)
    p[:nb] = partial
    p = p.reshape(rows, 256)
    t = torch.zeros(256, dtype=torch.float64, device=partial.device)
    for r in range(rows):
        t = t + p[r]
    o = 128
    while o > 0:
        t = t[:o] + t[o:2 * o]
        o >>= 1
    return float(t[0].item())


def solve(w, g, pow_fn=None, no_shrink=False, flip_sign=False, extra_iters=0, max_iters=ITERS):
    """The HQQ solve of bf16 w [N, K] with groups of g along K, as the kernels compute it.  max_iters < 20 truncates
    the solve (what a stop decided on the host while a CUDA graph was captured would bake in)."""
    assert w.dtype == torch.bfloat16 and w.dim() == 2 and g in (32, 64, 128, 256)
    N, K = w.shape
    assert K % g == 0
    pow_fn = pow_fn or default_pow
    EPL = g // 32
    G = N * K // g
    nb = nblocks_of(G)
    numel = float(N) * float(K)
    W = w.contiguous().float().reshape(G, EPL, 32)

    # init_kernel
    mn, mx = _signed_min_max(W)
    s = torch.clamp(torch.div(torch.full_like(mn, 15.0), mx - mn), max=SCALE_CLAMP)
    z = torch.round(-mn * s)

    best, stop, iters = 1e4, 0, 0
    beta = BETA0
    partial = torch.zeros(nb, dtype=torch.float64, device=w.device)
    active, margin = [], math.inf
    remaining = None   # extra zero updates still to run after the solver stopped
    for it in range(max_iters + extra_iters):
        if remaining == 0:
            break
        inv_beta = float(np.float32(1.0 / beta))
        wq = _quantize(W, s, z)
        wr = torch.div(wq - z[:, None, None], s[:, None, None])
        d = W - wr
        a = torch.abs(d)
        pos = a > 0
        pw = pow_fn(a)
        shr = torch.where(pos, a - (inv_beta * pw), torch.zeros_like(a))
        shr = torch.clamp(shr, min=0.0)
        if no_shrink:
            shr = torch.zeros_like(shr)
        we = torch.where(d > 0, shr, -shr)
        if flip_sign:
            we = -we
        t = wq - ((W - we) * s[:, None, None])
        acc = torch.zeros(G, 32, dtype=torch.float32, device=w.device)
        err = torch.zeros(G, 32, dtype=torch.float32, device=w.device)
        for j in range(EPL):
            acc = acc + t[:, j, :]
            err = err + a[:, j, :]
        z = torch.div(_butterfly(acc), torch.full((G,), float(g), dtype=torch.float32, device=w.device))
        partial = _block_partials(_butterfly(err), nb)
        beta *= KAPPA
        if remaining is not None:
            remaining -= 1
            continue

        active.append(int((shr > 0).sum().item()))
        if bool(pos.any()):
            a64 = a[pos].double()
            ratio = inv_beta * torch.pow(a64, float(np.float32(EXPONENT))) / a64
            margin = min(margin, float(ratio.min().item()))
        cur = float(np.float32(_decide_total(partial) / numel))
        iters += 1
        if cur < best:
            best = cur
        else:
            stop = 1
        if stop or it == max_iters - 1:
            remaining = extra_iters

    # final_kernel
    q = _quantize(W, s, z).to(torch.uint8).reshape(N, K)
    s_inv = torch.div(torch.ones_like(s), s)
    scale = s_inv.to(torch.bfloat16).reshape(N, K // g)
    zero = ((torch.full_like(z, 8.0) - z) * s_inv).to(torch.bfloat16).reshape(N, K // g)
    return Solve(q=q, scale=scale, zero=zero, s=s, z=z, partial=partial, best=best, stop=stop, iters=iters,
                 active=active, margin=margin)


# ---------------------------------------------------------------------------------------------- test weights
# std 0.02 is LLM-scale (Tier 1); std 1 and 2 put a group's error past the point where the shrinkage switches on
STD = {"s002": 0.02, "s002_outlier": 0.02, "s1": 1.0, "s2": 2.0}


def weight(regime, N, K, seed):
    """bf16 [N, K] randn * std on the CPU (the same bits whatever device a test moves it to); the outlier regime
    scales every 3rd row's every 97th column by 12."""
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=gen) * STD[regime]
    if regime.endswith("outlier"):
        w[::3, ::97] *= 12.0
    return w.to(torch.bfloat16)


SPECIAL_GROUPS = ("constant", "zeros", "mixed_signed_zeros", "huge_outlier", "tiny_range", "subnormal_range",
                  "constant_negative", "negative_zeros")


def special_weight(g):
    """bf16 [4, 8g], std-0.02 groups except the 8 groups of row 0, one per SPECIAL_GROUPS entry: a nonzero constant
    and a zero range (the scale clamps to 2e4), +0 only, alternating +0 / -0, one element of 1000 among std-0.02 values,
    two values one bf16 ulp apart near 1e-3 (15 / range > 2e4), 0 and the smallest bf16 subnormal (15 / range
    overflows to inf), a negative constant, -0 only."""
    gen = torch.Generator().manual_seed(g)
    w = torch.randn(4, 8 * g, generator=gen) * 0.02
    r = w[0].view(8, g)
    r[0] = 0.37
    r[1] = 0.0
    r[2] = torch.tensor([0.0, -0.0]).repeat(g // 2)
    r[3, 5] = 1000.0
    r[4] = torch.tensor([1e-3, 1e-3 + 2.0 ** -17]).repeat(g // 2)
    r[5] = torch.tensor([0.0, 2.0 ** -133]).repeat(g // 2)
    r[6] = -2.5
    r[7] = -0.0
    return w.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------- solver tolerance
# Bars against a solve that differs in the last bits (libm powf, another summation order): a last-bit difference in a
# zero point can move a code on a rounding boundary, and a few groups then settle on the equivalent (q + 1, zero -
# scale).  Scales bit-exact; codes never more than one apart and <= 1 % different; zero points <= 3 % different in
# their bits, <= 1 % more than 0.01 step apart, none more than one step; mean |W - dequant| within 0.1 %.
BARS = {"code_max": 1, "code_frac": 1e-2, "zero_bits_frac": 3e-2, "zero_far_frac": 1e-2, "zero_steps_max": 1.0,
        "recon_rel": 1e-3}


def _bf16_f32(bits):
    return (np.asarray(bits).astype(np.uint32) << 16).view(np.float32)


def bar_report(w_bits, g, q, s, z, qr, sr, zr):
    """How far a solve (q, s, z: codes and bf16 bits) is from a reference solve (qr, sr, zr) of bf16 w_bits."""
    q, qr = np.asarray(q).astype(np.int32), np.asarray(qr).astype(np.int32)
    diff = np.abs(q - qr)
    steps = np.abs(_bf16_f32(z) - _bf16_f32(zr)) / _bf16_f32(sr)
    wf = _bf16_f32(w_bits).reshape(-1, g)

    def recon(qq, ss, zz):
        deq = (qq.reshape(-1, g).astype(np.float32) - 8.0) * _bf16_f32(ss).reshape(-1, 1) + _bf16_f32(zz).reshape(-1, 1)
        return float(np.abs(wf - deq).mean())

    e, er = recon(q, s, z), recon(qr, sr, zr)
    return {"scale_equal": bool(np.array_equal(s, sr)), "code_max": int(diff.max()), "code_frac": float((diff != 0).mean()),
            "zero_bits_frac": float((np.asarray(z) != np.asarray(zr)).mean()), "zero_far_frac": float((steps > 0.01).mean()),
            "zero_steps_max": float(steps.max()), "recon_rel": abs(e - er) / er}


def within_bars(rep, bars=BARS):
    return rep["scale_equal"] and all(rep[k] <= v for k, v in bars.items())


def _f64_to_bf16_bits(x):
    """Round float64 to bf16 bits, nearest-even, with one rounding: round to odd in fp32 first (24 bits leave room
    for the 8 of bf16), then nearest-even on the fp32 bits."""
    f = x.astype(np.float32)
    f = np.where(np.abs(f.astype(np.float64)) > np.abs(x), np.nextafter(f, np.float32(0)), f)
    b = f.view(np.uint32) | (f.astype(np.float64) != x).astype(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def dequant_tinygemm_bits(q, scale, zero, g):
    """bf16 bits of (q - 8) * scale + zero with one rounding (the __hfma of the tile-packed dequantisation); q uint8
    [N, K], scale / zero bf16 [N, K/g].  The float64 value is exact: (q - 8) * scale has at most 12 significant bits."""
    q = q.cpu().numpy().astype(np.float64)
    sf = np.repeat(scale.float().cpu().numpy().astype(np.float64), g, axis=1)
    zf = np.repeat(zero.float().cpu().numpy().astype(np.float64), g, axis=1)
    return _f64_to_bf16_bits((q - 8.0) * sf + zf)
