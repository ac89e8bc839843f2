"""Every quantized GEMM on realistic operands (Gaussian bf16 with outlier rows, quantized by the package's own
quantizers, so every scale has a full mantissa): an element-wise error envelope and a rounding census against fp64
(tests/realistic_operands.py).  The exact-operand tests cannot see a scale product carried in bf16, a chunk partial
rounded before it is promoted, a dequantization that rounds in the wrong place or a stream-K partial rounded on its way
to the owner; each of those moves far more outputs off the correctly rounded value than a correct fp32 sum does.

Shapes: the Llama-3-8B projections at 1, 4, 32, 33 and 200 tokens (each token count with one projection, all four
projections covered), ragged expert offsets for the grouped GEMMs, and forced stream-K grids that split every tile
of the o projection over 2 to 5 contributors (owner gathers included).
"""
import zlib

import pytest
import torch

import realistic_operands as ro
from exact_operands import sparse_compress

pytestmark = pytest.mark.gpu
DEV = "cuda"

PROJ = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}
SHAPES = [(1, "qkv"), (4, "o"), (32, "gate_up"), (33, "down"), (200, "qkv")]
GRIDS = [37, 100, 132]   # at M = 32 on the o projection (1024 units): 2, 4 and 5 contributors per tile
FORCED = (32, "o")
E2M1 = [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, -0.0, -0.5, -1.0, -1.5, -2.0, -3.0, -4.0, -6.0]


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


@pytest.fixture
def grid(ops):
    """ops.debug_set_streamk_ctas, reset to the default grid afterwards."""
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


class Seg:
    """One GEMM of a case (a dense linear, or one expert / batch of a grouped one): rows [r0, r1) of the output,
    the dequantized operands X [m, K] and W [n, K] (fp64), the epilogue epi(acc) -> fp64 of bf16, and (e4m3 formats) the
    model's chunk partials parts() -> [KT, m, n] fp32 with an optional per-chunk combine (realistic_operands.add_chunks_f32)
    and alt(), a second comparator."""

    def __init__(self, r0, r1, X, W, epi, parts=None, combine=None, alt=None):
        self.r0, self.r1, self.X, self.W, self.epi, self.parts, self.combine = r0, r1, X, W, epi, parts, combine
        self.alt = alt   # e4m3 with rowwise-expressible scales: torch._scaled_mm's bf16 output of the segment


# The blockwise quantizers compute their scales in bf16 (the reference's rule on bf16 inputs), but the GEMMs take fp32
# scales: widened by this factor, every scale has a full fp32 mantissa, so a scale the kernel rounds to bf16 shows.
WIDEN = 1.0 + 2.0**-11 + 2.0**-19


def e4m3_parts(xq, wq):
    """The tensor core's own e4m3 chunk partials: cuBLAS's fp8 GEMM on one 128-k chunk (unit scales, fp32 out), the
    wgmma chain the kernel promotes from; [KT, M, N] fp32."""
    one = torch.ones((), device=DEV)
    return torch.stack([torch._scaled_mm(xq[:, k:k + 128].contiguous(), wq[:, k:k + 128].contiguous().t(), scale_a=one,
                                         scale_b=one, out_dtype=torch.float32) for k in range(0, xq.shape[1], 128)])


def e4m3_chain(xq, wq):
    """One e4m3 wgmma chain over the whole K (no promotion): cuBLAS's fp8 GEMM with fast accumulation, [1, M, N]."""
    one = torch.ones((), device=DEV)
    return torch._scaled_mm(xq, wq.t(), scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=True)[None]


def bias_for(N, g):
    return torch.randn(N, device=DEV, generator=g).to(torch.bfloat16)


def b64(b):
    return None if b is None else b.double()[None, :]


def col(v):
    return v.double().reshape(-1, 1)


def row(v):
    return v.double().reshape(1, -1)


def weights(N, K, g):
    return ro.realistic(N, K, g, scale=0.02, outlier_rows=8)


def unblocked(quant, t):
    """(codes, plain scales, blocked scales) of one MX / NVFP4 quantizer call pair."""
    q, s = quant(t, False)
    qb, sb = quant(t, True)
    assert torch.equal(q.view(torch.uint8), qb.view(torch.uint8))
    return q, s, sb


def fp4_values(q, s_plain, block, scale_of):
    lut = torch.tensor(E2M1, dtype=torch.float64, device=DEV)
    v = torch.stack([lut[(q & 15).long()], lut[(q >> 4).long()]], -1).reshape(q.shape[0], -1)
    return v * scale_of(s_plain).repeat_interleave(block, 1)


def e8m0(s):
    return ro.pow2(s.view(torch.uint8).long() - 127)


def e4m3_bytes(s):
    return s.view(torch.float8_e4m3fn).double()


# ------------------------------------------------------------------------------------------------ dense builders
def build(ops, op, M, N, K, seed=0):
    """(run() -> y [M, N] bf16, [Seg], accumulation kind of tau_for)"""
    g = gen(op, M, N, K, seed)
    x = ro.realistic(M, K, g)
    w = weights(N, K, g)
    b = bias_for(N, g)
    if op in ("int8_dyn", "int8_mm_i32"):
        xq, sx = ops.int8_quantize_rowwise(x)
        wq, sw = ops.int8_quantize_rowwise(w)
        sw = sw.reshape(-1)
        X, W = xq.double(), wq.double()
        if op == "int8_mm_i32":
            return lambda: ops.int8_mm_i32(xq, wq), [Seg(0, M, X, W, lambda a: a)], "s32"
        return (lambda: ops.int8_dyn_linear(xq, sx, wq, sw, b),
                [Seg(0, M, X, W, lambda a: ro.epi_i8(a, col(sx), row(sw), b64(b)))], "s32")
    if op in ("fp8", "fp8_static"):
        if op == "fp8":
            xq, sx = ops.fp8_quantize_rowwise(x)
        else:   # a calibrated scale: the activation amax over 448, times a factor that is not a power of two
            s = (x.float().abs().max() / 448.0 * 1.37).reshape(1)
            xq, sx = ops.fp8_quantize_static(x, s)
        wq, sw = ops.fp8_quantize_rowwise(w)
        sx, sw = sx.reshape(-1), sw.reshape(-1)
        if op == "fp8":
            run = lambda: ops.fp8_rowwise_linear(xq, sx, wq, sw, b)
        else:
            run = lambda: ops.fp8_static_linear(xq, sx.expand(M).contiguous(), wq, sw, b, None)
        sxm = sx.expand(M)
        return (run, [Seg(0, M, xq.double(), wq.double(), lambda a: ro.epi_f8(a, col(sxm), row(sw), b64(b)),
                          parts=lambda: e4m3_parts(xq, wq), alt=lambda: scaled_mm_rowwise(xq, sxm, wq, sw, b))], "e4m3")
    if op == "fp8_blockwise":
        from ao_b200.quantization import Float8Tensor, PerBlock

        xq, st = ops.fp8_quantize_1x128(x)
        st = st * WIDEN
        a_s = st[:, :M].t()                      # [M, K/128]
        wt = Float8Tensor.from_hp(w, granularity=PerBlock([128, 128]))
        wq, w_s = wt.qdata, wt.scale * WIDEN     # [N/128, K/128]
        X = xq.double() * a_s.double().repeat_interleave(128, 1)
        W = wq.double() * w_s.double().repeat_interleave(128, 0).repeat_interleave(128, 1)
        nb = torch.arange(N, device=DEV) // 128

        def combine(acc, part, kc):   # acc = fma(part * a_s[m][kc], w_s[n/128][kc], acc), fp32 (BlockwiseF8Fmt::promote)
            t = ro.r32(part.double() * a_s[:, kc].double()[:, None])
            v = t * w_s[nb, kc].double()[None, :] + (0.0 if acc is None else acc.double())
            return ro.r32(v).float()
        return (lambda: ops.fp8_blockwise_linear(xq, st, wq, w_s, b),
                [Seg(0, M, X, W, lambda a: ro.epi_bf16(a, b64(b)), parts=lambda: e4m3_parts(xq, wq), combine=combine)],
                "e4m3")
    if op == "fp8_sparse":
        from ao_b200.quantization import Float8Tensor, PerRow

        keep = w.float().abs().reshape(N, K // 4, 4).topk(2, -1).indices
        mask = torch.zeros(N, K // 4, 4, device=DEV, dtype=torch.bool).scatter_(-1, keep, True).reshape(N, K)
        xt = Float8Tensor.from_hp(x, granularity=PerRow())
        wt = Float8Tensor.from_hp(w * mask, granularity=PerRow())
        qd, meta = sparse_compress(wt.qdata)
        sx, sw = xt.scale.reshape(-1), wt.scale.reshape(-1)
        return (lambda: ops.fp8_sparse_linear(xt.qdata, sx, qd, meta, sw, b),
                [Seg(0, M, xt.qdata.double(), wt.qdata.double(), lambda a: ro.epi_f8_sparse(a, col(sx), row(sw), b64(b)),
                     parts=lambda: e4m3_chain(xt.qdata, wt.qdata))], "e4m3_chain")
    if op == "int8wo":
        wq, s = ops.int8_quantize_rowwise(w)   # the weight-only handler's per-row symmetric int8
        s = s.reshape(-1)
        return (lambda: ops.int8_weight_linear(x, wq, s, b),
                [Seg(0, M, x.double(), wq.double(), lambda a: ro.epi_bf16_wscale(a, row(s), b64(b)))], "f32")
    if op == "fp8wo":
        wq, s = ops.fp8_quantize_rowwise(w)
        s = s.reshape(-1)
        W = ro.r16(ro.r32(wq.double() * col(s)))   # bf16(fp32(e4m3 * scale)), the reference's dequantize
        return (lambda: ops.fp8_weight_linear(x, wq, s, b),
                [Seg(0, M, x.double(), W, lambda a: ro.epi_bf16(a, b64(b)))], "f32")
    if op in ("int4", "int4_hqq"):
        from ao_b200.quantization.quantize_.workflows.int4.int4_choose_qparams_algorithm import Int4ChooseQParamsAlgorithm
        from ao_b200.quantization.quantize_.workflows.int4.int4_tile_packed_to_4d_tensor import Int4TilePackedTo4dTensor

        gs = 128
        algo = Int4ChooseQParamsAlgorithm.HQQ if op == "int4_hqq" else Int4ChooseQParamsAlgorithm.TINYGEMM
        t = Int4TilePackedTo4dTensor.from_hp(w, [1, gs], int4_choose_qparams_algorithm=algo)
        u8 = ops.int4_unpack_tile4d(t.qdata)                       # [N, K/2], even k in the high nibble
        q = torch.stack([(u8 >> 4).long(), (u8 & 15).long()], -1).reshape(N, K)
        sz = t.scale_and_zero.double()                             # [K/g, N, 2]
        s = sz[..., 0].t().repeat_interleave(gs, 1)
        z = sz[..., 1].t().repeat_interleave(gs, 1)
        W = ro.r16((q.double() - 8) * s + z)                       # bf16(fma(q - 8, s, z)), one rounding
        return (lambda: ops.int4_tilepacked_linear(x, t.qdata, gs, t.scale_and_zero, b, N, 1),
                [Seg(0, M, x.double(), W, lambda a: ro.epi_float(a, bias=b64(b)))], "f32")
    if op == "nf4":
        from ao_b200.quantization import to_nf4

        t = to_nf4(w, 64, 256)
        codes = t.quantized_data.reshape(-1)
        c = torch.stack([(codes >> 4).long(), (codes & 15).long()], -1).reshape(N, K)
        qs = t.quantized_scalers.double().reshape(-1)
        f = t.quantization_factor.double().reshape(-1).repeat_interleave(256)[: qs.numel()]
        scal = ro.r16(ro.r32(ro.r16(ro.r32(qs / f)) + t.scaler_mean.double()))   # bf16(bf16(qs / f) + mean)
        W = ro.r16(t.nf4.double()[c] * scal.reshape(N, K // 64).repeat_interleave(64, 1))
        return (lambda: ops.nf4_linear(x, t.quantized_data, t.quantized_scalers, t.quantization_factor, t.scaler_mean,
                                       t.nf4, 64, 256, b),
                [Seg(0, M, x.double(), W, lambda a: ro.epi_bf16(a, b64(b)))], "f32")
    if op in ("mxfp8", "mxfp4"):
        quant = ops.mxfp8_quantize if op == "mxfp8" else ops.mxfp4_quantize
        xq, xs, xsb = unblocked(quant, x)
        wq, ws, wsb = unblocked(quant, w)
        if op == "mxfp8":
            X = xq.double() * e8m0(xs).repeat_interleave(32, 1)
            W = wq.double() * e8m0(ws).repeat_interleave(32, 1)
            run = lambda: ops.mxfp8_linear(xq, xsb, wq, wsb, b)
        else:
            X, W = fp4_values(xq, xs, 32, e8m0), fp4_values(wq, ws, 32, e8m0)
            run = lambda: ops.mxfp4_linear(xq, xsb, wq, wsb, b)
        return run, [Seg(0, M, X, W, lambda a: ro.epi_float(a, bias=b64(b)))], "f32"
    if op == "nvfp4":
        pa = (x.float().abs().max() / (448.0 * 6.0)).reshape(1)
        pb = (w.float().abs().max() / (448.0 * 6.0)).reshape(1)
        xq, xs, xsb = unblocked(lambda t, sw: ops.nvfp4_quantize(t, pa, sw), x)
        wq, ws, wsb = unblocked(lambda t, sw: ops.nvfp4_quantize(t, pb, sw), w)
        X, W = fp4_values(xq, xs, 16, e4m3_bytes), fp4_values(wq, ws, 16, e4m3_bytes)
        return (lambda: ops.nvfp4_linear(xq, xsb, pa, wq, wsb, pb, b),
                [Seg(0, M, X, W, lambda a: ro.epi_float(a, out_scale=float(pa), out_scale2=float(pb), bias=b64(b)))],
                "f32")
    if op in ("nvfp4w", "nvfp4w_xs"):
        pb = (w.float().abs().max() / (448.0 * 6.0)).reshape(1)
        wq, ws, wsb = unblocked(lambda t, sw: ops.nvfp4_quantize(t, pb, sw), w)
        W = fp4_values(wq, ws, 16, e4m3_bytes)
        if op == "nvfp4w_xs":
            xq, sx = ops.fp8_fakequant_rowwise(x)
            sx = sx.reshape(-1)
            return (lambda: ops.nvfp4_weight_linear(xq, sx, wq, wsb, pb, b),
                    [Seg(0, M, xq.double(), W, lambda a: ro.epi_float(a, row_scale=col(sx), out_scale=float(pb),
                                                                        bias=b64(b)))], "f32")
        return (lambda: ops.nvfp4_weight_linear(x, None, wq, wsb, pb, b),
                [Seg(0, M, x.double(), W, lambda a: ro.epi_float(a, out_scale=float(pb), bias=b64(b)))], "f32")
    raise ValueError(op)


# ------------------------------------------------------------------------------------------------ grouped builders
def ragged_offs(M, E, g):
    """E experts over M rows, one of them empty and one with a single row (cumulative ends, int32)."""
    cuts = torch.sort(torch.randint(2, M + 1, (E - 1,), device=DEV, generator=g)).values
    cuts[0] = 0                        # expert 0: empty
    cuts[1] = 1                        # expert 1: one row
    return torch.cat([cuts, torch.tensor([M], device=DEV)]).to(torch.int32)


def build_grouped(ops, op, M, E, N, K, seed=0):
    g = gen(op, M, E, N, K, seed)
    x = ro.realistic(M, K, g)
    w = weights(E * N, K, g)
    offs = ragged_offs(M, E, g)
    ends = offs.tolist()
    starts = [0] + ends[:-1]
    segs = []
    if op == "fp8_bmm":   # B batches of M / B tokens, weights stored [B, K, N]
        B, Mb = E, M // E
        xq, sx = ops.fp8_quantize_rowwise(x[: B * Mb])
        wq, sw = ops.fp8_quantize_rowwise(w)
        wq3, sw3 = wq.reshape(B, N, K), sw.reshape(B, N)
        w_kn = wq3.transpose(1, 2).contiguous()
        for e in range(B):
            r0, r1 = e * Mb, (e + 1) * Mb
            segs.append(Seg(r0, r1, xq[r0:r1].double(), wq3[e].double(),
                            lambda a, e=e, r0=r0, r1=r1: ro.epi_f8(a, col(sx[r0:r1]), row(sw3[e]), None),
                            parts=lambda e=e, r0=r0, r1=r1: e4m3_parts(xq[r0:r1], wq3[e]),
                            alt=lambda e=e, r0=r0, r1=r1: scaled_mm_rowwise(xq[r0:r1], sx[r0:r1], wq3[e], sw3[e], None)))
        return (lambda: ops.fp8_rowwise_bmm(xq.reshape(B, Mb, K), sx.reshape(-1), w_kn, sw3.reshape(-1)).reshape(B * Mb, N),
                segs, "e4m3")
    if op in ("fp8_grouped", "int8_dyn_grouped"):
        quant = ops.fp8_quantize_rowwise if op == "fp8_grouped" else ops.int8_quantize_rowwise
        xq, sx = quant(x)
        wq, sw = quant(w)
        sx, wq3, sw3 = sx.reshape(-1), wq.reshape(E, N, K), sw.reshape(E, N)
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue
            if op == "fp8_grouped":
                epi = lambda a, e=e, r0=r0, r1=r1: ro.epi_f8(a, col(sx[r0:r1]), row(sw3[e]), None)
                parts = lambda e=e, r0=r0, r1=r1: e4m3_parts(xq[r0:r1], wq3[e])
                alt = lambda e=e, r0=r0, r1=r1: scaled_mm_rowwise(xq[r0:r1], sx[r0:r1], wq3[e], sw3[e], None)
            else:
                epi = lambda a, e=e, r0=r0, r1=r1: ro.epi_i8(a, col(sx[r0:r1]), row(sw3[e]), None)
                parts = alt = None
            segs.append(Seg(r0, r1, xq[r0:r1].double(), wq3[e].double(), epi, parts=parts, alt=alt))
        run = ((lambda: ops.fp8_rowwise_grouped_mm(xq, sx, wq3, sw3, offs)) if op == "fp8_grouped"
               else (lambda: ops.int8_dyn_grouped_mm(xq, sx, wq3, sw3, offs)))
        return run, segs, ("e4m3" if op == "fp8_grouped" else "s32")
    if op in ("int8wo_grouped", "fp8wo_grouped"):
        quant = ops.int8_quantize_rowwise if op == "int8wo_grouped" else ops.fp8_quantize_rowwise
        wq, sw = quant(w)
        wq3, sw3 = wq.reshape(E, N, K), sw.reshape(E, N)
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue
            if op == "int8wo_grouped":
                W, epi = wq3[e].double(), (lambda a, e=e: ro.epi_bf16_wscale(a, row(sw3[e]), None))
            else:
                W, epi = ro.r16(ro.r32(wq3[e].double() * col(sw3[e]))), (lambda a: ro.epi_bf16(a, None))
            segs.append(Seg(r0, r1, x[r0:r1].double(), W, epi))
        run = ((lambda: ops.int8_weight_grouped_mm(x, wq3, sw3, offs)) if op == "int8wo_grouped"
               else (lambda: ops.fp8_weight_grouped_mm(x, wq3, sw3, offs)))
        return run, segs, "f32"
    if op == "fp8_blockwise_grouped":
        from ao_b200.quantization import Float8Tensor, PerBlock

        xq, st = ops.fp8_quantize_1x128(x)
        st = st * WIDEN
        a_s = st[:, :M].t()                                        # [M, K/128]
        wt = Float8Tensor.from_hp(w.reshape(E, N, K), granularity=PerBlock([128, 128]))
        wq3, ws3 = wt.qdata, wt.scale * WIDEN                      # [E, N, K], [E, N/128, K/128]
        assert ws3.shape == (E, N // 128, K // 128), ws3.shape
        nb = torch.arange(N, device=DEV) // 128
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue

            def combine(acc, part, kc, e=e, r0=r0, r1=r1):   # BlockwiseF8Fmt::promote with the expert's w_s block
                t = ro.r32(part.double() * a_s[r0:r1, kc].double()[:, None])
                v = t * ws3[e, nb, kc].double()[None, :] + (0.0 if acc is None else acc.double())
                return ro.r32(v).float()
            X = xq[r0:r1].double() * a_s[r0:r1].double().repeat_interleave(128, 1)
            W = wq3[e].double() * ws3[e].double().repeat_interleave(128, 0).repeat_interleave(128, 1)
            segs.append(Seg(r0, r1, X, W, lambda a: ro.epi_bf16(a, None),
                            parts=lambda e=e, r0=r0, r1=r1: e4m3_parts(xq[r0:r1], wq3[e]), combine=combine))
        return lambda: ops.fp8_blockwise_grouped_mm(xq, st, wq3, ws3, offs), segs, "e4m3"
    if op == "nvfp4_grouped":   # fake-quantized nvfp4 activations with per-token scales, per-expert weight scales
        xhat, xs = ops.nvfp4_fakequant_grouped(x, offs)
        xs = xs.reshape(-1)
        w3 = w.reshape(E, N, K)
        wp = torch.stack([w3[e].float().abs().max() / (448.0 * 6.0) for e in range(E)])
        q = [unblocked(lambda t, sw, e=e: ops.nvfp4_quantize(t, wp[e:e + 1], sw), w3[e]) for e in range(E)]
        wq3, wsb3 = torch.stack([t[0] for t in q]), torch.stack([t[2] for t in q])
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue
            W = fp4_values(q[e][0], q[e][1], 16, e4m3_bytes)
            segs.append(Seg(r0, r1, xhat[r0:r1].double(), W,
                            lambda a, e=e, r0=r0, r1=r1: ro.epi_float(a, row_scale=col(xs[r0:r1]), out_scale=wp[e].double())))
        return lambda: ops.nvfp4_grouped_mm(xhat, xs, wq3, wsb3, wp, offs), segs, "f32"
    if op in ("mxfp8_grouped", "mxfp4_grouped"):   # the dense MX recipe's fake-quantized activations, no scale, no bias
        fmt = op.split("_")[0]
        quant = getattr(ops, f"{fmt}_quantize")
        xhat = getattr(ops, f"{fmt}_fakequant")(x)
        w3 = w.reshape(E, N, K)
        q = [unblocked(quant, w3[e]) for e in range(E)]
        wq3, wsb3 = torch.stack([t[0] for t in q]), torch.stack([t[2] for t in q])
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue
            W = (q[e][0].double() * e8m0(q[e][1]).repeat_interleave(32, 1) if fmt == "mxfp8"
                 else fp4_values(q[e][0], q[e][1], 32, e8m0))
            segs.append(Seg(r0, r1, xhat[r0:r1].double(), W, lambda a: ro.epi_float(a)))
        return lambda: getattr(ops, f"{fmt}_grouped_mm")(xhat, wq3, wsb3, offs), segs, "f32"
    if op == "int4_grouped":
        from ao_b200.quantization.quantize_.workflows.int4.int4_tile_packed_to_4d_tensor import Int4TilePackedTo4dTensor

        gs = 128
        t = Int4TilePackedTo4dTensor.from_hp(w.reshape(E, N, K), [1, 1, gs])
        assert t.scale_and_zero.shape == (E, K // gs, N, 2), t.scale_and_zero.shape
        u8 = ops.int4_unpack_tile4d(t.qdata.reshape(E * N // 8, K // 128, 32, 4))   # [E N, K/2], even k high
        q = torch.stack([(u8 >> 4).long(), (u8 & 15).long()], -1).reshape(E, N, K)
        sz = t.scale_and_zero.double()
        for e in range(E):
            r0, r1 = starts[e], ends[e]
            if r1 == r0:
                continue
            s_, z_ = sz[e, ..., 0].t().repeat_interleave(gs, 1), sz[e, ..., 1].t().repeat_interleave(gs, 1)
            W = ro.r16((q[e].double() - 8) * s_ + z_)                # bf16(fma(q - 8, s, z)), one rounding
            segs.append(Seg(r0, r1, x[r0:r1].double(), W, lambda a: ro.epi_float(a)))
        return lambda: ops.int4_tilepacked_grouped_mm(x, t.qdata, gs, t.scale_and_zero, offs, N), segs, "f32"
    raise ValueError(op)



# ------------------------------------------------------------------------------------------------ the check
def check(y, segs, kind, K, contributors, what):
    """Envelope and census of y [M, N] over its segments; returns the report line.  The census model: e4m3, each
    segment's chunk partials from the tensor core (e4m3_parts) added in fp32 in k order; otherwise one truncating
    fp32 chain of k16 steps (realistic_operands.chain_f32); then the epilogue.  Where every segment has alt()
    (e4m3 with rowwise-expressible scales), the kernel must also stay within the census of torch._scaled_mm without
    fast accumulation, the cuBLAS path whose per-128-k promotion DESIGN §1 says the kernel matches."""
    tau = ro.tau_for(kind, K, contributors)
    ys, rs, ms, alts, worst, nbad = [], [], [], [], 0.0, 0
    for s in segs:
        yv = y[s.r0:s.r1].double()
        acc = s.X @ s.W.t()
        S = s.X.abs() @ s.W.abs().t()
        ratio, bad = ro.envelope(yv, s.epi, acc, S, tau)
        worst = max(worst, ratio)
        if bad.any():
            m, n = (int(v) for v in bad.nonzero()[0])
            nbad += int(bad.sum())
            first = f"first at ({s.r0 + m}, {n}): y {float(yv[m, n])!r} r {float(s.epi(acc)[m, n])!r}"
        r = s.epi(acc)
        if kind == "s32":
            model = r
        elif kind == "f32":   # no promotion: one accumulator chain per segment (ts_gemm.cuh)
            model = s.epi(ro.chain_f32(s.X, s.W))
        else:
            model = s.epi(ro.add_chunks_f32(s.parts(), s.combine))
        ys.append(yv.reshape(-1))
        rs.append(r.reshape(-1))
        ms.append(model.reshape(-1))
        if s.alt is not None:
            alts.append(s.alt().double().reshape(-1))
        del acc, S
    yv, r, model = torch.cat(ys), torch.cat(rs), torch.cat(ms)
    assert nbad == 0, f"{what}: {nbad} outputs outside the envelope (tau {tau:.3g}); {first}"
    if kind == "s32":
        assert torch.equal(yv, r), f"{what}: {int((yv != r).sum())} outputs differ from the exact recipe"
        rep = f"{what}: exact"
    else:
        ok, rep = ro.check_census(yv, r, model)
        rep = f"{what}: {rep} max|y-r|/env {worst:.3f}"
        assert ok, rep
        if alts and len(alts) == len(segs):
            ok, rep_alt = ro.check_census(yv, r, torch.cat(alts))
            rep += f" | vs _scaled_mm: {rep_alt}"
            assert ok, rep
    print(rep)
    return rep


def contributors_of(M, N, K, grid_n=None):
    """An upper bound on the stream-K partials summed into one output: every CTA holding a chunk of its tile."""
    units_per_tile = -(-K // 128)
    G = 132 if grid_n is None else grid_n
    tiles = -(-N // 128) * max(1, -(-M // 16))
    per_cta = max(1, (tiles * units_per_tile) // G)
    return -(-units_per_tile // per_cta) + 1


DENSE = ["int8_dyn", "int8_mm_i32", "fp8", "fp8_static", "fp8_blockwise", "fp8_sparse", "int8wo", "fp8wo", "int4",
         "int4_hqq", "nf4", "mxfp8", "mxfp4", "nvfp4", "nvfp4w", "nvfp4w_xs"]


def scaled_mm_rowwise(xq, sx, wq, sw, b):
    return torch._scaled_mm(xq, wq.t(), scale_a=sx.reshape(-1, 1).contiguous(), scale_b=sw.reshape(1, -1).contiguous(), bias=b,
                            out_dtype=torch.bfloat16, use_fast_accum=False)


@pytest.mark.parametrize("op", DENSE)
def test_dense_rounding_at_llama_shapes(ops, op):
    for M, proj in SHAPES:
        N, K = PROJ[proj]
        run, segs, kind = build(ops, op, M, N, K)
        y = run()
        torch.cuda.synchronize()
        check(y, segs, kind, K, contributors_of(M, N, K), f"{op} M={M} {proj}")
        del segs


@pytest.mark.parametrize("op", DENSE)
def test_dense_rounding_under_forced_splits(ops, grid, op):
    M, proj = FORCED
    N, K = PROJ[proj]
    run, segs, kind = build(ops, op, M, N, K, seed=1)
    for n in GRIDS:
        grid(n)
        y = run()
        torch.cuda.synchronize()
        check(y, segs, kind, K, contributors_of(M, N, K, n), f"{op} M={M} {proj} grid={n}")


GROUPED = ["fp8_grouped", "int8_dyn_grouped", "int8wo_grouped", "fp8wo_grouped", "fp8_bmm", "fp8_blockwise_grouped",
           "nvfp4_grouped", "mxfp8_grouped", "mxfp4_grouped", "int4_grouped"]


@pytest.mark.parametrize("op", GROUPED)
@pytest.mark.parametrize("n", [None, 37, 132])
def test_grouped_rounding_at_an_expert_shape(ops, grid, op, n):
    """8 experts of a 1024 x 2048 layer (K = 2048: 16 chunks) over 200 ragged tokens (one expert empty, one with a
    single token; bmm: 8 batches of 25)."""
    M, E, N, K = 200, 8, 1024, 2048
    run, segs, kind = build_grouped(ops, op, M, E, N, K)
    if n is not None:
        grid(n)
    y = run()
    torch.cuda.synchronize()
    check(y, segs, kind, K, contributors_of(M, E * N, K, n), f"{op} M={M} E={E} grid={n or 'default'}")
