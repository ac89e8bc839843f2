"""Exactly representable operands for the quantized linears, and their fp64 references (GPU tests only).

Each builder draws codes and scales straight from small sets instead of quantizing random floats.  With those sets
every product X[m,k] * W[n,k] is an integer multiple of one quantum u and every sum stays below 2^24 u, so fp32
accumulates exactly in any order and under any stream-K split; the epilogue's scale products are exact in fp32 as
well.  The kernel's bf16 output must then equal the fp64 reference rounded to bf16, bit for bit, in every element.
Each builder asserts that premise before anything is compared.  Scales have mantissa bits set (int4 s, the e4m3
block scales of nvfp4, the fp8 row scales), so the scale arithmetic is checked too, not only powers of two.

The weight-only int8 and fp8 linears and mxfp4 round where their recipes round, so their references are not the fp64
sum rounded once: the sum is exact in fp32 and the reference applies the recipe's own roundings to it (recipe()).
"""
import torch

DEV = "cuda"
E2M1 = [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, -0.0, -0.5, -1.0, -1.5, -2.0, -3.0, -4.0, -6.0]
ODD = [5, 6, 7, 9, 11, 13]       # scale mantissas: 3 significant bits, never a power of two alone
POISON_BF16 = 0x7FC0             # a NaN: outputs are scrubbed with it after use, so an unwritten element cannot
POISON_I32 = -2**31              # inherit a correct value from an earlier launch through the caching allocator


def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randint(lo, hi, shape, g):
    return torch.randint(lo, hi + 1, shape, device=DEV, generator=g)


def pick(values, shape, g):
    v = torch.tensor(values, dtype=torch.float64, device=DEV)
    return v[torch.randint(0, len(values), shape, device=DEV, generator=g)]


def lowbit(t):
    """The largest power of two that divides every entry of the fp64 tensor t."""
    nz = t[t != 0].abs()
    if nz.numel() == 0:
        return 1.0
    m, e = torch.frexp(nz)
    mi = (m * 2.0**53).to(torch.int64)
    # the lowest set bit of each 53-bit significand, 2^(j - 1) with j its frexp exponent: only integer exponents are
    # formed on the device (torch.pow on CUDA is not exact), the one power of two on the host
    j = torch.frexp((mi & -mi).double())[1]
    return 2.0 ** int((j - 1 + e - 53).min())


def pow2(e):
    """2^e for an integer tensor, exactly (a table: torch.pow on CUDA rounds)."""
    table = torch.tensor([2.0**i for i in range(-160, 161)], dtype=torch.float64, device=e.device)
    return table[e.long() + 160]


def fp32_exact(t, what):
    assert torch.equal(t.float().double(), t), f"premise: {what} is not exact in fp32"


def premise(X, W, bias_acc=None, chunk=False, segment=False):
    """Asserts max(|X| @ |W|^T) + |bias| < 2^24 u (u = the quantum of every product); returns u.  chunk: the e4m3
    wgmma chain of one 128-k chunk adds in the tensor core's reduced-precision accumulator (DESIGN.md §1), so each
    chunk's sum is also kept under 2^13 u, an assumed width under which that adder is exact.  Above ANALYTIC_ABOVE
    elements of M x N x KT the chunk sums are bounded by 128 max|X| max|W| instead of materialised.  segment: the
    kernel never promotes (2:4-sparse e4m3), so a whole segment's K sum stays in that accumulator: the whole sum is
    kept under 2^13 u."""
    u = lowbit(X) * lowbit(W)
    extra = float(bias_acc.abs().max()) if bias_acc is not None else 0.0
    top = float((X.abs() @ W.abs().t()).max()) + extra
    assert top < 2.0**24 * u, f"premise: sums reach {top / u:.0f} u >= 2^24 u"
    assert not segment or top < 2.0**13 * u, f"premise: a segment's sum reaches {top / u:.0f} u >= 2^13 u"
    if chunk and X.shape[0] * W.shape[0] * -(-X.shape[1] // 128) > ANALYTIC_ABOVE:
        top_c = 128 * float(X.abs().max()) * float(W.abs().max())
        assert top_c < 2.0**13 * u, f"premise: a 128-k chunk may reach {top_c / u:.0f} u >= 2^13 u"
    elif chunk:
        K = X.shape[1]
        KT = -(-K // 128)
        Xp = torch.nn.functional.pad(X.abs(), (0, KT * 128 - K)).reshape(X.shape[0], KT, 128)
        Wp = torch.nn.functional.pad(W.abs(), (0, KT * 128 - K)).reshape(W.shape[0], KT, 128)
        top_c = float(torch.einsum("mkc,nkc->mnk", Xp, Wp).max())
        assert top_c < 2.0**13 * u, f"premise: a 128-k chunk reaches {top_c / u:.0f} u >= 2^13 u"
    return u


def recipe(op, acc, scale=None, bias=None):
    """The bf16 output of a linear whose epilogue rounds as its reference does, from the exact sums acc (fp64 [M, n]):
    int8wo bf16(bf16(bf16(acc) * bf16(scale)) + bias) (torch.mm in bf16, then the bf16 scale and bias);
    fp8wo bf16(bf16(acc) + bias) (the weights are already bf16(e4m3 * scale)); mxfp4 bf16(fp32(acc) + bias)."""
    fp32_exact(acc, f"{op}: the sums")
    a = acc.float()
    if op == "int8wo":
        y = a.to(torch.bfloat16) * scale.to(torch.bfloat16)
    elif op == "fp8wo":
        y = a.to(torch.bfloat16)
    elif op == "mxfp4":
        return (a + bias.float()).to(torch.bfloat16) if bias is not None else a.to(torch.bfloat16)
    else:
        raise ValueError(op)
    return y if bias is None else y + bias


def int8_epilogue(acc, x_scale, w_scale, bias=None):
    """EPI_I8 on exact int32 sums acc (fp64 [M, n]): the reference's order, bf16 between the two scales,
    bf16(bf16(acc * x_scale[m]) * w_scale[n] + bias[n]) (x_scale f32 [M, 1], w_scale f32 [n], bias bf16 [n] or None);
    fp64 of the fp32 value before the last rounding."""
    assert float(acc.abs().max()) < 2.0**24, "premise: int32 sums must convert to fp32 exactly"
    t = (acc.float() * x_scale).to(torch.bfloat16).float()
    fp32_exact(t.double() * w_scale.double(), "int8: bf16(acc * x_scale) * w_scale")   # fma == mul then add
    return (t * w_scale if bias is None else t * w_scale + bias.float()).double()


def mxfp4_value(codes, scale_bytes):
    """fp64 e2m1 codes [R, K] times e8m0 bytes [R, K/32] (every byte here is a normal power of two)."""
    return e2m1_value(codes) * pow2(scale_bytes.long() - 127).repeat_interleave(32, 1)[:, : codes.shape[1]]


def bias_for(n, q, g):
    """bf16 bias, an integer multiple of the output quantum q (exact in bf16: 8 significant bits)."""
    return randint(-127, 127, (n,), g).double() * q * 16


def to_blocked(plain):
    """[R, C] scale bytes -> the 128 x 4 -> 32 x 16 blocked layout (ao_b200/prototype/mx_formats/utils.py)."""
    R, C = plain.shape
    rb, cb = -(-R // 128), -(-C // 4)
    p = torch.zeros(rb * 128, cb * 4, dtype=torch.uint8, device=plain.device)
    p[:R, :C] = plain
    blocks = p.view(rb, 128, cb, 4).permute(0, 2, 1, 3).reshape(-1, 4, 32, 4).transpose(1, 2).reshape(rb * 32, cb * 16)
    return blocks.contiguous()


def e4m3_bytes_value(b):
    return b.to(torch.uint8).view(torch.float8_e4m3fn).double()


def pack_e2m1(codes):
    """[R, K] nibbles -> [R, K/2] bytes, even k in the low nibble."""
    return (codes[:, 0::2] | (codes[:, 1::2] << 4)).to(torch.uint8).contiguous()


def e2m1_value(codes):
    return torch.tensor(E2M1, dtype=torch.float64, device=DEV)[codes.long()]


class Case:
    """One linear with exact operands at token count M_max.  run(M) launches it on the first M tokens; ref(M) is the
    expected output (bf16, or int32 for int8_mm_i32).  fmt / n_plan give the work split of tests/streamk_model.py."""

    def __init__(self, op, fmt, M, N, K, n_plan, y64, launch, out_int=False, ref=None):
        self.op, self.fmt, self.M, self.N, self.K, self.n_plan = op, fmt, M, N, K, n_plan
        self.launch = launch
        self.out_int = out_int
        if ref is not None:   # already rounded (served(): built block by block)
            self.ref_full = ref
        elif out_int:
            self.ref_full = y64.to(torch.int32)
        else:
            fp32_exact(y64, f"{op}: the fp64 reference")   # so the cast below rounds once
            self.ref_full = y64.float().to(torch.bfloat16)

    def run(self, M=None):
        return self.launch(self.M if M is None else M)

    def ref(self, M=None):
        return self.ref_full[: (self.M if M is None else M)]

    def bits(self, y):
        return y if self.out_int else y.view(torch.int16)

    def scrub(self, y):
        self.bits(y).fill_(POISON_I32 if self.out_int else POISON_BF16)


def int4_weights(n, K, group_size, g):
    """n exact int4 weight rows: codes 0..15, s = ODD 2^-9, z = -24..24 2^-9.  Returns (W fp64 [n, K], qdata
    [n/8, K/128, 32, 4], scale_and_zero bf16 [n, K/g, 2]); asserts that bf16(fma(q - 8, s, z)) is W itself."""
    o = ops()
    q = randint(0, 15, (n, K), g)
    s = pick(ODD, (n, K // group_size), g) * 2.0**-9
    z = randint(-24, 24, (n, K // group_size), g).double() * 2.0**-9
    W = (q.double() - 8) * s.repeat_interleave(group_size, 1) + z.repeat_interleave(group_size, 1)
    qdata = o.int4_pack_tile4d(((q[:, 0::2] << 4) | q[:, 1::2]).to(torch.uint8).contiguous(), 8)
    sz = torch.stack([s, z], -1).to(torch.bfloat16)
    assert torch.equal(o.int4_dequant_tile4d(qdata, sz.transpose(0, 1).contiguous(), group_size).double(), W), \
        "premise: int4 weights not exact in bf16"
    return W, qdata, sz


def transposed_scales(s):
    """1x128 token scales [M, K/128] -> the kernel's [K/128, round_up(M, 4)] layout (ao_fp8_quantize_1x128), pads 0."""
    M, KB = s.shape
    out = torch.zeros(KB, (M + 3) // 4 * 4, dtype=torch.float32, device=s.device)
    out[:, :M] = s.t()
    return out


def blockwise_values(codes, scales, rows):
    """fp64 codes [R, K] times their block scales [R / rows, K/128] (rows = 1: 1x128 token scales, 128: 128x128
    weight blocks).  Every scale is a power of two, so the reference loop's sum over chunks of dot(x_kb, w_kb) a_s w_s
    is X @ W^T of these values, exactly."""
    return codes * scales.double().repeat_interleave(rows, 0).repeat_interleave(128, 1)


def blockwise_epilogue(acc, bias):
    """EPI_BF16 on exact sums acc (fp64 [M, n]): bf16(acc), then the bf16 add of the bias."""
    fp32_exact(acc, "fp8_blockwise: the sums")
    y = acc.float().to(torch.bfloat16)
    return y if bias is None else y + bias


def sparse_codes(n, K, r, g):
    """n rows of 2:4-pruned nonzero integer codes -r..r (fp64 [n, K]): two random positions of each 4-k group kept,
    except that one group in sixteen is left empty and one in sixteen, for each position p, holds a single code at p."""
    keep = torch.rand(n, K // 4, 4, device=DEV, generator=g).argsort(-1)[..., :2]
    mask = torch.zeros(n, K // 4, 4, dtype=torch.bool, device=DEV).scatter_(-1, keep, True)
    kind = randint(0, 15, (n, K // 4), g)
    mask[kind == 0] = False
    for p in range(4):
        mask[kind == 1 + p] = torch.arange(4, device=DEV) == p
    codes = randint(1, r, (n, K), g) * (randint(0, 1, (n, K), g) * 2 - 1)
    return codes.double() * mask.reshape(n, K)


def sparse_activations(M, K, r, nnz, g):
    """codes -r..r [M, K] (fp64) with at most nnz nonzeros per row (None: no cap) at random positions, so that every
    position of every 4-k group still meets nonzero activations"""
    X = randint(-r, r, (M, K), g).double()
    if nnz is not None and nnz < K:
        X.scatter_(1, torch.rand(M, K, device=DEV, generator=g).argsort(-1)[:, nnz:], 0.0)
    return X


def sparse_scales(n, g):
    """per-row scales 2^[-3, 1] ODD / 8: mantissa bits, so the epilogue's rounding order shows"""
    return (pow2(randint(-3, 1, (n,), g)) * pick(ODD, (n,), g) / 8).float()


def sparse_compress(wq):
    """The package's 2:4 compressor on the e4m3 codes wq [N, K]; asserts that decompressing gives every code back."""
    from ao_b200.quantization.quantize_.workflows.float8.float8_sparse_2x4_2d_data_2d_metadata_tensor import (
        compress_2x4_e4m3, decompress_2x4_e4m3)

    qd, meta = compress_2x4_e4m3(wq)
    assert torch.equal(decompress_2x4_e4m3(qd, meta).float(), wq.float()), "premise: the compressor keeps every code"
    return qd, meta


def sparse_epilogue(acc, x_s, w_s, bias):
    """EPI_F8_SPARSE on exact sums acc (fp64 [M, n]): t = fp32(acc * w_s[n]), then fp32(t * x_s[m] + bias[n]) rounded
    once (an FFMA); fp64 of that fp32 value."""
    fp32_exact(acc, "fp8_sparse: the sums")
    t = (acc.float() * w_s[None, :]).double() * x_s[:, None].double()   # exact in fp64
    if bias is not None:
        t = t + bias.double()[None, :]
    return t.float().double()


def build(op, M, N, K, seed=0, n_out=None, w_bytes=None, group_size=64):
    """op: int4 | int8_dyn | int8_mm_i32 | fp8 | mxfp8 | nvfp4 | nvfp4w | nvfp4w_xs | nvfp4w_rowpts | int8wo | fp8wo |
    mxfp4 | fp8_blockwise | fp8_sparse.
    n_out: int4 output features (<= N).  w_bytes: nvfp4 weight scale bytes [N, K/16] (default: a window of normal
    bytes with mantissa bits set).  group_size: int4 (32, 64, 128 or 256).  The value windows are fixed and the
    premise is checked on the drawn values: for the test shapes (K <= 16384, M x N small); served() picks the windows
    from K instead (fp8_blockwise and fp8_sparse take that window here too)."""
    o = ops()
    g = gen(seed * 7919 + M * 31 + N * 7 + K)
    if op == "int4":
        grp = group_size
        n_out = n_out or N
        W, qdata, sz = int4_weights(N, K, grp, g)
        sz = sz.transpose(0, 1).contiguous()
        X = randint(-8, 8, (M, K), g).double() * 2.0**-3
        x = X.to(torch.bfloat16)
        W = W[:n_out]
        u = lowbit(X) * lowbit(W)
        bias = bias_for(n_out, u, g)
        premise(X, W, bias)
        b = bias.to(torch.bfloat16)
        return Case(op, "int4", M, N, K, n_out, X @ W.t() + bias,
                    lambda m: o.int4_tilepacked_linear(x[:m], qdata, grp, sz, b, n_out, 1))
    if op in ("int8_dyn", "int8_mm_i32"):
        xq = randint(-128, 127, (M, K), g).to(torch.int8)
        wq = randint(-128, 127, (N, K), g).to(torch.int8)
        acc = xq.double() @ wq.double().t()
        assert float(acc.abs().max()) < 2.0**24, "premise: int32 sums must convert to fp32 exactly"
        if op == "int8_mm_i32":
            return Case(op, "int8", M, N, K, N, acc, lambda m: o.int8_mm_i32(xq[:m], wq), out_int=True)
        sx = (pick(ODD, (M, 1), g) * 2.0**-14).float()
        sw = (pick(ODD, (N,), g) * 2.0**-10).float()
        b = (randint(-127, 127, (N,), g).double() * 2.0**-8).to(torch.bfloat16)
        # the reference's rounding order (test_lowp_gpu.py::test_int8_linear_exact): bf16 between the two scales
        t = (acc.float() * sx).to(torch.bfloat16).float()
        fp32_exact(t.double() * sw.double(), "int8: bf16(acc * x_scale) * w_scale")   # fma == mul then add
        y = t * sw + b.float()
        return Case(op, "int8", M, N, K, N, y.double(), lambda m: o.int8_dyn_linear(xq[:m], sx[:m], wq, sw, b))
    if op == "fp8":
        X = randint(-7, 7, (M, K), g).double() * 2.0**-2
        W = randint(-7, 7, (N, K), g).double() * 2.0**-3
        xq, wq = X.to(torch.float8_e4m3fn), W.to(torch.float8_e4m3fn)
        assert torch.equal(xq.double(), X) and torch.equal(wq.double(), W)
        premise(X, W, chunk=True)
        rs = pick(ODD, (M,), g) * 2.0**-8
        sw = pick(ODD, (N,), g) * 2.0**-9
        sc = rs[:, None] * sw[None, :]
        fp32_exact(sc, "fp8: x_scale * w_scale")
        prod = (X @ W.t()) * sc
        fp32_exact(prod, "fp8: acc * scales")
        bias = bias_for(N, lowbit(prod), g)
        b = bias.to(torch.bfloat16)
        rsf, swf = rs.float(), sw.float()
        return Case(op, "fp8", M, N, K, N, prod + bias, lambda m: o.fp8_rowwise_linear(xq[:m], rsf[:m], wq, swf, b))
    if op == "mxfp8":
        Xc = randint(-7, 7, (M, K), g).double() * 2.0**-2
        Wc = randint(-7, 7, (N, K), g).double() * 2.0**-3
        # e8m0 bytes >= 3: below that small e4m3 codes times the scale round in bf16 (lowp_linear.cu)
        xb = randint(125, 128, (M, K // 32), g)
        wb = randint(124, 127, (N, K // 32), g)
        X = Xc * pow2(xb - 127).repeat_interleave(32, 1)
        W = Wc * pow2(wb - 127).repeat_interleave(32, 1)
        xq, wq = Xc.to(torch.float8_e4m3fn), Wc.to(torch.float8_e4m3fn)
        assert torch.equal(xq.double(), Xc) and torch.equal(wq.double(), Wc)
        u = lowbit(X) * lowbit(W)
        bias = bias_for(N, u, g)
        premise(X, W, bias)
        b = bias.to(torch.bfloat16)
        xb8, wsb = xb.to(torch.uint8), to_blocked(wb.to(torch.uint8))
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = to_blocked(xb8[:m])
            return o.mxfp8_linear(xq[:m], cache[m], wq, wsb, b)
        c = Case(op, "mxfp8", M, N, K, N, X @ W.t() + bias, run)
        c.raw = dict(xq=xq, x_bytes=xb8, wq=wq, w_blocked=wsb, bias=b)
        return c
    if op in ("nvfp4", "nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts"):
        wc = randint(0, 15, (N, K), g)
        if w_bytes is None:
            w_bytes = randint(0x30, 0x37, (N, K // 16), g)   # one binade, every mantissa: sums stay < 2^24 u at K = 16384
        W = e2m1_value(wc) * e4m3_bytes_value(w_bytes).repeat_interleave(16, 1)
        wq, wsb = pack_e2m1(wc), to_blocked(w_bytes.to(torch.uint8))
        if op == "nvfp4":
            xc = pick([0, 1, 2, 8, 9, 10], (M, K), g).long()   # |e2m1| <= 1, for the same bound
            xbytes = randint(0x38, 0x3F, (M, K // 16), g).to(torch.uint8)
            X = e2m1_value(xc) * e4m3_bytes_value(xbytes).repeat_interleave(16, 1)
            xq = pack_e2m1(xc)
            premise(X, W)
            a_pts = torch.tensor([0.75], device=DEV)
            b_pts = torch.tensor([1.25], device=DEV)
            prod = (X @ W.t()) * (0.75 * 1.25)
            fp32_exact(prod, "nvfp4: acc * a_pts * b_pts")
            bias = bias_for(N, lowbit(prod), g)
            b = bias.to(torch.bfloat16)
            cache = {}

            def run(m):
                if m not in cache:
                    cache[m] = to_blocked(xbytes[:m])
                return o.nvfp4_linear(xq[:m], cache[m], a_pts, wq, wsb, b_pts, b)
            c = Case(op, "nvfp4", M, N, K, N, prod + bias, run)
            c.raw = dict(xq=xq, x_bytes=xbytes, wq=wq, w_blocked=wsb, bias=b, a_pts=a_pts, b_pts=b_pts)
            return c
        X = randint(-3, 3, (M, K), g).double() * 2.0**-1   # small: acc * x_scale * b_pts stays exact in fp32
        x = X.to(torch.bfloat16)
        premise(X, W)
        acc = X @ W.t()
        rs = pick(ODD, (M,), g) * 2.0**-6 if op != "nvfp4w" else None
        if rs is not None:
            acc = acc * rs[:, None]
            fp32_exact(acc, "nvfp4w: acc * x_scale")
        bp = pick(ODD, (N,), g) * 2.0**-4 if op == "nvfp4w_rowpts" else torch.tensor([1.25], dtype=torch.float64, device=DEV)
        prod = acc * bp.reshape(1, -1)
        fp32_exact(prod, "nvfp4w: acc * b_pts")
        bias = bias_for(N, lowbit(prod), g)
        b = bias.to(torch.bfloat16)
        rsf = rs.float() if rs is not None else None
        bpf = bp.float()
        return Case(op, "nvfp4", M, N, K, N, prod + bias,
                    lambda m: o.nvfp4_weight_linear(x[:m], rsf[:m] if rsf is not None else None, wq, wsb, bpf, b))
    if op == "int8wo":
        # any int8 weight; scales with 12 significant bits over 13 binades, so bf16(scale) rounds
        X = randint(-8, 8, (M, K), g).double() * 2.0**-3
        wq = randint(-128, 127, (N, K), g).to(torch.int8)
        premise(X, wq.double())
        s = (randint(2048, 4095, (N,), g).double() * 2.0**-20 * pow2(randint(-6, 6, (N,), g))).float()
        assert not torch.equal(s.to(torch.bfloat16).float(), s), "premise: bf16(scale) rounds"
        b = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16)
        x = X.to(torch.bfloat16)
        return Case(op, "int8wo", M, N, K, N, None, lambda m: o.int8_weight_linear(x[:m], wq, s, b),
                    ref=recipe(op, X @ wq.double().t(), s, b))
    if op == "fp8wo":
        # codes c/8, row scales odd * 2^p over nine binades: bf16(e4m3 * s) = c * s exactly, and each output
        # feature's products are multiples of its own quantum 2^(p-6)
        X = randint(-8, 8, (M, K), g).double() * 2.0**-3
        c = randint(-7, 7, (N, K), g).double() * 2.0**-3
        p = randint(-12, -4, (N,), g)
        s = (pick([3, 5, 7], (N,), g) * pow2(p)).float()
        wq = c.to(torch.float8_e4m3fn)
        W = (wq.float() * s[:, None]).to(torch.bfloat16).double()   # the reference's dequantize
        assert torch.equal(W, c * s.double()[:, None]), "premise: e4m3 * scale exact in bf16"
        assert bool(((X.abs() @ W.abs().t()) < 2.0**24 * 2.0**-6 * pow2(p)[None, :]).all()), "premise: sums < 2^24 quanta"
        b = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16)
        x = X.to(torch.bfloat16)
        return Case(op, "fp8wo", M, N, K, N, None, lambda m: o.fp8_weight_linear(x[:m], wq, s, b),
                    ref=recipe(op, X @ W.t(), bias=b))
    if op == "mxfp4":
        # every e2m1 code; e8m0 bytes from 80..171 per row (x) or feature (w), +1 in some blocks: each (m, n) sums
        # multiples of its own quantum 2^-2 2^(x byte + w byte - 254) of the lowest bytes
        nb = -(-K // 32)
        xc, wc = randint(0, 15, (M, K), g), randint(0, 15, (N, K), g)
        xs = randint(80, 170, (M, 1), g) + randint(0, 1, (M, nb), g)
        ws = randint(80, 170, (N, 1), g) + randint(0, 1, (N, nb), g)
        X, W = mxfp4_value(xc, xs), mxfp4_value(wc, ws)
        u = 0.25 * pow2(xs.min(1).values[:, None] + ws.min(1).values[None, :] - 254)
        assert bool(((X.abs() @ W.abs().t()) < 2.0**24 * u).all()), "premise: sums < 2^24 quanta"
        b = (torch.randn(N, device=DEV, generator=g) * 2.0**20).to(torch.bfloat16)
        xq, wq = pack_e2m1(xc), pack_e2m1(wc)
        xs8, wsb = xs.to(torch.uint8), to_blocked(ws.to(torch.uint8))
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = to_blocked(xs8[:m])
            return o.mxfp4_linear(xq[:m], cache[m], wq, wsb, b)
        return Case(op, "mxfp4", M, N, K, N, None, run, ref=recipe(op, X @ W.t(), bias=b))
    if op == "fp8_blockwise":
        # integer codes, power-of-two 1x128 / 128x128 scales: each chunk's code sum under 2^13, the whole scaled sum
        # under 2^24 of the smallest quantum; the epilogue rounds as the reference does (blockwise_epilogue)
        win = window(op, K)
        Xc = randint(-win["xr"], win["xr"], (M, K), g).double()
        Wc = randint(-win["wr"], win["wr"], (N, K), g).double()
        a_s = pow2(randint(-2, -2 + win["da"], (M, K // 128), g)).float()
        w_s = pow2(randint(-1, -1 + win["dw"], (N // 128, K // 128), g)).float()
        X, W = blockwise_values(Xc, a_s, 1), blockwise_values(Wc, w_s, 128)
        premise(Xc, Wc, chunk=True)
        premise(X, W)
        b = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16)
        xq, wq = Xc.to(torch.float8_e4m3fn), Wc.to(torch.float8_e4m3fn)
        cache = {}

        def run(m):
            if m not in cache:   # the layout depends on round_up(m, 4): one tensor per token count
                cache[m] = transposed_scales(a_s[:m])
            return o.fp8_blockwise_linear(xq[:m], cache[m], wq, w_s, b)
        return Case(op, "fp8_blockwise", M, N, K, N, None, run, ref=blockwise_epilogue(X @ W.t(), b))
    if op == "fp8_sparse":
        # no promotion: the whole K sum stays under 2^13 (the activation rows' nonzeros capped where K needs it)
        win = window(op, K)
        X = sparse_activations(M, K, win["xr"], win["nnz"], g)
        W = sparse_codes(N, K, win["wr"], g)
        premise(X, W, segment=True)
        x_s, w_s = sparse_scales(M, g), sparse_scales(N, g)
        b = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16)
        xq = X.to(torch.float8_e4m3fn)
        qd, meta = sparse_compress(W.to(torch.float8_e4m3fn))
        ref = sparse_epilogue(X @ W.t(), x_s, w_s, b).float().to(torch.bfloat16)
        return Case(op, "fp8_sparse", M, N, K, N, None,
                    lambda m: o.fp8_sparse_linear(xq[:m], x_s[:m], qd, meta, w_s, b), ref=ref)
    raise ValueError(op)


def first_mismatch(case, y, M=None):
    bad = (case.bits(y) != case.bits(case.ref(M))).nonzero()
    if bad.numel() == 0:
        return None
    m, n = (int(v) for v in bad[0])
    return m, n, float(y[m, n]), float(case.ref(M)[m, n]), int(bad.shape[0])


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count



# ------------------------------------------------------------------------------------------------ served shapes
# At the shapes the library serves (K up to 28672, thousands of tokens, tens of thousands of features) the fixed
# windows of build() are no longer exact by construction, and the checks that need M x N x KT or a whole fp64 weight
# in memory do not fit.  served() draws from windows picked from K so that the analytic bound holds, checks the
# premise block by block, and builds the fp64 reference W_BLOCK output features at a time.
ANALYTIC_ABOVE = 1 << 26   # elements of M x N x KT above which the 128-k chunk sums are bounded, not materialised
W_BLOCK = 4096             # output features per block of the fp64 reference
BIAS_UNITS = 127 * 16      # bias_for(): |bias| <= 2032 output quanta
I4_W = (2.0**-2, 2.0**-9)  # int4 W = (q - 8) s + z, s = ODD 2^-9, z = -24..24 2^-9: |W| <= 128 2^-9


def span(values):
    """(max |v|, the largest power of two that divides every v) of a set of exactly representable numbers."""
    import math

    low = None
    for v in values:
        if v == 0:
            continue
        m, e = math.frexp(abs(v))
        mi = int(m * 2**53)
        b = (mi & -mi) * 2.0 ** (e - 53)
        low = b if low is None else min(low, b)
    return max(abs(v) for v in values), low or 1.0


def units(factors):
    """max |product| / its quantum for a product of independent factors, each (max, quantum)."""
    r = 1.0
    for mx, low in factors:
        r *= mx / low
    return r


def _codes(r, scale=1.0):
    return [c * scale for c in range(-r, r + 1)]


def _e4m3(byte):
    s, e, m = byte >> 7, (byte >> 3) & 15, byte & 7
    v = (m / 8.0) * 2.0**-6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7)
    return -v if s else v


E2M1_UPTO1 = [0, 1, 2, 8, 9, 10]   # codes of 0, +-0.5, +-1


def served_candidates(op):
    """The value windows of op in the order served() tries them: widest first.  Each is a dict of the value sets
    (plain Python lists); factors() turns one into the (max, quantum) of X, W and the epilogue."""
    if op == "int4":
        return [dict(xr=r) for r in (8, 4, 2, 1)]
    if op in ("int8_dyn", "int8_mm_i32"):
        return [dict(r=r) for r in (127, 96, 63, 45, 34, 24, 16, 8)]
    if op == "fp8":
        return [dict(xr=a, wr=b, odd=[3, 5, 7]) for a, b in ((7, 7), (6, 6), (5, 4), (3, 3), (2, 2), (1, 1))]
    if op == "mxfp8":
        return [dict(dx=dx, dw=dw) for dx, dw in ((3, 3), (3, 2), (2, 2), (2, 1), (1, 1), (1, 0), (0, 0))]
    if op == "nvfp4":
        x4, x2 = list(range(0x38, 0x3C)), [0x38, 0x3C]
        w4, w2 = list(range(0x30, 0x34)), [0x30, 0x34]
        return [dict(xb=x4, wb=w4, pts=(0.75, 1.0)), dict(xb=x4, wb=w2, pts=(0.75, 0.5)),
                dict(xb=x2, wb=w2, pts=(0.75, 0.5)), dict(xb=x2, wb=w2, pts=(0.5, 2.0))]
    if op in ("nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts"):
        return [dict(xr=3, wb=list(range(0x30, 0x34)), odd=[3, 5, 7], bp=1.25),
                dict(xr=1, wb=[0x30, 0x34], odd=[3, 5, 7], bp=1.25),
                dict(xr=1, wb=[0x30, 0x34], odd=[3], bp=0.75)]
    if op == "int8wo":
        return [dict(xr=r) for r in (8, 4, 2, 1)]
    if op == "fp8wo":
        return [dict(xr=a, wr=b) for a, b in ((8, 7), (4, 7), (2, 3), (1, 1))]
    if op == "mxfp4":
        return [dict(xc=list(range(16)), d=1), dict(xc=list(range(16)), d=0), dict(xc=E2M1_UPTO1, d=0)]
    if op == "fp8_blockwise":   # token scales 2^[-2, -2 + da], weight block scales 2^[-1, -1 + dw]
        return [dict(xr=r, wr=r, da=3, dw=2) for r in (7, 4, 2, 1)]
    if op == "fp8_sparse":      # nnz: nonzero activations per row at most (None: every k)
        return [dict(xr=2, wr=2, nnz=None), dict(xr=2, wr=1, nnz=None), dict(xr=1, wr=1, nnz=None),
                dict(xr=1, wr=1, nnz=2**13 - 1)]
    raise ValueError(op)


def factors(op, win):
    """(X factors, W factors, epilogue factors) of a window, each a list of (max, quantum)."""
    if op == "int4":
        return [span(_codes(win["xr"], 2.0**-3))], [I4_W], []
    if op in ("int8_dyn", "int8_mm_i32"):
        return [span(_codes(win["r"]))], [span(_codes(win["r"]))], []
    if op == "fp8":
        sc = [o * 2.0**-8 for o in win["odd"]]
        return ([span(_codes(win["xr"], 0.25))], [span(_codes(win["wr"], 0.125))],
                [span(sc), span([v * 2.0**-1 for v in sc])])
    if op == "mxfp8":
        return ([span(_codes(7, 0.25)), span([2.0**e for e in range(-2, -2 + win["dx"] + 1)])],
                [span(_codes(7, 0.125)), span([2.0**e for e in range(-3, -3 + win["dw"] + 1)])], [])
    if op == "nvfp4":
        return ([span([E2M1[c] for c in E2M1_UPTO1]), span([_e4m3(b) for b in win["xb"]])],
                [span(E2M1), span([_e4m3(b) for b in win["wb"]])], [span([win["pts"][0]]), span([win["pts"][1]])])
    if op in ("nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts"):
        epi = [] if op == "nvfp4w" else [span([o * 2.0**-6 for o in win["odd"]])]
        epi.append(span([o * 2.0**-4 for o in win["odd"]]) if op == "nvfp4w_rowpts" else span([win["bp"]]))
        return [span(_codes(win["xr"], 0.5))], [span(E2M1), span([_e4m3(b) for b in win["wb"]])], epi
    if op == "int8wo":
        return [span(_codes(win["xr"], 2.0**-3))], [span(list(range(-128, 128)))], []
    if op == "fp8wo":   # bf16(e4m3 * scale) = (c / 8) * odd * 2^-8, odd in {3, 5, 7}
        return [span(_codes(win["xr"], 2.0**-3))], [span(_codes(win["wr"], 2.0**-3)), span([3.0, 5.0, 7.0])], []
    if op == "mxfp4":
        pw = span([2.0**j for j in range(win["d"] + 1)])
        return [span([E2M1[c] for c in win["xc"]]), pw], [span(E2M1), pw], []
    if op == "fp8_blockwise":   # the codes first: bound() takes the chunk's code sum from them
        return ([span(_codes(win["xr"])), span([2.0**e for e in range(-2, -1 + win["da"])])],
                [span(_codes(win["wr"])), span([2.0**e for e in range(-1, win["dw"])])], [])
    if op == "fp8_sparse":
        return [span(_codes(win["xr"]))], [span(_codes(win["wr"]))], []
    raise ValueError(op)


def bound(op, K, win):
    """(sum bound, chunk bound or None) in output quanta: K max|X| max|W| (times the epilogue's scales) plus the bias,
    and 128 max|X| max|W| for the e4m3 chunk.  Exact when the first is < 2^24 and the second < 2^13."""
    xf, wf, ef = factors(op, win)
    xw = units(xf) * units(wf)
    if op == "fp8_blockwise":   # the chunk's wgmma adds codes; the epilogue rounds as the reference does
        return K * xw, 128 * units(xf[:1]) * units(wf[:1])
    if op == "fp8_sparse":      # one accumulator chain over the whole K; a 4-k group holds at most two weights
        c = min(win["nnz"] or K, K // 2) * xw
        return c, c
    if op in ("int8_dyn", "int8_mm_i32", "int8wo", "fp8wo", "mxfp4"):
        return K * xw, None   # the sum is exact in fp32; the epilogue rounds as the reference does (recipe())
    return K * xw * units(ef) + BIAS_UNITS, (128 * xw if op == "fp8" else None)


def exact(op, K, win):
    s, c = bound(op, K, win)
    return s < 2.0**24 and (c is None or c < 2.0**13)


def window(op, K):
    """The widest window of op that is exact at K."""
    for win in served_candidates(op):
        if exact(op, K, win):
            return win
    raise AssertionError(f"premise: no window of {op} is exact at K={K}")


def _quantum(fs):
    q = 1.0
    for _, low in fs:
        q *= low
    return q


def _reference(op, X, n, wblock, epi, chunk, segment=False):
    """The bf16 (int32) reference [M, n], W_BLOCK features at a time: wblock(n0, n1) -> fp64 W rows; epi(acc, n0, n1)
    -> fp64 output.  The premise is checked on the drawn values of each block as well."""
    M = X.shape[0]
    ref = torch.empty(M, n, dtype=torch.int32 if op == "int8_mm_i32" else torch.bfloat16, device=DEV)
    for n0 in range(0, n, W_BLOCK):
        n1 = min(n, n0 + W_BLOCK)
        W = wblock(n0, n1)
        premise(X, W, chunk=chunk, segment=segment)
        y = epi(X @ W.t(), n0, n1)
        del W
        if op == "int8_mm_i32":
            ref[:, n0:n1] = y.to(torch.int32)
        else:
            fp32_exact(y, f"{op}: the fp64 reference")
            ref[:, n0:n1] = y.float().to(torch.bfloat16)
    return ref


def served(op, M, N, K, seed=0, group_size=32, n_out=None, x_seed=None):
    """A Case of op at a served shape: windows from window(op, K), weights drawn and packed W_BLOCK rows at a time,
    the fp64 reference built per block (no whole fp64 weight is ever resident).  x_seed: other activations (and
    activation scales and bias) with the same weights; case.inputs lists those tensors in a fixed order, so a CUDA
    graph captured on one case can be replayed on another's inputs copied into them."""
    o = ops()
    win = window(op, K)
    xf, wf, ef = factors(op, win)
    Q = _quantum(xf) * _quantum(wf) * _quantum(ef)   # the output quantum: the bias is a multiple of it
    gx = gen((seed if x_seed is None else 1000003 + x_seed) * 7919 + M * 31 + N * 7 + K)
    gw = gen(seed * 7919 + N * 7 + K + 1)
    parts = []

    def blocks(n, make):
        """Runs make(n0, n1) for every block once, in order (the weight generator is sequential)."""
        def wblock(n0, n1):
            W, packed = make(n1 - n0)
            parts.append(packed)
            return W
        return wblock

    if op == "int4":
        g = group_size
        n_out = n_out or N
        X = randint(-win["xr"], win["xr"], (M, K), gx).double() * 2.0**-3
        bias = bias_for(N, Q, gx)

        def make(nb):
            W, qd, sz = int4_weights(nb, K, g, gw)
            return W, (qd, sz)
        # every one of the N packed rows is drawn; the rows past n_out are computed by the tail tile and not stored
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: acc + bias[n0:n1], False)[:, :n_out].contiguous()
        qdata = torch.cat([p[0] for p in parts], 0).contiguous()
        sz = torch.cat([p[1] for p in parts], 0).transpose(0, 1).contiguous()
        x, b = X.to(torch.bfloat16), bias[:n_out].to(torch.bfloat16)
        c = Case(op, "int4", M, N, K, n_out, None, lambda m: o.int4_tilepacked_linear(x[:m], qdata, g, sz, b, n_out, 1),
                 ref=ref)
        c.inputs = [x, b]
        return c
    if op in ("int8_dyn", "int8_mm_i32"):
        r = win["r"]
        xq = randint(-r, r, (M, K), gx).to(torch.int8)
        sx = (pick(ODD, (M, 1), gx) * 2.0**-14).float()
        sw = (pick(ODD, (N,), gw) * 2.0**-10).float()
        b = (randint(-127, 127, (N,), gx).double() * 2.0**-8).to(torch.bfloat16)

        def make(nb):
            wq = randint(-r, r, (nb, K), gw).to(torch.int8)
            return wq.double(), wq

        def epi(acc, n0, n1):
            if op == "int8_mm_i32":
                assert float(acc.abs().max()) < 2.0**24, "premise: int32 sums must convert to fp32 exactly"
                return acc
            return int8_epilogue(acc, sx, sw[n0:n1], b[n0:n1])
        ref = _reference(op, xq.double(), N, blocks(N, make), epi, False)
        wq = torch.cat(parts, 0)
        if op == "int8_mm_i32":
            c = Case(op, "int8", M, N, K, N, None, lambda m: o.int8_mm_i32(xq[:m], wq), out_int=True, ref=ref)
        else:
            c = Case(op, "int8", M, N, K, N, None, lambda m: o.int8_dyn_linear(xq[:m], sx[:m], wq, sw, b), ref=ref)
        c.inputs = [xq, sx, b]
        return c
    if op == "fp8":
        X = randint(-win["xr"], win["xr"], (M, K), gx).double() * 2.0**-2
        rs = pick(win["odd"], (M,), gx) * 2.0**-8
        sw = pick(win["odd"], (N,), gw) * 2.0**-9
        bias = bias_for(N, Q, gx)

        def make(nb):
            W = randint(-win["wr"], win["wr"], (nb, K), gw).double() * 2.0**-3
            return W, W.to(torch.float8_e4m3fn)

        def epi(acc, n0, n1):
            sc = rs[:, None] * sw[None, n0:n1]
            fp32_exact(sc, "fp8: x_scale * w_scale")
            prod = acc * sc
            fp32_exact(prod, "fp8: acc * scales")
            return prod + bias[n0:n1]
        ref = _reference(op, X, N, blocks(N, make), epi, True)
        xq, wq = X.to(torch.float8_e4m3fn), torch.cat(parts, 0)
        rsf, swf, b = rs.float(), sw.float(), bias.to(torch.bfloat16)
        c = Case(op, "fp8", M, N, K, N, None, lambda m: o.fp8_rowwise_linear(xq[:m], rsf[:m], wq, swf, b), ref=ref)
        c.inputs = [xq, rsf, b]
        return c
    if op == "mxfp8":
        Xc = randint(-7, 7, (M, K), gx).double() * 2.0**-2
        xb = randint(125, 125 + win["dx"], (M, K // 32), gx)
        X = Xc * pow2(xb - 127).repeat_interleave(32, 1)
        bias = bias_for(N, Q, gx)

        def make(nb):
            Wc = randint(-7, 7, (nb, K), gw).double() * 2.0**-3
            wb = randint(124, 124 + win["dw"], (nb, K // 32), gw)
            return Wc * pow2(wb - 127).repeat_interleave(32, 1), (Wc.to(torch.float8_e4m3fn), wb.to(torch.uint8))
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: acc + bias[n0:n1], False)
        xq, wq = Xc.to(torch.float8_e4m3fn), torch.cat([p[0] for p in parts], 0)
        xsb, wsb = to_blocked(xb.to(torch.uint8)), to_blocked(torch.cat([p[1] for p in parts], 0))
        b = bias.to(torch.bfloat16)
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = to_blocked(xb[:m].to(torch.uint8))
            return o.mxfp8_linear(xq[:m], cache[m], wq, wsb, b)
        return Case(op, "mxfp8", M, N, K, N, None, run, ref=ref)
    if op == "nvfp4":
        xc = pick(E2M1_UPTO1, (M, K), gx).long()
        xbytes = pick(win["xb"], (M, K // 16), gx).to(torch.uint8)
        X = e2m1_value(xc) * e4m3_bytes_value(xbytes).repeat_interleave(16, 1)
        a, bp = win["pts"]
        bias = bias_for(N, Q, gx)

        def make(nb):
            wc = randint(0, 15, (nb, K), gw)
            wbytes = pick(win["wb"], (nb, K // 16), gw).to(torch.uint8)
            return e2m1_value(wc) * e4m3_bytes_value(wbytes).repeat_interleave(16, 1), (pack_e2m1(wc), wbytes)

        def epi(acc, n0, n1):
            prod = acc * (a * bp)
            fp32_exact(prod, "nvfp4: acc * a_pts * b_pts")
            return prod + bias[n0:n1]
        ref = _reference(op, X, N, blocks(N, make), epi, False)
        xq, wq = pack_e2m1(xc), torch.cat([p[0] for p in parts], 0)
        wsb = to_blocked(torch.cat([p[1] for p in parts], 0))
        a_pts, b_pts = torch.tensor([a], device=DEV), torch.tensor([bp], device=DEV)
        b = bias.to(torch.bfloat16)
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = to_blocked(xbytes[:m])
            return o.nvfp4_linear(xq[:m], cache[m], a_pts, wq, wsb, b_pts, b)
        return Case(op, "nvfp4", M, N, K, N, None, run, ref=ref)
    if op in ("nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts"):
        X = randint(-win["xr"], win["xr"], (M, K), gx).double() * 0.5
        rs = pick(win["odd"], (M,), gx) * 2.0**-6 if op != "nvfp4w" else None
        bp = (pick(win["odd"], (N,), gw) * 2.0**-4 if op == "nvfp4w_rowpts"
              else torch.tensor([win["bp"]], dtype=torch.float64, device=DEV))
        bias = bias_for(N, Q, gx)

        def make(nb):
            wc = randint(0, 15, (nb, K), gw)
            wbytes = pick(win["wb"], (nb, K // 16), gw).to(torch.uint8)
            return e2m1_value(wc) * e4m3_bytes_value(wbytes).repeat_interleave(16, 1), (pack_e2m1(wc), wbytes)

        def epi(acc, n0, n1):
            if rs is not None:
                acc = acc * rs[:, None]
                fp32_exact(acc, "nvfp4w: acc * x_scale")
            prod = acc * (bp[n0:n1] if bp.numel() > 1 else bp).reshape(1, -1)
            fp32_exact(prod, "nvfp4w: acc * b_pts")
            return prod + bias[n0:n1]
        ref = _reference(op, X, N, blocks(N, make), epi, False)
        x, wq = X.to(torch.bfloat16), torch.cat([p[0] for p in parts], 0)
        wsb = to_blocked(torch.cat([p[1] for p in parts], 0))
        rsf, bpf, b = (rs.float() if rs is not None else None), bp.float(), bias.to(torch.bfloat16)
        return Case(op, "nvfp4", M, N, K, N, None,
                    lambda m: o.nvfp4_weight_linear(x[:m], rsf[:m] if rsf is not None else None, wq, wsb, bpf, b), ref=ref)
    if op == "int8wo":
        X = randint(-win["xr"], win["xr"], (M, K), gx).double() * 2.0**-3
        s = (randint(2048, 4095, (N,), gw).double() * 2.0**-20 * pow2(randint(-6, 6, (N,), gw))).float()
        b = (randint(-127, 127, (N,), gx).double() * 2.0**-4).to(torch.bfloat16)

        def make(nb):
            wq = randint(-128, 127, (nb, K), gw).to(torch.int8)
            return wq.double(), wq
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: recipe(op, acc, s[n0:n1], b[n0:n1]).double(), False)
        x, wq = X.to(torch.bfloat16), torch.cat(parts, 0)
        c = Case(op, "int8wo", M, N, K, N, None, lambda m: o.int8_weight_linear(x[:m], wq, s, b), ref=ref)
        c.inputs = [x, b]
        return c
    if op == "fp8wo":
        X = randint(-win["xr"], win["xr"], (M, K), gx).double() * 2.0**-3
        s = (pick([3, 5, 7], (N,), gw) * 2.0**-8).float()
        b = (randint(-127, 127, (N,), gx).double() * 2.0**-4).to(torch.bfloat16)

        def make(nb):
            wq = (randint(-win["wr"], win["wr"], (nb, K), gw).double() * 2.0**-3).to(torch.float8_e4m3fn)
            return (wq.float() * s[len(parts) * W_BLOCK:][:nb, None]).to(torch.bfloat16).double(), wq
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: recipe(op, acc, bias=b[n0:n1]).double(), False)
        x, wq = X.to(torch.bfloat16), torch.cat(parts, 0)
        c = Case(op, "fp8wo", M, N, K, N, None, lambda m: o.fp8_weight_linear(x[:m], wq, s, b), ref=ref)
        c.inputs = [x, b]
        return c
    if op == "mxfp4":
        xc = pick(win["xc"], (M, K), gx).long()
        xs = 126 + randint(0, win["d"], (M, K // 32), gx)
        X = mxfp4_value(xc, xs)
        b = (randint(-127, 127, (N,), gx).double() * 2.0**-4).to(torch.bfloat16)

        def make(nb):
            wc = randint(0, 15, (nb, K), gw)
            ws = 125 + randint(0, win["d"], (nb, K // 32), gw)
            return mxfp4_value(wc, ws), (pack_e2m1(wc), ws.to(torch.uint8))
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: recipe(op, acc, bias=b[n0:n1]).double(), False)
        xq, wq = pack_e2m1(xc), torch.cat([p[0] for p in parts], 0)
        xs8, wsb = xs.to(torch.uint8), to_blocked(torch.cat([p[1] for p in parts], 0))
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = to_blocked(xs8[:m])
            return o.mxfp4_linear(xq[:m], cache[m], wq, wsb, b)
        return Case(op, "mxfp4", M, N, K, N, None, run, ref=ref)
    if op == "fp8_blockwise":
        KB = K // 128
        Xc = randint(-win["xr"], win["xr"], (M, K), gx).double()
        a_s = pow2(randint(-2, -2 + win["da"], (M, KB), gx)).float()
        b = (torch.randn(N, device=DEV, generator=gx) * 4.0).to(torch.bfloat16)
        X = blockwise_values(Xc, a_s, 1)

        def make(nb):
            Wc = randint(-win["wr"], win["wr"], (nb, K), gw).double()
            w_s = pow2(randint(-1, -1 + win["dw"], (nb // 128, KB), gw)).float()
            return blockwise_values(Wc, w_s, 128), (Wc.to(torch.float8_e4m3fn), w_s)
        # the chunk's code sums are bounded by the window (window()); the block premise checks the scaled sums
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: blockwise_epilogue(acc, b[n0:n1]).double(),
                         False)
        xq, wq = Xc.to(torch.float8_e4m3fn), torch.cat([p[0] for p in parts], 0)
        w_s = torch.cat([p[1] for p in parts], 0)
        cache = {}

        def run(m):
            if m not in cache:
                cache[m] = transposed_scales(a_s[:m])
            return o.fp8_blockwise_linear(xq[:m], cache[m], wq, w_s, b)
        return Case(op, "fp8_blockwise", M, N, K, N, None, run, ref=ref)
    if op == "fp8_sparse":
        X = sparse_activations(M, K, win["xr"], win["nnz"], gx)
        x_s, w_s = sparse_scales(M, gx), sparse_scales(N, gw)
        b = (torch.randn(N, device=DEV, generator=gx) * 4.0).to(torch.bfloat16)

        def make(nb):
            W = sparse_codes(nb, K, win["wr"], gw)
            return W, W.to(torch.float8_e4m3fn)
        ref = _reference(op, X, N, blocks(N, make), lambda acc, n0, n1: sparse_epilogue(acc, x_s, w_s[n0:n1], b[n0:n1]),
                         False, segment=True)
        xq = X.to(torch.float8_e4m3fn)
        qd, meta = sparse_compress(torch.cat(parts, 0))   # the metadata's atoms interleave row blocks: compress once
        parts.clear()
        c = Case(op, "fp8_sparse", M, N, K, N, None, lambda m: o.fp8_sparse_linear(xq[:m], x_s[:m], qd, meta, w_s, b),
                 ref=ref)
        c.inputs = [xq, x_s, b]
        return c
    raise ValueError(op)
