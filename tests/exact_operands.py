"""Exactly representable operands for the quantized linears, and their fp64 references (GPU tests only).

Each builder draws codes and scales straight from small sets instead of quantizing random floats.  With those sets
every product X[m,k] * W[n,k] is an integer multiple of one quantum u and every sum stays below 2^24 u, so fp32
accumulates exactly in any order and under any stream-K split; the epilogue's scale products are exact in fp32 as
well.  The kernel's bf16 output must then equal the fp64 reference rounded to bf16, bit for bit, in every element.
Each builder asserts that premise before anything is compared.  Scales have mantissa bits set (int4 s, the e4m3
block scales of nvfp4, the fp8 row scales), so the scale arithmetic is checked too, not only powers of two.
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
    nz = t[t != 0].abs().cpu()   # on the CPU: torch.pow(2.0, e) on CUDA is not exact
    if nz.numel() == 0:
        return 1.0
    m, e = torch.frexp(nz)
    mi = (m * 2.0**53).to(torch.int64)
    return float(((mi & -mi).double() * torch.pow(2.0, (e - 53).double())).min())


def pow2(e):
    """2^e for an integer tensor, exactly (a table: torch.pow on CUDA rounds)."""
    table = torch.tensor([2.0**i for i in range(-160, 161)], dtype=torch.float64, device=e.device)
    return table[e.long() + 160]


def fp32_exact(t, what):
    assert torch.equal(t.float().double(), t), f"premise: {what} is not exact in fp32"


def premise(X, W, bias_acc=None, chunk=False):
    """Asserts max(|X| @ |W|^T) + |bias| < 2^24 u (u = the quantum of every product); returns u.  chunk: the e4m3
    wgmma chain of one 128-k chunk adds in the tensor core's reduced-precision accumulator (DESIGN.md §1), so each
    chunk's sum is also kept under 2^13 u, an assumed width under which that adder is exact."""
    u = lowbit(X) * lowbit(W)
    extra = float(bias_acc.abs().max()) if bias_acc is not None else 0.0
    top = float((X.abs() @ W.abs().t()).max()) + extra
    assert top < 2.0**24 * u, f"premise: sums reach {top / u:.0f} u >= 2^24 u"
    if chunk:
        K = X.shape[1]
        KT = -(-K // 128)
        Xp = torch.nn.functional.pad(X.abs(), (0, KT * 128 - K)).reshape(X.shape[0], KT, 128)
        Wp = torch.nn.functional.pad(W.abs(), (0, KT * 128 - K)).reshape(W.shape[0], KT, 128)
        top_c = float(torch.einsum("mkc,nkc->mnk", Xp, Wp).max())
        assert top_c < 2.0**13 * u, f"premise: a 128-k chunk reaches {top_c / u:.0f} u >= 2^13 u"
    return u


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

    def __init__(self, op, fmt, M, N, K, n_plan, y64, launch, out_int=False):
        self.op, self.fmt, self.M, self.N, self.K, self.n_plan = op, fmt, M, N, K, n_plan
        self.launch = launch
        self.out_int = out_int
        if out_int:
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


def build(op, M, N, K, seed=0, n_out=None, w_bytes=None):
    """op: int4 | int8_dyn | int8_mm_i32 | fp8 | mxfp8 | nvfp4 | nvfp4w | nvfp4w_xs | nvfp4w_rowpts.
    n_out: int4 output features (<= N).  w_bytes: nvfp4 weight scale bytes [N, K/16] (default: a window of normal
    bytes with mantissa bits set)."""
    o = ops()
    g = gen(seed * 7919 + M * 31 + N * 7 + K)
    if op == "int4":
        grp = 64
        n_out = n_out or N
        q = randint(0, 15, (N, K), g)
        s = pick(ODD, (N, K // grp), g) * 2.0**-9
        z = randint(-24, 24, (N, K // grp), g).double() * 2.0**-9
        W = (q.double() - 8) * s.repeat_interleave(grp, 1) + z.repeat_interleave(grp, 1)
        qdata = o.int4_pack_tile4d(((q[:, 0::2] << 4) | q[:, 1::2]).to(torch.uint8).contiguous(), 8)
        sz = torch.stack([s, z], -1).to(torch.bfloat16).transpose(0, 1).contiguous()
        # premise: bf16(fma(q - 8, s, z)) is exact, so the kernel's weights are W itself
        assert torch.equal(o.int4_dequant_tile4d(qdata, sz, grp).double(), W), "premise: int4 weights not exact in bf16"
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
    raise ValueError(op)


def first_mismatch(case, y, M=None):
    bad = (case.bits(y) != case.bits(case.ref(M))).nonzero()
    if bad.numel() == 0:
        return None
    m, n = (int(v) for v in bad[0])
    return m, n, float(y[m, n]), float(case.ref(M)[m, n]), int(bad.shape[0])


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count

