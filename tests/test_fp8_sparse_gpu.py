"""2:4-sparse e4m3 linears on the H100 (Float8DynamicActivationFloat8WeightConfig, packing_format
SPARSE_2D_DATA_2D_METADATA): the compressed layout and the GEMM against the reference's own CUTLASS kernels
(oracle/_ref, built by oracle/ref_sparse.py), the GEMM bit for bit on exact operands under every forced stream-K grid,
the handler end to end, and a PDL chain against a serialized run.
"""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import streamk_model as sk
from exact_operands import ODD, POISON_BF16, gen, lowbit, pow2, randint

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
E4M3 = torch.float8_e4m3fn
SERVED = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


@pytest.fixture(scope="module")
def ref():
    sys.path.insert(0, ROOT)
    from oracle import ref_sparse

    try:
        return ref_sparse.load()
    except FileNotFoundError as e:
        pytest.skip(f"the reference's sparse fp8 kernels are not built: missing {e}")


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def bits(t):
    return t.contiguous().view(torch.int16)


def u8(t):
    return t.contiguous().view(torch.uint8)


def compress(q):
    from ao_b200.quantization.quantize_.workflows.float8.float8_sparse_2x4_2d_data_2d_metadata_tensor import \
        compress_2x4_e4m3

    return compress_2x4_e4m3(q)


def prune_mask(N, K, g, keep=2):
    """[N, K] bool: `keep` random positions of each group of 4"""
    r = torch.rand(N, K // 4, 4, device=DEV, generator=g)
    idx = r.argsort(-1)[..., :keep]
    return torch.zeros(N, K // 4, 4, dtype=torch.bool, device=DEV).scatter_(-1, idx, True).reshape(N, K)


def pruned_codes(N, K, seed, edge=True):
    """random e4m3 codes, 2:4 pruned; with edge: groups with 0 and 1 nonzero codes (at every position) and -0.0"""
    g = gen(seed)
    w = torch.randn(N, K, device=DEV, generator=g) * 3.0
    w = w * prune_mask(N, K, g)
    q = w.to(E4M3)
    if edge:
        u = q.view(torch.uint8).reshape(N, K // 4, 4)
        kind = torch.randint(0, 8, (N, K // 4), device=DEV, generator=g)
        u[kind == 0] = 0                                            # empty group
        for p in range(4):                                          # one code at position p
            one = torch.zeros(4, dtype=torch.uint8, device=DEV)
            one[p] = 0x38 + p
            u[kind == 1 + p] = one
        u[kind == 5] = torch.tensor([0x80, 0x44, 0x80, 0xC0], dtype=torch.uint8, device=DEV)   # -0.0 beside codes
        u[kind == 6] = torch.tensor([0x80, 0x80, 0x80, 0x80], dtype=torch.uint8, device=DEV)   # all -0.0
    return q


# ---------------------------------------------------------------- 1. the layout against the reference's compressor
@pytest.mark.parametrize("N,K", [(64, 128), (128, 160), (192, 192), (80, 224), (48, 4096 + 96), (16, 32), (200, 352)])
def test_layout_matches_reference_compressor(ref, N, K):
    q = pruned_codes(N, K, seed=N * 31 + K)
    qd, meta = compress(q)
    rq, rm = ref.to_sparse_semi_structured_cutlass_sm9x_f8(q)
    torch.cuda.synchronize()
    assert tuple(rm.shape) == tuple(meta.shape) == ((N + 63) // 64 * 64, (K + 127) // 128 * 16)
    assert torch.equal(u8(qd), u8(rq)), "compressed codes"
    assert torch.equal(u8(meta), u8(rm)), f"metadata: {int((u8(meta) != u8(rm)).sum())} bytes differ"


@pytest.mark.parametrize("proj", sorted(SERVED))
def test_layout_matches_reference_compressor_llama3_8b(ref, proj):
    N, K = SERVED[proj]
    q = pruned_codes(N, K, seed=7, edge=False)
    qd, meta = compress(q)
    rq, rm = ref.to_sparse_semi_structured_cutlass_sm9x_f8(q)
    assert torch.equal(u8(qd), u8(rq)) and torch.equal(u8(meta), u8(rm)), proj


# ---------------------------------------------------------------- 2. the GEMM on exact operands
def accumulator_premise(X, W):
    """SparseF8Fmt does not promote: a whole segment's K sum stays in the tensor core's fp8 accumulator, assumed exact
    below 2^13 quanta (exact_operands.premise, chunk=True, for one chunk).  Asserts max(|X| @ |W|^T) < 2^13 u for the
    codes X [M, K] and the decompressed weight codes W [N, K] (fp64), so that no split or K order can round."""
    u = lowbit(X) * lowbit(W)
    top = float((X.abs() @ W.abs().t()).max())
    assert top < 2.0**13 * u, f"premise: a sum reaches {top / u:.0f} u >= 2^13 u"


class Exact:
    """codes x, w in -r..r (e4m3 integers; r = 2, or 1 once K/2 * 4 would pass 2^13), w 2:4 pruned: every sum is an
    integer below 2^13 (asserted), exact in the fp8 accumulator and in fp32 in any order and under any split.  Scales
    2^e * ODD / 8 have mantissa bits, so the epilogue's node order is checked: the reference is
    t = fp32(acc * w_s[n]), then fp32(t * x_s[m] + bias[n]) rounded once (the FFMA of the reference's build,
    DESIGN §2g), then bf16."""

    def __init__(self, M, N, K, seed=0, bias=True):
        g = gen(seed * 1000003 + M * 131 + N * 7 + K)
        self.M, self.N, self.K = M, N, K
        r = 2 if 4 * (K // 2) < 2**13 else 1
        X = randint(-r, r, (M, K), g).double()
        W = randint(-r, r, (N, K), g).double() * prune_mask(N, K, g)
        accumulator_premise(X, W)
        self.x_s = (pow2(randint(-3, 1, (M,), g)) * torch.tensor(ODD, device=DEV, dtype=torch.float64)[
            randint(0, len(ODD) - 1, (M,), g)] / 8).float()
        self.w_s = (pow2(randint(-3, 1, (N,), g)) * torch.tensor(ODD, device=DEV, dtype=torch.float64)[
            randint(0, len(ODD) - 1, (N,), g)] / 8).float()
        self.xq, wq = X.to(E4M3), W.to(E4M3)
        self.qd, self.meta = compress(wq)
        self.bias = (torch.randn(N, device=DEV, generator=g) * 4.0).to(torch.bfloat16) if bias else None
        acc = X @ W.t()
        assert torch.equal(acc.float().double(), acc), "premise: the sums are exact in fp32"
        t = (acc.float() * self.w_s[None, :]).double() * self.x_s[:, None].double()   # exact in fp64
        t = t + (self.bias.double()[None, :] if bias else 0.0)
        self.ref = t.float().to(torch.bfloat16)

    def run(self, ops, m=None, meta=None):
        m = self.M if m is None else m
        return ops.fp8_sparse_linear(self.xq[:m], self.x_s[:m], self.qd, self.meta if meta is None else meta,
                                     self.w_s, self.bias)

    def check(self, ops, m=None, what="", meta=None):
        m = self.M if m is None else m
        y = self.run(ops, m, meta)
        bad = bits(y) != bits(self.ref[:m])
        assert not bool(bad.any()), f"M={m} N={self.N} K={self.K} {what}: {int(bad.sum())} wrong, first at {bad.nonzero()[0].tolist()}"
        assert not bool(ops.debug_workspace(y).view(torch.int32)[:4096].ne(0).any()), f"M={m} {what}: flags left raised"
        bits(y).fill_(POISON_BF16)


def grids(M, N, K):
    U = sk.plan("fp8_sparse", M, N, K, grid=1).U
    return list(range(1, min(U, 132) + 1))


@pytest.mark.parametrize("M,N,K", [(16, 256, 1024), (64, 384, 2048), (129, 128, 4096), (200, 80, 1440)])
def test_every_forced_grid_bit_exact(ops, set_ctas, M, N, K):
    case = Exact(M, N, K)
    for G in grids(M, N, K):
        set_ctas(G)
        case.check(ops, what=f"grid={G}")
    set_ctas(0)
    case.check(ops, what="default grid")


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("N,K", [(128, 128), (384, 1184), (48, 96)])
def test_token_tiles_and_tails_bit_exact(ops, set_ctas, N, K, bias):
    case = Exact(300, N, K, seed=1, bias=bias)
    for G in (0, 1, 3, 7, 132):
        set_ctas(G)
        for m in (1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 300):
            case.check(ops, m, what=f"grid={G}")


@pytest.mark.parametrize("proj", sorted(SERVED))
def test_llama3_8b_shapes_bit_exact(ops, proj):
    N, K = SERVED[proj]
    case = Exact(512, N, K, seed=4)
    for m in (1, 4, 32, 128, 512):
        case.check(ops, m, what=proj)


def test_padding_metadata_is_never_used(ops):
    """pad rows (n >= N) and pad k (k >= K) of the metadata filled with every byte value, among them the undefined
    nibbles 0b0000 / 0b0101 / 0b1010 / 0b1111: the outputs stay bit-exact"""
    case = Exact(37, 80, 160, seed=5)
    rows = meta_rows(case.meta).clone()
    g = gen(11)
    garbage = torch.randint(0, 256, rows.shape, device=DEV, generator=g, dtype=torch.int32).to(torch.uint8)
    pad = torch.ones_like(rows, dtype=torch.bool)
    pad[:80, :160 // 8] = False
    rows[pad] = garbage[pad]
    for m in (1, 16, 37):
        case.check(ops, m, what="garbage pad", meta=from_rows(rows))


def meta_rows(meta):
    from ao_b200.quantization.quantize_.workflows.float8.float8_sparse_2x4_2d_data_2d_metadata_tensor import \
        metadata_rows

    return metadata_rows(meta)


def from_rows(rows):
    Np, kb = rows.shape
    return rows.reshape(Np // 64, 64, kb // 16, 16).permute(2, 0, 1, 3).contiguous().reshape(Np, kb)


# ---------------------------------------------------------------- 3. against the reference's GEMM
def ref_linear(ref, xq, x_s, qd, meta, w_s, bias):
    return ref.rowwise_scaled_linear_sparse_cutlass_f8f8(xq, x_s, qd, meta, w_s, bias, torch.bfloat16)


@pytest.mark.parametrize("M,N,K", [(1, 64, 128), (16, 128, 256), (33, 48, 160), (128, 256, 1024), (300, 64, 4096),
                                   (77, 4096, 4096)])
@pytest.mark.parametrize("bias", [False, True])
def test_exact_operands_bit_identical_to_reference_gemm(ops, ref, M, N, K, bias):
    case = Exact(M, N, K, seed=2, bias=bias)
    r = ref_linear(ref, case.xq, case.x_s, case.qd, case.meta, case.w_s, case.bias)
    y = case.run(ops)
    assert torch.equal(bits(r), bits(case.ref)), "the reference GEMM differs from the restated epilogue order"
    assert torch.equal(bits(y), bits(r))


@pytest.mark.parametrize("M,N,K", [(33, 48, 160), (7, 64, 4096 + 96)])
def test_garbage_metadata_padding_matches_reference_gemm(ops, ref, M, N, K):
    """the metadata's pad rows (n >= N, up to 64) and pad k (k >= K, up to the next 128) filled with every byte value,
    among them the undefined nibbles 0b0000 / 0b0101 / 0b1010 / 0b1111: this engine's output on it equals, bit for
    bit, the reference GEMM's on the compressor's own (zero) padding"""
    case = Exact(M, N, K, seed=9)
    rows = meta_rows(case.meta).clone()
    pad = torch.ones_like(rows, dtype=torch.bool)
    pad[:N, :K // 8] = False
    assert bool(pad.any()), "premise: the shape has metadata padding"
    garbage = torch.randint(0, 256, rows.shape, device=DEV, generator=gen(12), dtype=torch.int32).to(torch.uint8)
    rows[pad] = garbage[pad]
    r = ref_linear(ref, case.xq, case.x_s, case.qd, case.meta, case.w_s, case.bias)
    y = case.run(ops, meta=from_rows(rows))
    assert torch.equal(bits(y), bits(r))


# |y - ref| <= RANDOM_TOL * sum_k |x[m,k] w[n,k]| (dequantized) + one bf16 ulp of ref.  Both GEMMs accumulate in the
# tensor core's fp8 accumulator without promotion (FP8FastAccum), which keeps fewer bits than fp32, and they split K
# differently, so the results differ by a fraction of the sum of |products|: at most 1.9e-4 on an H100 (DESIGN §2g).
# With one CTA per tile (no stream-K split) the two agreed bit for bit at every shape here
RANDOM_TOL = 2**-11


@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (32, 6144, 4096), (128, 4096, 14336), (512, 1024, 4096),
                                   (5, 64, 4096 + 96)])
def test_random_operands_agree_with_reference_gemm(ops, ref, set_ctas, M, N, K):
    from ao_b200.quantization import Float8Tensor, PerRow

    g = gen(M + N + K)
    x = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV, generator=g) * prune_mask(N, K, g)).to(torch.bfloat16)
    xt = Float8Tensor.from_hp(x, granularity=PerRow())
    wt = Float8Tensor.from_hp(w, granularity=PerRow())
    qd, meta = compress(wt.qdata)
    bias = torch.randn(N, device=DEV, generator=g).to(torch.bfloat16)
    args = (xt.qdata, xt.scale.reshape(-1), qd, meta, wt.scale.reshape(-1), bias)
    y, r = ops.fp8_sparse_linear(*args), ref_linear(ref, *args)
    absprod = (xt.qdata.float().abs() * xt.scale.float()) @ (wt.qdata.float().abs() * wt.scale.float()).t()
    ulp = torch.finfo(torch.bfloat16).eps * r.float().abs()
    ratio = float(((y.float() - r.float()).abs() - ulp).clamp_min(0).div(absprod.clamp_min(1e-30)).max())
    # one CTA per tile (no stream-K split): an observation, not a requirement
    set_ctas((N + 127) // 128 * ((M + 127) // 128 if M > 64 else 1))
    unsplit = bool(torch.equal(bits(ops.fp8_sparse_linear(*args)), bits(r)))
    set_ctas(0)
    print(f"M={M} N={N} K={K}: max |diff| / sum|products| {ratio:.3e}; bit-identical: default grid "
          f"{bool(torch.equal(bits(y), bits(r)))}, one CTA per tile {unsplit}")
    assert ratio <= RANDOM_TOL


# ---------------------------------------------------------------- 4. end to end through quantize_
def sparse_config():
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8PackingFormat, PerRow

    return Float8DynamicActivationFloat8WeightConfig(granularity=PerRow(),
                                                     packing_format=Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA)


def pruned_linear(K, N, bias, seed, exact=False):
    """a 2:4-pruned bf16 linear; exact: weights in {-2..2} with every row reaching |2|, so the per-row codes are
    0, +-224, +-448 and every product sum of the GEMM is exact in fp32"""
    torch.manual_seed(seed)
    lin = nn.Linear(K, N, bias=bias, device=DEV, dtype=torch.bfloat16)
    g = gen(seed)
    with torch.no_grad():
        mask = prune_mask(N, K, g)
        if exact:
            w = randint(-2, 2, (N, K), g).to(torch.bfloat16)
            w[:, 0] = 2.0
            mask[:, :4] = torch.tensor([True, False, False, True], device=DEV)
            lin.weight.copy_(w)
        lin.weight.mul_(mask)
    return lin


def exact_input(*shape):
    """activations in {-2..2} with every row reaching |2| (per-token codes 0, +-224, +-448) and at most 16 nonzeros
    per row, so that with exact weights every sum stays under the accumulator premise"""
    g = gen(sum(shape))
    x = torch.zeros(shape, device=DEV)
    pos = torch.rand(shape, device=DEV, generator=g).argsort(-1)[..., :15]
    x.scatter_(-1, pos, randint(-2, 2, (*shape[:-1], 15), g).float())
    x[..., 0] = -2.0
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("shape", [(7, 1024), (2, 9, 1024), (300, 1024), (1, 1024)])
@pytest.mark.parametrize("bias", [False, True])
def test_quantize_end_to_end_equals_reference_recipe(ops, ref, shape, bias):
    """each linear of a quantized stack on exact activations (every sum exact in fp32, so the two GEMMs' different
    accumulation cannot show) against the reference's recipe: this engine's per-token quantizer, then the reference op"""
    from ao_b200.quantization import Float8Sparse2x4_2DData2DMetadataTensor, Float8Tensor, PerRow, quantize_

    stack = nn.Sequential(pruned_linear(1024, 512, bias, 1, exact=True), pruned_linear(512, 1024, bias, 2, exact=True))
    w_hp = [l.weight.detach().clone() for l in stack]
    quantize_(stack, sparse_config())
    assert all(isinstance(l.weight, Float8Sparse2x4_2DData2DMetadataTensor) for l in stack)
    with torch.no_grad():
        for l in stack:
            x = exact_input(*shape[:-1], l.weight.shape[1])
            y = l(x)
            xt = Float8Tensor.from_hp(x.reshape(-1, x.shape[-1]), granularity=PerRow())
            w = l.weight
            accumulator_premise(xt.qdata.double(), decompressed(w).double())
            r = ref_linear(ref, xt.qdata, xt.scale.reshape(-1), w.qdata, w.sparse_metadata, w.scale.reshape(-1),
                           l.bias).reshape(*x.shape[:-1], -1)
            assert y.shape == (*shape[:-1], w.shape[0]) and y.dtype == torch.bfloat16
            assert torch.equal(bits(y), bits(r))
        y = stack(x.new_ones(*shape[:-1], 1024))
        assert y.shape == (*shape[:-1], 1024)
    for l, hp in zip(stack, w_hp):
        w = l.weight
        rd = ref_linear(ref, torch.eye(w.shape[1], device=DEV).to(E4M3), torch.ones(w.shape[1], device=DEV),
                        w.qdata, w.sparse_metadata, w.scale.reshape(-1), None).t()
        assert torch.equal(bits(w.dequantize()), bits(rd))
        assert torch.equal(w.to(torch.float).view(torch.int32), rd.float().view(torch.int32))
        dense = Float8Tensor.from_hp(hp, granularity=PerRow())
        dq = u8(dense.qdata)
        dq = torch.where((dq & 0x7F) == 0, torch.zeros_like(dq), dq)   # -0.0 is never stored
        assert torch.equal(dq, u8(decompressed(w))), "codes are the dense PerRow codes"


def decompressed(w):
    from ao_b200.quantization.quantize_.workflows.float8.float8_sparse_2x4_2d_data_2d_metadata_tensor import \
        decompress_2x4_e4m3

    return decompress_2x4_e4m3(w.qdata, w.sparse_metadata)


# ---------------------------------------------------------------- 5. PDL handoff
CHAIN = """
import sys, torch
sys.path.insert(0, {root!r})
sys.path.insert(0, {tests!r})
from test_fp8_sparse_gpu import pruned_linear, sparse_config
from ao_b200.quantization import quantize_
ls = [pruned_linear(2048, 2048, True, 20 + i) for i in range(2)]
for l in ls:
    quantize_(l, sparse_config())
outs = []
with torch.no_grad():
    for M in (1, 32, 300):
        torch.manual_seed(M)
        x = torch.randn(M, 2048, device="cuda", dtype=torch.bfloat16)
        outs.append(ls[1](ls[0](x)))
torch.cuda.synchronize()
sys.stdout.buffer.write(b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs))
"""


def test_pdl_chain_matches_serialized():
    """Two sparse linears back to back (the second's quantizer and GEMM start under the kernel ahead of them) against
    the same launches separated by synchronisations, and against a process that launches without PDL."""
    from ao_b200.quantization import quantize_

    ls = [pruned_linear(2048, 2048, True, 20 + i) for i in range(2)]
    for l in ls:
        quantize_(l, sparse_config())
    outs = []
    with torch.no_grad():
        for M in (1, 32, 300):
            torch.manual_seed(M)
            x = torch.randn(M, 2048, device=DEV, dtype=torch.bfloat16)
            chained = ls[1](ls[0](x))
            a = ls[0](x)
            torch.cuda.synchronize()
            serial = ls[1](a)
            torch.cuda.synchronize()
            assert torch.equal(bits(chained), bits(serial)), f"M={M}"
            outs.append(chained)
    here = b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs)
    for no_pdl in ("0", "1"):
        env = dict(os.environ, AO_B200_NO_PDL=no_pdl)
        r = subprocess.run([sys.executable, "-c", CHAIN.format(root=ROOT, tests=os.path.dirname(__file__))], env=env,
                           stdout=subprocess.PIPE, check=True)
        assert r.stdout == here, f"AO_B200_NO_PDL={no_pdl}: the chain's outputs differ"


def test_save_load_and_clone_on_device(tmp_path):
    from ao_b200.quantization import quantize_

    lin = pruned_linear(512, 256, True, 3)
    quantize_(lin, sparse_config())
    x = torch.randn(5, 512, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y = lin(x)
    torch.save(lin.state_dict(), tmp_path / "w.pt")
    lin2 = nn.Linear(512, 256, device=DEV, dtype=torch.bfloat16)
    lin2.load_state_dict(torch.load(tmp_path / "w.pt", weights_only=True), assign=True)
    w3 = lin.weight.clone()
    with torch.no_grad():
        assert torch.equal(bits(lin2(x)), bits(y))
        assert torch.equal(bits(torch.nn.functional.linear(x, w3, lin.bias)), bits(y))
