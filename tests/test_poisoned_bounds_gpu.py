"""Every GEMM and activation quantizer run inside poisoned neighbourhoods (tests/poison_arena.py): each operand is copied
into a view whose surroundings (before it, after it, and the gap columns of a row pitch wider than K) hold NaN or
huge finite bytes, and each output and workspace is a view with 4 KiB of poison on either side.

* Dense linears, through the torch ops and through the C ABI: the exact operands of tests/exact_operands.py (and the
  NF4 and static-e4m3 ones of their own modules), every tensor operand carved, bf16 activations at row pitches K + 8
  and K + 64, at M = 1, 33, 200 with N off the 128-row tile and K tails where the format has them, at the default grid
  and at a forced grid under which a tile has 3 or more contributors.  y must equal the exact reference bit for bit.
  Through the ABI, y and the workspace are guarded too: every element of y is written, no guard byte changes, and the
  split-tile flags are back to zero.
* Grouped expert GEMMs and the fp8 bmm, through the C ABI: ragged offs with an empty and a one-token expert, the x rows
  (and per-row scales) from offs[-1] on poisoned as well as everything past M, and the rows of y from offs[-1] on must
  keep their poison.
* Activation quantizers and the RMSNorm / SiLU-mul prologues, through the C ABI: strided rows whose gap columns hold
  poison must give the codes and scales of the same call on a dense copy (so a huge value in the gap moves no scale),
  at K tails off 128 and at K = 16384 + a tail, past the register / CTA schedule boundary; every output guarded.

What these tests cannot see: an over-read whose value never reaches a kept output (a load that is masked afterwards,
or a product with a weight the kernel zero-fills anyway under both poisons) stays invisible, as does a stray write
that lands beyond the 4 KiB guards.  Inputs that the kernels must leave alone are checked to be unchanged as well.
"""
import contextlib
import ctypes
import os

import pytest
import torch

import exact_operands as ex
import grouped_model as gm
import poison_arena as pa
import streamk_model as sk
from test_served_shapes_exact_gpu import ABI as GROUPED_ABI
from test_served_shapes_exact_gpu import BmmCase, MoECase

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 4096          # poison bytes on either side of an output or workspace
FLAG_BYTES = 16384    # the split-tile flag area at the start of the workspace
TOKENS = (1, 33, 200)

# p: pointer (tensor or None), i: int, f: float, z: size_t; the last p is the stream, which call() appends
SIGS = {
    "ao_int8_dyn_linear": "ppiippipppzp", "ao_int8_weight_linear": "piiippipppzp", "ao_int8_mm_i32": "piipippzp",
    "ao_fp8_rowwise_linear": "ppiippipppzp", "ao_fp8_static_linear": "ppiippiippippzp",
    "ao_fp8_blockwise_linear": "ppiippipppzp", "ao_fp8_sparse_linear": "ppiipppipppzp",
    "ao_fp8_weight_linear": "piiippipppzp", "ao_mxfp8_linear": "ppiippipppzp", "ao_mxfp4_linear": "ppiippipppzp",
    "ao_nvfp4_linear": "pppiipppipppzp", "ao_nvfp4_weight_linear_ex": "pipiipppiipppzp",
    "ao_int4_tilepacked_linear_strided": "piiippiippipzip", "ao_nf4_linear": "piiipppppiiipppzp",
    "ao_int8_quantize_rowwise_ld": "piiippp", "ao_fp8_quantize_rowwise_ld": "piiippp",
    "ao_fp8_fakequant_rowwise_ld": "piiippp", "ao_fp8_quantize_1x128_ld": "piiippp",
    "ao_mxfp8_quantize_ld": "piiippip", "ao_mxfp4_quantize_ld": "piiippip", "ao_nvfp4_quantize_ld": "piiipppip",
    "ao_mxfp8_fakequant": "piiipp", "ao_mxfp4_fakequant": "piiipp", "ao_nvfp4_fakequant_grouped": "piiipipppp",
    "ao_int8_quantize_static": "piiipipipiiipppp", "ao_fp8_quantize_static": "piiipippp",
    "ao_rmsnorm_quantize_rowwise": "pipfiiippp", "ao_silu_mul_quantize_rowwise": "pipiiiippp",
}
SIGS.update({name: sig for name, sig in GROUPED_ABI.values()})
_CT = {"p": ctypes.c_void_p, "i": ctypes.c_int, "f": ctypes.c_float, "z": ctypes.c_size_t}


@pytest.fixture(scope="module")
def lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    lib.ao_b200_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    for name, sig in SIGS.items():
        getattr(lib, name).argtypes = [_CT[c] for c in sig]
    return lib


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def call(lib, name, *args):
    conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(lib, name)(*conv, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, f"{name}: {lib.ao_b200_last_error()}"


def guarded(shape, dtype, poison, kind=None):
    """An output arena: the view and 4 KiB on either side hold the poison."""
    return pa.carve(shape, dtype, poison=poison, kind=kind, before=GUARD, after=GUARD)


def workspace(lib, poison, M=0, N=0):
    """A workspace of exactly ao_b200_workspace_bytes, zeroed, inside 4 KiB of poison on either side."""
    ws = pa.carve((int(lib.ao_b200_workspace_bytes(M, N)),), torch.uint8, poison=poison, before=GUARD, after=GUARD)
    ws.view.zero_()
    return ws


def ws_problems(ws):
    bad = []
    if (msg := pa.intact(ws)) is not None:
        bad.append(f"workspace guard: {msg}")
    raised = int(ws.view[:FLAG_BYTES].ne(0).sum())
    if raised:
        bad.append(f"workspace: {raised} flag bytes left raised")
    return bad


def first_diff(got, want):
    bad = (got != want).nonzero()
    if bad.numel() == 0:
        return None
    return f"{bad.shape[0]} elements differ, first at {tuple(int(v) for v in bad[0])}"


# ------------------------------------------------------------------------------------------------ dense linears
# Each torch op's tensor arguments in order, with the poison kind of each (None: not a tensor, or passed through);
# "x" is the bf16 activation, carved at a row pitch wider than K.
KINDS = {
    "int8_dyn_linear": ("i8", "f32", "i8", "f32", "bf16"),
    "int8_weight_linear": ("x", "i8", "f32", "bf16"),
    "int8_mm_i32": ("i8", "i8"),
    "fp8_rowwise_linear": ("e4m3", "f32", "e4m3", "f32", "bf16"),
    "fp8_static_linear": ("e4m3", "f32", "e4m3", "f32", "bf16", None),
    "fp8_blockwise_linear": ("e4m3", "f32", "e4m3", "f32", "bf16"),
    "fp8_sparse_linear": ("e4m3", "f32", "e4m3", "u8", "f32", "bf16"),
    "fp8_weight_linear": ("x", "e4m3", "f32", "bf16"),
    "mxfp8_linear": ("e4m3", "e8m0", "e4m3", "e8m0", "bf16"),
    "mxfp4_linear": ("fp4", "e8m0", "fp4", "e8m0", "bf16"),
    "nvfp4_linear": ("fp4", "e4m3", "f32", "fp4", "e4m3", "f32", "bf16"),
    "nvfp4_weight_linear": ("x", "f32", "fp4", "e4m3", "f32", "bf16"),
    "int4_tilepacked_linear": ("x", "int4", None, "bf16", "bf16", None, None),
    "nf4_linear": ("x", "u8", "i8", "bf16", "bf16", "bf16", None, None, "bf16"),
}


def _ldx(x):
    return x.stride(0) if x.shape[0] > 1 else x.shape[1]


def abi_call(name, a, ws):
    """The C entry point behind torch op `name` called on the op's arguments a: (function name, y shape, y dtype,
    args(y) -> the C arguments without the stream, writing y and using the workspace arena ws)."""
    W = (ws.view, ws.view.numel())
    x = a[0]
    M = x.shape[0]
    if name == "int8_dyn_linear":
        xq, xs, wq, sw, b = a
        return "ao_int8_dyn_linear", (M, wq.shape[0]), torch.bfloat16, lambda y: (xq, xs, M, xq.shape[1], wq, sw, wq.shape[0], b, y, *W)
    if name in ("int8_weight_linear", "fp8_weight_linear"):
        _, wq, s, b = a
        return (f"ao_{name}", (M, wq.shape[0]), torch.bfloat16,
                lambda y: (x, _ldx(x), M, x.shape[1], wq, s, wq.shape[0], b, y, *W))
    if name == "int8_mm_i32":
        xq, wq = a
        return "ao_int8_mm_i32", (M, wq.shape[0]), torch.int32, lambda y: (xq, M, xq.shape[1], wq, wq.shape[0], y, *W)
    if name in ("fp8_rowwise_linear", "fp8_blockwise_linear", "mxfp8_linear", "mxfp4_linear"):
        xq, xs, wq, sw, b = a
        K = xq.shape[1] * (2 if name == "mxfp4_linear" else 1)
        return f"ao_{name}", (M, wq.shape[0]), torch.bfloat16, lambda y: (xq, xs, M, K, wq, sw, wq.shape[0], b, y, *W)
    if name == "fp8_static_linear":   # a per-row weight scale, no output fake-quant
        xq, xs, wq, sw, b, _ = a
        return ("ao_fp8_static_linear", (M, wq.shape[0]), torch.bfloat16,
                lambda y: (xq, xs, M, xq.shape[1], wq, sw, 1, wq.shape[0], b, None, 0, y, *W))
    if name == "fp8_sparse_linear":
        xq, xs, qd, meta, sw, b = a
        return ("ao_fp8_sparse_linear", (M, qd.shape[0]), torch.bfloat16,
                lambda y: (xq, xs, M, xq.shape[1], qd, meta, sw, qd.shape[0], b, y, *W))
    if name == "nvfp4_linear":
        xq, xs, ap, wq, sw, bp, b = a
        return ("ao_nvfp4_linear", (M, wq.shape[0]), torch.bfloat16,
                lambda y: (xq, xs, ap, M, xq.shape[1] * 2, wq, sw, bp, wq.shape[0], b, y, *W))
    if name == "nvfp4_weight_linear":
        _, xs, wq, sw, bp, b = a
        return ("ao_nvfp4_weight_linear_ex", (M, wq.shape[0]), torch.bfloat16,
                lambda y: (x, _ldx(x), xs, M, x.shape[1], wq, sw, bp, int(bp.numel() > 1), wq.shape[0], b, y, *W))
    if name == "int4_tilepacked_linear":
        _, qd, g, sz, b, n_out, impl = a
        return ("ao_int4_tilepacked_linear_strided", (M, n_out), torch.bfloat16,
                lambda y: (x, _ldx(x), M, x.shape[1], qd, sz, g, qd.shape[0] * 8, b, y, n_out, *W, impl))
    if name == "nf4_linear":
        _, qd, qs, f, mean, table, bs, sbs, b = a
        K = x.shape[1]
        N = qd.numel() * 2 // K
        return ("ao_nf4_linear", (M, N), torch.bfloat16,
                lambda y: (x, _ldx(x), M, K, qd, qs, f, mean, table, bs, sbs, N, b, y, *W))
    raise ValueError(name)


class Poisoned:
    """One way of running a GEMM among poison: every tensor operand copied into a carved view (the bf16 activation at
    row pitch K + extra), then the torch op, or (abi) the C entry point with a guarded y and workspace.  Collects what
    went wrong in self.problems."""

    def __init__(self, lib, poison, extra, abi, alias=None):
        self.lib, self.poison, self.extra, self.abi, self.alias = lib, poison, extra, abi, alias
        self.problems = []

    def __call__(self, name, args):
        name = self.alias or name
        carved, new = [], []
        for t, kind in zip(args, KINDS[name] + (None,) * (len(args) - len(KINDS[name]))):
            if isinstance(t, torch.Tensor) and kind is not None:
                pitch = t.shape[1] + self.extra if kind == "x" else None
                arena = pa.carve_like(t, pitch=pitch, poison=self.poison, kind="bf16" if kind == "x" else kind)
                carved.append(arena)
                new.append(arena.view)
            else:
                new.append(t)
        if self.alias == "fp8_static_linear":
            new = new[:5] + [None]
        if not self.abi:
            y = getattr(torch.ops.ao_b200, name)(*new)
        else:
            ws = workspace(self.lib, self.poison)
            cname, shape, dtype, build = abi_call(name, new, ws)
            ya = guarded(shape, dtype, self.poison, kind="i32" if dtype == torch.int32 else None)
            call(self.lib, cname, *build(ya.view))
            if (msg := pa.intact(ya)) is not None:
                self.problems.append(f"y guard: {msg}")
            self.problems += ws_problems(ws)
            y = ya.view
        for i, arena in enumerate(carved):
            if (msg := pa.intact(arena)) is not None:
                self.problems.append(f"operand {i}: {msg}")
        return y


class Carving:
    """torch.ops.ao_b200 as the cases of exact_operands see it: the GEMMs of KINDS go through self.mode when one is
    set, everything else (and every call without a mode) straight to the op."""

    def __init__(self, real):
        self.real, self.mode = real, None

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in KINDS:
            return fn

        def run(*args):
            return fn(*args) if self.mode is None else self.mode(name, args)
        return run


CARVING = Carving(None)


@contextlib.contextmanager
def carving_ops():
    """exact_operands.ops() returns CARVING while cases are built, so their launches go through it."""
    CARVING.real = torch.ops.ao_b200
    saved = ex.ops
    ex.ops = lambda: CARVING
    try:
        yield CARVING
    finally:
        ex.ops = saved


# torch op -> (exact_operands op, N, K, n_out): N off the 128-row tile, K with a tail inside the last 128-k chunk
# where the format allows one (blockwise e4m3 needs K % 128 = N % 128 = 0; nvfp4 K % 256; int4 pads K to 1024)
DENSE = {
    "int8_dyn_linear": ("int8_dyn", 136, 1040, None),
    "int8_weight_linear": ("int8wo", 200, 1040, None),
    "int8_mm_i32": ("int8_mm_i32", 136, 1040, None),
    "fp8_rowwise_linear": ("fp8", 144, 1040, None),
    "fp8_static_linear": ("fp8", 144, 1040, None),   # computes as the rowwise linear does (include/ao_b200.h)
    "fp8_blockwise_linear": ("fp8_blockwise", 256, 1152, None),
    "fp8_sparse_linear": ("fp8_sparse", 208, 1056, None),
    "fp8_weight_linear": ("fp8wo", 200, 1040, None),
    "mxfp8_linear": ("mxfp8", 144, 1056, None),
    "mxfp4_linear": ("mxfp4", 200, 1056, None),
    "nvfp4_linear": ("nvfp4", 144, 1280, None),
    "nvfp4_weight_linear": ("nvfp4w_xs", 144, 1152, None),
    "int4_tilepacked_linear": ("int4", 272, 1024, 264),
}
# NF4: 64-element blocks, 3 scalers per scaler block (its boundaries inside every tile), N = 130, K = 576 (a K tail)
NF4 = (64, 3, 130, 576)


def forced_grid(fmt, M, N, K):
    """A CTA count under which some tile is split over 3 or more CTAs (one CTA per work unit)."""
    U = sk.plan(fmt, M, N, K, grid=1).U
    G = min(U, ex.sm_count())
    p = sk.plan(fmt, M, N, K, grid=G, sm=ex.sm_count())
    assert max(p.contributor_counts(), default=0) >= 2, f"premise: {fmt} M={M} N={N} K={K} grid {G}"
    return G


def _nf4_cases():
    from test_nf4_gpu import Exact

    bs, sbs, N, K = NF4
    cases = {}
    for M in TOKENS:
        c = Exact(M, N, K, bs=bs, sbs=sbs, seed=M)
        t = c.t
        cases[M] = (c, lambda o, t=t, c=c: o.nf4_linear(c.x, t.quantized_data, t.quantized_scalers,
                                                          t.quantization_factor, t.scaler_mean, t.nf4, bs, sbs, c.bias))
    return cases


@pytest.fixture(scope="module")
def dense_cases():
    with carving_ops():
        cases = {op: ex.build(key, max(TOKENS), N, K, seed=11, n_out=n_out) for op, (key, N, K, n_out) in DENSE.items()
                 if op != "fp8_static_linear"}
    cases["fp8_static_linear"] = cases["fp8_rowwise_linear"]
    return cases


@pytest.mark.parametrize("route", ["torch", "abi"])
@pytest.mark.parametrize("poison", pa.POISONS)
@pytest.mark.parametrize("op", list(DENSE) + ["nf4_linear"])
def test_dense_linear_among_poison(lib, set_ctas, dense_cases, op, poison, route):
    bf16_x = KINDS[op][0] == "x"
    extras = (8, 64) if bf16_x else (0,)
    problems = []
    if op == "nf4_linear":   # no stream-K model of its own: 132 CTAs, clamped to the work units, split every tile
        runs = [(M, case, fn, case.ref, 132) for M, (case, fn) in _nf4_cases().items()]
    else:
        case = dense_cases[op]
        runs = [(M, case, None, case.ref(M), forced_grid(case.fmt, M, case.n_plan, case.K)) for M in TOKENS]
    for M, case, fn, ref, G in runs:
        for extra in extras:
            for grid in (0, G):
                mode = Poisoned(lib, poison, extra, route == "abi", alias="fp8_static_linear" if op == "fp8_static_linear" else None)
                CARVING.mode = mode
                set_ctas(grid)
                try:
                    y = fn(CARVING) if fn is not None else case.run(M)
                finally:
                    CARVING.mode = None
                    set_ctas(0)
                where = f"M={M} pitch K+{extra} grid={grid or 'default'}"
                got = y.view(torch.int16) if y.dtype == torch.bfloat16 else y
                want = ref.view(torch.int16) if ref.dtype == torch.bfloat16 else ref
                if (d := first_diff(got, want)) is not None:
                    problems.append(f"{where}: y: {d}")
                problems += [f"{where}: {p}" for p in mode.problems]
    assert not problems, f"{op} [{poison}, {route}]: {len(problems)} problems; " + "; ".join(problems[:4])


# ------------------------------------------------------------------------------------------------ grouped and bmm
ROWS = [37, 0, 1, 90]   # an empty expert and a one-token expert; MoECase adds 3 rows past offs[-1]
# kind -> (N, K): N off the 128-row tile and K tails where the kernel allows them
GROUPED = {"fp8": (144, 1152), "nvfp4": (256, 1152), "int4": (136, 1024), "int8": (136, 1040), "int8wo": (200, 1040),
           "fp8wo": (136, 1040), "fp8_blockwise": (256, 1152), "mxfp8": (256, 1056), "mxfp4": (256, 1056)}
# poison kinds of the uint8 weight tensors of each kind, in argument order
U8_KINDS = {"nvfp4": ["fp4", "e4m3"], "mxfp8": ["e8m0"], "mxfp4": ["fp4", "e8m0"]}
_DT_KIND = {torch.bfloat16: "bf16", torch.float32: "f32", torch.float8_e4m3fn: "e4m3", torch.int8: "i8"}


def _grouped_grid(kind, offs, M, N, K):
    U = gm.plan(offs, M, N, K, grid=1, sm=ex.sm_count(), fmt=kind).U
    G = min(U, ex.sm_count())
    p = gm.plan(offs, M, N, K, grid=G, sm=ex.sm_count(), fmt=kind)
    assert max(p.contributor_counts(), default=0) >= 2, f"premise: grouped {kind} grid {G}"
    return G


@pytest.mark.parametrize("poison", pa.POISONS)
@pytest.mark.parametrize("kind", list(GROUPED))
def test_grouped_gemm_among_poison(lib, set_ctas, kind, poison):
    N, K = GROUPED[kind]
    case = MoECase(lib, kind, ROWS, N, K, seed=5)
    args = list(case.args())
    valid, M = case.valid, case.M
    n_x = next(i for i, a in enumerate(args) if not isinstance(a, torch.Tensor))
    u8 = list(U8_KINDS.get(kind, []))
    kinds = []
    for i, a in enumerate(args[:-1]):
        if not isinstance(a, torch.Tensor):
            kinds.append(None)
        elif i == len(args) - 2:
            kinds.append("i32")   # offs
        elif a.dtype == torch.uint8:
            kinds.append(u8.pop(0))
        elif a.dtype == torch.int32:
            kinds.append("int4")
        else:
            kinds.append(_DT_KIND[a.dtype])
    problems = []
    for grid in (0, _grouped_grid(kind, case.offs_list, M, N, K)):
        carved, new = [], []
        for i, (a, k) in enumerate(zip(args[:-1], kinds)):
            if k is None:
                new.append(a)
                continue
            arena = pa.carve_like(a, poison=poison, kind=k)
            if i < n_x:   # activations and their per-row scales: the rows from offs[-1] on are poison too
                if kind == "fp8_blockwise" and i == 1:
                    arena.fill((slice(None), slice(valid, None)))
                else:
                    arena.fill(slice(valid, None))
            carved.append(arena)
            new.append(arena.view)
        ya = guarded((M, N), torch.int16, poison, kind="bf16")
        ws = workspace(lib, poison, M, N)
        set_ctas(grid)
        call(lib, GROUPED_ABI[kind][0], *new, ya.view, ws.view, ws.view.numel())
        set_ctas(0)
        where = f"grid={grid or 'default'}"
        if (d := first_diff(ya.view[:valid], case.ref.view(torch.int16))) is not None:
            problems.append(f"{where}: y: {d}")
        fill = pa.carve((M - valid, N), torch.int16, poison=poison, kind="bf16", device=ex.DEV).view
        if (d := first_diff(ya.view[valid:], fill)) is not None:
            problems.append(f"{where}: rows from offs[-1] = {valid} on written: {d}")
        if (msg := pa.intact(ya)) is not None:
            problems.append(f"{where}: y guard: {msg}")
        problems += [f"{where}: {p}" for p in ws_problems(ws)]
        problems += [f"{where}: operand {i}: {m}" for i, a in enumerate(carved) if (m := pa.intact(a)) is not None]
    assert not problems, f"grouped {kind} [{poison}] offs={case.offs_list} M={M}: " + "; ".join(problems[:4])


@pytest.mark.parametrize("poison", pa.POISONS)
@pytest.mark.parametrize("layout", ["nk", "kn"])
def test_fp8_bmm_among_poison(lib, set_ctas, layout, poison):
    B, K, N, Ms = 3, 1040, 144, (1, 33)
    case = BmmCase(lib, layout, B, K, N, Ms, seed=9)
    problems = []
    wq = pa.carve_like(case.wq, poison=poison, kind="e4m3")
    sw = pa.carve_like(case.sw, poison=poison)
    for M in Ms:
        xq_t, rs_t, ref = case.x[M]
        xq = pa.carve_like(xq_t.view(torch.uint8), poison=poison, kind="e4m3")
        rs = pa.carve_like(rs_t, poison=poison)
        U = gm.plan([(b + 1) * M for b in range(B)], B * M, N, K, grid=1, fmt="fp8").U
        for grid in (0, min(U, ex.sm_count())):
            ya = guarded((B * M, N), torch.int16, poison, kind="bf16")
            ws = workspace(lib, poison)
            set_ctas(grid)
            call(lib, "ao_fp8_rowwise_bmm", xq.view, rs.view, B, M, K, wq.view, sw.view, N, int(layout == "kn"), ya.view,
                 ws.view, ws.view.numel())
            set_ctas(0)
            where = f"M={M} grid={grid or 'default'}"
            if (d := first_diff(ya.view, ref.view(torch.int16))) is not None:
                problems.append(f"{where}: y: {d}")
            if (msg := pa.intact(ya)) is not None:
                problems.append(f"{where}: y guard: {msg}")
            problems += [f"{where}: {p}" for p in ws_problems(ws)]
        problems += [f"M={M}: operand: {m}" for a in (xq, rs) if (m := pa.intact(a)) is not None]
    problems += [f"weights: {m}" for a in (wq, sw) if (m := pa.intact(a)) is not None]
    assert not problems, f"bmm {layout} [{poison}]: " + "; ".join(problems[:4])


# ------------------------------------------------------------------------------------------------ quantizers
def _blocked(rows, scale_cols):
    return (-(-rows // 128) * 32, -(-scale_cols // 4) * 16)


def quantizers():
    """name -> (K multiple, outputs(M, K) -> [(shape, dtype, kind)], launch(lib, x, ldx, M, K, outs, extra) where extra
    holds the call's other inputs)."""
    def rowwise(fn, code_dtype, code_kind):
        return (8, lambda M, K: [((M, K), code_dtype, code_kind), ((M,), torch.float32, "f32")],
                lambda lib, x, ldx, M, K, o, e: call(lib, fn, x, ldx, M, K, *o))

    def mx(fn, fp4, swz):
        def outs(M, K):
            codes = ((M, K // 2), torch.uint8, "fp4") if fp4 else ((M, K), torch.uint8, "e4m3")
            return [codes, (_blocked(M, K // 32) if swz else (M, K // 32), torch.uint8, "e8m0")]
        return 32, outs, lambda lib, x, ldx, M, K, o, e: call(lib, fn, x, ldx, M, K, *o, int(swz))

    def nvfp4(swz):
        def outs(M, K):
            return [((M, K // 2), torch.uint8, "fp4"), (_blocked(M, K // 16) if swz else (M, K // 16), torch.uint8, "e4m3")]
        return (16, outs, lambda lib, x, ldx, M, K, o, e: call(lib, "ao_nvfp4_quantize_ld", x, ldx, M, K, e["pts"], *o,
                                                              int(swz)))

    def fakequant(fn, mult):
        return mult, lambda M, K: [((M, K), torch.bfloat16, "bf16")], lambda lib, x, ldx, M, K, o, e: call(lib, fn, x, ldx, M, K, *o)

    def grouped(M, K):
        return [((M, K), torch.bfloat16, "bf16"), ((M,), torch.float32, "f32"), ((M,), torch.float32, "f32")]

    def int8_static(pre):
        return (8, lambda M, K: [((M, K), torch.int8, "i8"), ((M,), torch.float32, "f32")],
                lambda lib, x, ldx, M, K, o, e: call(lib, "ao_int8_quantize_static", x, ldx, M, K,
                                                     e["pre"] if pre else None, 1 if pre else 0, e["scale"], 0, None, 0,
                                                     -128, 127, *o, None))

    def prologue(fmt):
        dt, kd = (torch.int8, "i8") if fmt == 0 else (torch.uint8, "e4m3")
        return (8, lambda M, K: [((M, K), dt, kd), ((M,), torch.float32, "f32")],
                lambda lib, x, ldx, M, K, o, e: call(lib, "ao_rmsnorm_quantize_rowwise", x, ldx, e["weight"], 1e-5, M, K,
                                                     fmt, *o))

    def silu(fmt):
        dt, kd = (torch.int8, "i8") if fmt == 0 else (torch.uint8, "e4m3")
        # gate at the pitch under test, up at a pitch 56 elements wider
        return (8, lambda M, K: [((M, K), dt, kd), ((M,), torch.float32, "f32")],
                lambda lib, x, ldx, M, K, o, e: call(lib, "ao_silu_mul_quantize_rowwise", x, ldx, e["up"](ldx), e["up_ld"](ldx),
                                                     M, K, fmt, *o))

    return {
        "int8_rowwise": rowwise("ao_int8_quantize_rowwise_ld", torch.int8, "i8"),
        "fp8_rowwise": rowwise("ao_fp8_quantize_rowwise_ld", torch.uint8, "e4m3"),
        "fp8_fakequant": (8, lambda M, K: [((M, K), torch.bfloat16, "bf16"), ((M,), torch.float32, "f32")],
                          lambda lib, x, ldx, M, K, o, e: call(lib, "ao_fp8_fakequant_rowwise_ld", x, ldx, M, K, *o)),
        "fp8_1x128": (128, lambda M, K: [((M, K), torch.uint8, "e4m3"), ((K // 128, (M + 3) // 4 * 4), torch.float32, "f32")],
                      lambda lib, x, ldx, M, K, o, e: call(lib, "ao_fp8_quantize_1x128_ld", x, ldx, M, K, *o)),
        "mxfp8": mx("ao_mxfp8_quantize_ld", False, False), "mxfp8_swizzled": mx("ao_mxfp8_quantize_ld", False, True),
        "mxfp4": mx("ao_mxfp4_quantize_ld", True, False), "mxfp4_swizzled": mx("ao_mxfp4_quantize_ld", True, True),
        "nvfp4": nvfp4(False), "nvfp4_swizzled": nvfp4(True),
        "mxfp8_fakequant": fakequant("ao_mxfp8_fakequant", 32), "mxfp4_fakequant": fakequant("ao_mxfp4_fakequant", 32),
        "nvfp4_fakequant_grouped": (16, grouped, lambda lib, x, ldx, M, K, o, e: call(
            lib, "ao_nvfp4_fakequant_grouped", x, ldx, M, K, e["offs"], 3, *o)),
        "int8_static": int8_static(False), "int8_static_prescale": int8_static(True),
        "fp8_static": (8, lambda M, K: [((M, K), torch.uint8, "e4m3"), ((M,), torch.float32, "f32")],
                       lambda lib, x, ldx, M, K, o, e: call(lib, "ao_fp8_quantize_static", x, ldx, M, K, e["scale"], 0, *o)),
        "rmsnorm_int8": prologue(0), "rmsnorm_fp8": prologue(1), "silu_mul_int8": silu(0), "silu_mul_fp8": silu(1),
    }


QUANTIZERS = quantizers()
# K = 1032 / 4104 / 16392 rounded up to each format's multiple: tails off 128, and past the 16384 boundary of the
# register / CTA row schedule
BASE_K = (1032, 4104, 16392)
Q_TOKENS = (1, 37)   # 37: the 1x128 scales carry 3 padding columns (round_up(M, 4) = 40)


def _k_values(mult):
    return sorted({-(-k // mult) * mult for k in BASE_K})


@pytest.mark.parametrize("poison", pa.POISONS)
@pytest.mark.parametrize("name", list(QUANTIZERS))
def test_quantizer_strided_rows_among_poison(lib, name, poison):
    """Strided rows with poison in the gap columns against the same call on a dense copy: every output byte equal (a
    huge value in the gap moves no scale), every output guarded.  The 1x128 scales' padding columns m >= M are written
    as 0, as include/ao_b200.h states; the blocked scale layouts' padding is whatever the dense call writes."""
    mult, outs, launch = QUANTIZERS[name]
    problems = []
    g = ex.gen(31)
    for K in _k_values(mult):
        for M in Q_TOKENS:
            x = (torch.randn(M, K, device=ex.DEV, generator=g) * 2).to(torch.bfloat16)
            up = (torch.randn(M, K, device=ex.DEV, generator=g)).to(torch.bfloat16)
            keep = []

            def up_at(ldx):
                a = pa.carve_like(up, pitch=ldx + 56 if ldx > K else None, poison=poison)
                keep.append(a)
                return a.view

            extra = {"pts": (x.float().abs().amax() / (448.0 * 6.0)).reshape(1),
                     "pre": (torch.rand(K, device=ex.DEV, generator=g) + 0.5).to(torch.bfloat16),
                     "scale": (x.float().abs().amax() / 100.0).reshape(1),
                     "weight": (torch.rand(K, device=ex.DEV, generator=g) + 0.5).to(torch.bfloat16),
                     "offs": torch.tensor([M // 3, M // 3, M], dtype=torch.int32, device=ex.DEV),
                     "up": up_at, "up_ld": lambda ldx: ldx + 56 if ldx > K else K}
            extra = {k: (pa.carve_like(v, poison=poison).view if isinstance(v, torch.Tensor) else v) for k, v in extra.items()}
            results = {}
            for extra_cols in (0, 8, 64):
                xa = pa.carve_like(x, pitch=K + extra_cols if extra_cols else None, poison=poison)
                oa = [guarded(s, dt, poison, kind=kd) for s, dt, kd in outs(M, K)]
                launch(lib, xa.view, K + extra_cols, M, K, [a.view for a in oa], extra)
                results[extra_cols] = oa
                where = f"K={K} M={M} pitch K+{extra_cols}"
                problems += [f"{where}: output {i} guard: {m}" for i, a in enumerate(oa) if (m := pa.intact(a)) is not None]
                problems += [f"{where}: input: {m}" for a in [xa] + keep if (m := pa.intact(a)) is not None]
                if extra_cols:
                    for i, (a, d) in enumerate(zip(oa, results[0])):
                        if (dd := first_diff(a.view.view(torch.uint8), d.view.view(torch.uint8))) is not None:
                            problems.append(f"{where}: output {i} differs from the dense call's: {dd}")
            if name == "fp8_1x128" and M % 4:
                pad = results[0][1].view[:, M:]
                if not bool((pad == 0).all()):
                    problems.append(f"K={K} M={M}: 1x128 scale padding columns not written as 0")
    assert not problems, f"{name} [{poison}]: {len(problems)} problems; " + "; ".join(problems[:4])
