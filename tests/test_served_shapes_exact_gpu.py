"""Every quantized GEMM checked bit for bit at the shapes the library serves: the Llama-3 projections of bench.py at
decode and prefill token counts; the MoE expert layers of Mixtral-8x7B and Qwen3-30B-A3B with routings drawn from a
skewed top-k (plus synthetic E = 256 and E = MAX_EXPERTS = 1024) for every grouped expert kernel, and DeepSeek-V3's
experts (weight stacks past 2^31 bytes) for the rowwise and blockwise e4m3 ones; the torch.bmm experts of
Llama-4-Scout in both weight layouts.

The operands are exact (tests/exact_operands.py served(): value windows picked from K so that every sum is exact in
fp32 in any order), so the bf16 output must equal the fp64 reference rounded once, in every element.  At these sizes
a handful of wrong elements in one tile is far below any SQNR bar; here it fails.  What the shapes reach that the toy
cases of test_exact_gemm_gpu.py do not (KT up to 224, 224 n-tiles, 16 to 32 m-blocks, hundreds of (expert, m-block)
pairs, E = 1024) is pinned on the CPU by tests/test_served_shapes_plan.py, which also
asserts the exactness bound of every case here.
"""
import ctypes
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import exact_operands as ex
import grouped_model as gm
from test_exact_gemm_gpu import OP_FORMAT, OPS, _sweep, shape_supported

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, N, K): the Llama-3 projections of bench.py (8B hidden 4096, intermediate 14336, kv 1024; 70B hidden 8192,
# intermediate 28672); q|k|v and gate|up are the fused launches bench.py runs
DENSE_SHAPES = [("8b_qkv", 6144, 4096), ("8b_o", 4096, 4096), ("8b_gate_up", 28672, 4096), ("8b_down", 4096, 14336),
                ("70b_qkv", 10240, 8192), ("70b_down", 8192, 28672)]
TOKENS = (1, 4, 32, 33, 128, 300, 2048)
PRIME_GRID = 127   # a prime CTA count below the SM count: splits no power-of-two tiling lines up with
DENSE_OPS = [(op, 32) for op in OPS if op != "int4"] + [("int4", g) for g in (32, 64, 128, 256)]


def dense_cases():
    return [(op, g, name, N, K) for op, g in DENSE_OPS for name, N, K in DENSE_SHAPES
            if shape_supported(op, max(TOKENS), N, K)]


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


# One 128-feature tile of the 70B down projection (K = 28672, KT = 224) under grids that split it across up to 132
# CTAs: the owner gathers the partials of 32 to 131 contributors, which no whole served projection reaches on 132 SMs
GATHER_SHAPE = ("70b_down_tile", 128, 28672)
GATHER_GRIDS = (33, 34, 65, 100, 132)


@pytest.mark.parametrize("op", OPS)
def test_owner_gathers_of_many_contributors_at_served_k_bit_exact(ops, set_ctas, op):
    name, N, K = GATHER_SHAPE
    case = ex.served(op, max(TOKENS), N, K, group_size=32)
    _sweep(ops, set_ctas, case, list(GATHER_GRIDS), Ms=list(TOKENS))


@pytest.mark.parametrize("op,g,name,N,K", dense_cases(), ids=lambda v: str(v))
def test_dense_served_shape_bit_exact(ops, set_ctas, op, g, name, N, K):
    """Every token count of TOKENS at the default grid (the heuristic that is served), one CTA, and a prime grid."""
    case = ex.served(op, max(TOKENS), N, K, group_size=g)
    _sweep(ops, set_ctas, case, [None, 1, PRIME_GRID], Ms=list(TOKENS))


# ------------------------------------------------------------------------------------------------ MoE expert layers
# (name, E, top-k, N, K)
MOE_SHAPES = [("mixtral_gate_up", 8, 2, 14336, 4096), ("mixtral_down", 8, 2, 4096, 14336),
              ("qwen3_gate_up", 128, 8, 1536, 2048), ("qwen3_down", 128, 8, 2048, 768),
              ("e256", 256, 8, 256, 1024), ("e1024", 1024, 8, 128, 1024)]
# DeepSeek-V3's routed experts (hidden 7168, expert intermediate 2048, 256 experts, top-8) in the formats its
# checkpoints and DESIGN §2a use: e4m3 weight stacks of 7.5 and 3.8 GB, past 2^31 bytes, so every weight and scale
# offset of the grouped kernels needs 64-bit arithmetic
DSV3_SHAPES = [("dsv3_gate_up", 256, 8, 4096, 7168), ("dsv3_down", 256, 8, 7168, 2048)]
DSV3_KINDS = ("fp8", "fp8_blockwise")
MOE_TOKENS = (1, 4, 32, 2048)   # decode batches and one prefill
MOE_TAIL = 3                    # rows past offs[-1]: never written
MOE_KINDS = ("fp8", "nvfp4", "int4", "int8", "int8wo", "fp8wo", "fp8_blockwise", "mxfp8", "mxfp4")
# (K multiple, N multiple) each grouped launcher requires; int4 as bench.py packs it (K % 1024 == 0)
MOE_RULES = {"fp8": (128, 16), "nvfp4": (128, 128), "int4": (1024, 8), "int8": (16, 8), "int8wo": (16, 1),
             "fp8wo": (16, 8), "fp8_blockwise": (128, 128), "mxfp8": (32, 128), "mxfp4": (32, 128)}


def moe_supported(kind, N, K):
    k, n = MOE_RULES[kind]
    return K % k == 0 and N % n == 0


def routing(E, topk, T, seed):
    """Rows per expert of a seeded top-k over skewed logits: expert 0 hot, every fourth expert (but 0) nearly never
    chosen, so some experts are empty at every size."""
    g = torch.Generator().manual_seed(seed)
    skew = torch.zeros(E)
    skew[0] = 3.0
    skew[4::4] = -30.0
    logits = torch.randn(T, E, generator=g) + skew
    idx = logits.topk(topk, dim=1).indices.reshape(-1)
    return torch.bincount(idx, minlength=E).tolist()


def moe_cases():
    return ([(kind, name, E, topk, N, K) for kind in MOE_KINDS for name, E, topk, N, K in MOE_SHAPES
             if moe_supported(kind, N, K)]
            + [(kind, name, E, topk, N, K) for kind in DSV3_KINDS for name, E, topk, N, K in DSV3_SHAPES])


def moe_activations(kind, win, M, K, g):
    """(the activation operands the kind's launcher takes, values(s, t): fp64 of rows s..t-1 as the kernel multiplies
    them, the per-token scales its epilogue applies or None), drawn from the window."""
    if kind == "fp8":
        xq = (ex.randint(-win["xr"], win["xr"], (M, K), g).double() * 2.0**-2).to(torch.float8_e4m3fn)
        rs = ex.pick(win["odd"], (M,), g) * 2.0**-8
        return (xq, rs.float()), lambda s, t: xq[s:t].double(), rs
    if kind == "int8":
        xq = ex.randint(-win["r"], win["r"], (M, K), g).to(torch.int8)
        sx = (ex.pick(ex.ODD, (M, 1), g) * 2.0**-14).float()
        return (xq, sx), lambda s, t: xq[s:t].double(), sx
    if kind == "fp8_blockwise":   # codes with 1x128 token scales, in the layout of ao_fp8_quantize_1x128
        xq = ex.randint(-win["xr"], win["xr"], (M, K), g).to(torch.float8_e4m3fn)
        a_s = ex.pow2(ex.randint(-2, -2 + win["da"], (M, K // 128), g)).float()
        return ((xq, ex.transposed_scales(a_s)), lambda s, t: ex.blockwise_values(xq[s:t].double(), a_s[s:t], 1),
                None)
    rs = None
    if kind == "nvfp4":
        X = ex.randint(-win["xr"], win["xr"], (M, K), g).double() * 0.5
        rs = ex.pick(win["odd"], (M,), g) * 2.0**-6
    elif kind in ("int4", "int8wo", "fp8wo"):
        X = ex.randint(-win["xr"], win["xr"], (M, K), g).double() * 2.0**-3
    elif kind == "mxfp8":   # xhat = code x 2^(e8 - 127), what the fakequant prologue writes
        xb = ex.randint(125, 125 + win["dx"], (M, K // 32), g)
        X = ex.randint(-7, 7, (M, K), g).double() * 2.0**-2 * ex.pow2(xb - 127).repeat_interleave(32, 1)
    else:
        X = ex.mxfp4_value(ex.pick(win["xc"], (M, K), g).long(), 126 + ex.randint(0, win["d"], (M, K // 32), g))
    x = X.to(torch.bfloat16)
    assert torch.equal(x.double(), X), f"premise: {kind} activations exact in bf16"
    del X
    return ((x, rs.float()) if kind == "nvfp4" else (x,)), lambda s, t: x[s:t].double(), rs


def moe_expert(kind, win, N, K, g):
    """One expert's weights: (fp64 values [N, K] as the kernel multiplies them, the packed tensors its stacks hold,
    epi(acc, rs) -> fp64 output of the exact sums acc of rows with per-token scales rs), each epilogue as
    include/ao_b200.h states it."""
    if kind == "fp8":
        W = ex.randint(-win["wr"], win["wr"], (N, K), g).double() * 2.0**-3
        sw = ex.pick(win["odd"], (N,), g) * 2.0**-9
        return W, (W.to(torch.float8_e4m3fn), sw.float()), lambda acc, rs: acc * (rs[:, None] * sw[None, :])
    if kind == "nvfp4":
        wc = ex.randint(0, 15, (N, K), g)
        wb = ex.pick(win["wb"], (N, K // 16), g).to(torch.uint8)
        wp = ex.pick(win["odd"], (1,), g) * 2.0**-4
        W = ex.e2m1_value(wc) * ex.e4m3_bytes_value(wb).repeat_interleave(16, 1)

        def epi(acc, rs):
            acc = acc * rs[:, None]
            ex.fp32_exact(acc, "grouped nvfp4: acc * x_scale")
            return acc * wp
        return W, (ex.pack_e2m1(wc), ex.to_blocked(wb), wp.float()), epi
    if kind == "int4":
        W, qd, sz = ex.int4_weights(N, K, 32, g)
        return W, (qd, sz.transpose(0, 1).contiguous()), lambda acc, rs: acc
    if kind == "int8":
        wq = ex.randint(-win["r"], win["r"], (N, K), g).to(torch.int8)
        sw = (ex.pick(ex.ODD, (N,), g) * 2.0**-10).float()
        return wq.double(), (wq, sw), lambda acc, rs: ex.int8_epilogue(acc, rs, sw)
    if kind == "int8wo":   # scales of 12 significant bits over 13 binades: bf16(scale) rounds
        wq = ex.randint(-128, 127, (N, K), g).to(torch.int8)
        s = (ex.randint(2048, 4095, (N,), g).double() * 2.0**-20 * ex.pow2(ex.randint(-6, 6, (N,), g))).float()
        return wq.double(), (wq, s), lambda acc, rs: ex.recipe(kind, acc, s).double()
    if kind == "fp8wo":    # the weights the kernel multiplies are bf16(e4m3 * scale) = (c / 8) * odd * 2^-8 exactly
        s = (ex.pick([3, 5, 7], (N,), g) * 2.0**-8).float()
        wq = (ex.randint(-win["wr"], win["wr"], (N, K), g).double() * 2.0**-3).to(torch.float8_e4m3fn)
        W = (wq.float() * s[:, None]).to(torch.bfloat16).double()
        return W, (wq, s), lambda acc, rs: ex.recipe(kind, acc).double()
    if kind == "fp8_blockwise":
        Wc = ex.randint(-win["wr"], win["wr"], (N, K), g).double()
        w_s = ex.pow2(ex.randint(-1, -1 + win["dw"], (N // 128, K // 128), g)).float()
        return (ex.blockwise_values(Wc, w_s, 128), (Wc.to(torch.float8_e4m3fn), w_s),
                lambda acc, rs: ex.blockwise_epilogue(acc, None).double())
    if kind == "mxfp8":
        Wc = ex.randint(-7, 7, (N, K), g).double() * 2.0**-3
        wb = ex.randint(124, 124 + win["dw"], (N, K // 32), g)
        W = Wc * ex.pow2(wb - 127).repeat_interleave(32, 1)
        return W, (Wc.to(torch.float8_e4m3fn), ex.to_blocked(wb.to(torch.uint8))), lambda acc, rs: acc
    wc = ex.randint(0, 15, (N, K), g)
    wb = 125 + ex.randint(0, win["d"], (N, K // 32), g)
    return (ex.mxfp4_value(wc, wb), (ex.pack_e2m1(wc), ex.to_blocked(wb.to(torch.uint8))),
            lambda acc, rs: acc)


class MoECase:
    """One grouped GEMM with exact operands at M = sum(rows) + MOE_TAIL rows, launched through the C ABI into a
    poisoned output.  Each expert's weights are drawn, packed into its slot of the preallocated stacks and turned into
    its fp64 reference in turn: no fp64 stack of all experts, and no second copy of the packed stack."""

    def __init__(self, lib, kind, rows, N, K, seed):
        E = len(rows)
        self.offs_list = gm.cumulative(rows)
        M = self.offs_list[-1] + MOE_TAIL
        gx, gw = ex.gen(seed * 7919 + M * 31 + K), ex.gen(seed * 7919 + N * 7 + K + E)
        win = ex.window(MOE_OP[kind], K)
        xs, values, rs = moe_activations(kind, win, M, K, gx)
        ref = torch.empty(self.offs_list[-1], N, dtype=torch.bfloat16, device=ex.DEV)
        stacks = None
        start = 0
        for e, end in enumerate(self.offs_list):
            W, packed, epi = moe_expert(kind, win, N, K, gw)
            if stacks is None:
                stacks = [torch.empty((E,) + p.shape, dtype=p.dtype, device=ex.DEV) for p in packed]
            for s, p in zip(stacks, packed):
                s[e] = p
            if end > start:
                X = values(start, end)
                ex.premise(X, W, chunk=kind == "fp8")
                y = epi(X @ W.t(), rs[start:end] if rs is not None else None)
                ex.fp32_exact(y, f"grouped {kind}: the fp64 reference of expert {e}")
                ref[start:end] = y.float().to(torch.bfloat16)
            del W, packed, epi
            start = end
        self.ref, self.valid = ref, self.offs_list[-1]
        self.offs = torch.tensor(self.offs_list, dtype=torch.int32, device=ex.DEV)
        self.y = torch.full((M, N), ex.POISON_BF16, dtype=torch.int16, device=ex.DEV)
        self.ws = torch.zeros(int(max(lib.ao_b200_workspace_bytes(0, 0), lib.ao_b200_workspace_bytes(M, N))),
                              dtype=torch.uint8, device=ex.DEV)
        self.flags = self.ws[:16384].view(torch.int32)
        mid, tail = ((32,), (N,)) if kind == "int4" else ((), ())   # int4: group size, and N_out = N
        offs, y = self.offs, self.y   # not self: a cycle through the closure would keep the stacks past `del case`
        self.args = lambda: (*xs, M, K, *stacks, *mid, E, N, *tail, offs, y)
        self.lib, self.fn = lib, getattr(lib, ABI[kind][0])
        self.kind, self.M, self.N, self.K, self.E = kind, M, N, K, E

    def launch(self):
        """Poisons y, launches, returns y (the rows past offs[-1] must keep the poison)."""
        self.y.fill_(ex.POISON_BF16)
        conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in self.args()]
        rc = self.fn(*conv, self.ws.data_ptr(), self.ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, self.lib.ao_b200_last_error()
        return self.y

    def first_mismatch(self):
        bad = (self.y[: self.valid] != self.ref.view(torch.int16)).nonzero()
        if bad.numel() == 0:
            bad = (self.y[self.valid:] != ex.POISON_BF16).nonzero()
            return None if bad.numel() == 0 else f"row {self.valid + int(bad[0, 0])} past offs[-1] written"
        m, n = (int(v) for v in bad[0])
        e = next(i for i, end in enumerate(self.offs_list) if end > m)
        got, want = self.y[m, n].view(torch.bfloat16).item(), self.ref[m, n].item()
        return f"first at row {m} (expert {e}, its row {m - (self.offs_list[e - 1] if e else 0)}), column {n}: got {got!r} want {want!r}"


# the dense op with the same exactness bound (the grouped kernels add no bias, so the dense bound is conservative)
MOE_OP = {"fp8": "fp8", "nvfp4": "nvfp4w_rowpts", "int4": "int4", "int8": "int8_dyn", "int8wo": "int8wo",
          "fp8wo": "fp8wo", "fp8_blockwise": "fp8_blockwise", "mxfp8": "mxfp8", "mxfp4": "mxfp4"}
ABI = {"fp8": ("ao_fp8_rowwise_grouped_mm", "ppiippiipppzp"), "nvfp4": ("ao_nvfp4_grouped_mm", "ppiipppiipppzp"),
       "int4": ("ao_int4_tilepacked_grouped_mm", "piippiiiipppzp"), "int8": ("ao_int8_dyn_grouped_mm", "ppiippiipppzp"),
       "int8wo": ("ao_int8_weight_grouped_mm", "piippiipppzp"), "fp8wo": ("ao_fp8_weight_grouped_mm", "piippiipppzp"),
       "fp8_blockwise": ("ao_fp8_blockwise_grouped_mm", "ppiippiipppzp"),
       "mxfp8": ("ao_mxfp8_grouped_mm", "piippiipppzp"), "mxfp4": ("ao_mxfp4_grouped_mm", "piippiipppzp"),
       "bmm": ("ao_fp8_rowwise_bmm", "ppiiippiippzp")}
_CT = {"p": ctypes.c_void_p, "i": ctypes.c_int, "z": ctypes.c_size_t}


@pytest.fixture(scope="module")
def lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    lib.ao_b200_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    for name, sig in ABI.values():
        getattr(lib, name).argtypes = [_CT[c] for c in sig]
    return lib


@pytest.mark.parametrize("kind,name,E,topk,N,K", moe_cases(), ids=lambda v: str(v))
def test_moe_served_shape_bit_exact(ops, set_ctas, lib, kind, name, E, topk, N, K):
    """Decode and prefill routings at the default grid and one CTA, each launch into a poisoned output: the valid rows
    must equal the reference, the MOE_TAIL rows past offs[-1] must keep the poison, and the flag area must be zero."""
    wrong, total = [], 0
    for T in MOE_TOKENS:
        case = MoECase(lib, kind, routing(E, topk, T, seed=T + E), N, K, seed=T)
        runs = []
        for G in (None, 1):
            set_ctas(G or 0)
            y = case.launch()
            runs.append((G, (y[: case.valid] != case.ref.view(torch.int16)).sum(),
                         (y[case.valid:] != ex.POISON_BF16).sum(), case.flags.ne(0).sum()))
        set_ctas(0)
        total += len(runs)
        for G, nb, nt, nr in runs:
            if int(nb) or int(nt) or int(nr):
                set_ctas(G or 0)
                case.launch()
                set_ctas(0)
                torch.cuda.synchronize()
                wrong.append((T, G, int(nb), int(nt), int(nr), case.offs_list, case.M, case.first_mismatch()))
        del case, y   # before the next case is built: the DeepSeek-V3 stacks are 7.5 GB each
    if wrong:
        T, G, nb, nt, nr, offs, M, where = wrong[0]
        p = gm.plan(offs, M, N, K, grid=G, sm=ex.sm_count(), fmt=kind)
        pytest.fail(f"{kind} {name} T={T} (M={M}, J={p.mbp[-1]}) grid={G or 'default'}: {nb} wrong elements, {nt} "
                    f"elements past offs[-1] written, {nr} flags left raised; {where} (U={p.U}, width {p.width}, "
                    f"device grid {p.G} of {p.G_host}); {len(wrong)} of {total} launches wrong")


# ------------------------------------------------------------------------------------------------ torch.bmm experts
# Llama-4-Scout's experts (hidden 5120, intermediate 8192, 16 experts): the fused gate|up [B, 5120, 16384] and the down
# projection [B, 8192, 5120] of torch.bmm, with the weight the transposed view of a stored [B, N, K] tensor ("nk": the
# grouped e4m3 kernel) or stored [B, K, N] ("kn": F8NMajorFmt's 3-D map and on-chip transpose)
BMM_SHAPES = [("scout_gate_up", 16, 5120, 16384), ("scout_down", 16, 8192, 5120)]
BMM_TOKENS = (1, 4, 32, 128)   # tokens per expert
BMM_LAYOUTS = ("nk", "kn")
# 32 experts of the fused gate|up, stored [B, K, N]: 2.7 GB, so the 3-D map spans more than 2^31 bytes
BMM_LARGE = ("kn", "b32_gate_up", 32, 5120, 16384, (1,))


def bmm_cases():
    return [(layout, name, B, K, N, BMM_TOKENS) for layout in BMM_LAYOUTS for name, B, K, N in BMM_SHAPES] + [BMM_LARGE]


class BmmCase:
    """torch.bmm of B experts with exact operands from ex.window("fp8", K), for every token count of Ms: each batch's
    weights are drawn, stored in the layout and turned into the fp64 references of every M in turn."""

    def __init__(self, lib, layout, B, K, N, Ms, seed):
        win = ex.window("fp8", K)
        gw = ex.gen(seed * 7919 + B * 131 + N * 7 + K)
        self.kn = layout == "kn"
        self.wq = torch.empty((B, K, N) if self.kn else (B, N, K), dtype=torch.uint8, device=ex.DEV)
        self.sw = torch.empty(B, N, dtype=torch.float32, device=ex.DEV)
        self.x = {}
        for M in Ms:
            gx = ex.gen(seed * 7919 + B * 131 + M * 31 + K)
            xq = (ex.randint(-win["xr"], win["xr"], (B * M, K), gx).double() * 2.0**-2).to(torch.float8_e4m3fn)
            rs = ex.pick(win["odd"], (B * M,), gx) * 2.0**-8
            self.x[M] = (xq, rs, torch.empty(B * M, N, dtype=torch.bfloat16, device=ex.DEV))
        for b in range(B):
            W = ex.randint(-win["wr"], win["wr"], (N, K), gw).double() * 2.0**-3
            sw = ex.pick(win["odd"], (N,), gw) * 2.0**-9
            wq = W.to(torch.float8_e4m3fn).view(torch.uint8)
            self.wq[b] = wq.t() if self.kn else wq
            self.sw[b] = sw.float()
            del wq
            for M, (xq, rs, ref) in self.x.items():
                X = xq[b * M:(b + 1) * M].double()
                ex.premise(X, W, chunk=True)
                sc = rs[b * M:(b + 1) * M, None] * sw[None, :]
                ex.fp32_exact(sc, "bmm: x_scale * w_scale")
                y = (X @ W.t()) * sc
                ex.fp32_exact(y, f"bmm: the fp64 reference of batch {b}")
                ref[b * M:(b + 1) * M] = y.float().to(torch.bfloat16)
            del W
        self.x = {M: (xq, rs.float(), ref) for M, (xq, rs, ref) in self.x.items()}
        self.ws = torch.zeros(int(lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=ex.DEV)
        self.flags = self.ws[:16384].view(torch.int32)
        self.lib, self.B, self.K, self.N = lib, B, K, N
        self.y = None

    def launch(self, M):
        xq, rs, _ = self.x[M]
        self.y = torch.full((self.B * M, self.N), ex.POISON_BF16, dtype=torch.int16, device=ex.DEV)
        rc = self.lib.ao_fp8_rowwise_bmm(xq.data_ptr(), rs.data_ptr(), self.B, M, self.K, self.wq.data_ptr(),
                                         self.sw.data_ptr(), self.N, int(self.kn), self.y.data_ptr(),
                                         self.ws.data_ptr(), self.ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, self.lib.ao_b200_last_error()
        return self.y

    def first_mismatch(self, M):
        bad = (self.y != self.x[M][2].view(torch.int16)).nonzero()
        if bad.numel() == 0:
            return None
        m, n = (int(v) for v in bad[0])
        got, want = self.y[m, n].view(torch.bfloat16).item(), self.x[M][2][m, n].item()
        return f"first at row {m} (batch {m // M}, its row {m % M}), column {n}: got {got!r} want {want!r}"


@pytest.mark.parametrize("layout,name,B,K,N,Ms", bmm_cases(), ids=[f"{c[0]}-{c[1]}" for c in bmm_cases()])
def test_bmm_served_shape_bit_exact(set_ctas, lib, layout, name, B, K, N, Ms):
    """Every token count per expert at the default grid and one CTA, each launch into a poisoned output: every row
    must equal the reference and the flag area must be zero."""
    case = BmmCase(lib, layout, B, K, N, Ms, seed=B + K)
    wrong, total = [], 0
    for M in Ms:
        runs = []
        for G in (None, 1):
            set_ctas(G or 0)
            y = case.launch(M)
            runs.append((G, (y != case.x[M][2].view(torch.int16)).sum(), case.flags.ne(0).sum()))
        set_ctas(0)
        total += len(runs)
        for G, nb, nr in runs:
            if int(nb) or int(nr):
                set_ctas(G or 0)
                case.launch(M)
                set_ctas(0)
                torch.cuda.synchronize()
                wrong.append((M, G, int(nb), int(nr), case.first_mismatch(M)))
    if wrong:
        M, G, nb, nr, where = wrong[0]
        # F8NMajorFmt runs the grouped schedule and token tiles of the e4m3 kernel
        p = gm.plan([(b + 1) * M for b in range(B)], B * M, N, K, grid=G, sm=ex.sm_count(), fmt="fp8")
        pytest.fail(f"bmm {layout} {name} B={B} M={M} grid={G or 'default'}: {nb} wrong elements, {nr} flags left "
                    f"raised; {where} (J={p.mbp[-1]}, U={p.U}, width {p.width}, device grid {p.G} of {p.G_host}); "
                    f"{len(wrong)} of {total} launches wrong")


# ------------------------------------------------------------------------------------------------ fused projections
# q|k|v and gate|up of Llama-3-8B (hidden 4096) fused by ao_b200.fusion.fuse_parallel_linears; int4's k member has
# 1000 features (not a multiple of 128), so the fused launch's N_out slicing is exercised
FUSED_GROUPS = {"qkv": (("q_proj", 4096), ("k_proj", 1024), ("v_proj", 1024)),
                "gate_up": (("gate_proj", 14336), ("up_proj", 14336))}
HIDDEN = 4096
FUSED_FORMATS = ("int4", "int8", "fp8", "mxfp8", "nvfp4")


def _template(fmt):
    """A weight quantized by the format's config: the attributes (activation kwargs, layouts) the exact weights copy."""
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig, NVFP4WeightOnlyConfig
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Int8DynamicActivationInt8WeightConfig,
                                      PerRow, quantize_)

    cfg = {"int8": Int8DynamicActivationInt8WeightConfig(), "fp8": Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()),
           "mxfp8": MXDynamicActivationMXWeightConfig(), "nvfp4": NVFP4WeightOnlyConfig()}[fmt]
    lin = nn.Linear(HIDDEN, 128, bias=False, device=ex.DEV, dtype=torch.bfloat16)
    quantize_(lin, cfg)
    return lin.weight


def _blocked_like(tmpl_scale, plain_bytes):
    b = ex.to_blocked(plain_bytes).view(tmpl_scale.dtype)
    return b.reshape(-1, tmpl_scale.shape[1]) if tmpl_scale.dim() == 2 else b.reshape(-1)


def _exact_member(fmt, n, g, index):
    """(exact quantized weight [n, HIDDEN], its fp64 values as the kernel multiplies them, epilogue scale per feature
    or None)."""
    from ao_b200.prototype.mx_formats import MXTensor, NVFP4Tensor
    from ao_b200.quantization import Float8Tensor, Int4TilePackedTo4dTensor, Int8Tensor

    K = HIDDEN
    if fmt == "int4":
        W, qd, sz = ex.int4_weights(n, K, 32, g)
        return Int4TilePackedTo4dTensor(qd, sz.transpose(0, 1).contiguous(), [1, 32], torch.Size([n, K])), W, None
    t = _template(fmt)
    if fmt == "int8":
        wq = ex.randint(-32, 32, (n, K), g).to(torch.int8)   # 4096 * 127 * 32 < 2^24 whatever the activation codes
        sw = (ex.pick(ex.ODD, (n, 1), g) * 2.0**-10).to(t.scale.dtype)
        return (Int8Tensor(wq, sw, [1, K], t.dtype, zero_point=torch.zeros_like(wq[:, :1]), act_quant_kwargs=t.act_quant_kwargs,
                           reduce_range=t.reduce_range), wq.double(), sw.double().reshape(-1))
    if fmt == "fp8":
        W = ex.randint(-7, 7, (n, K), g).double() * 2.0**-3
        sw = ex.pick([3, 5, 7], (n, 1), g) * 2.0**-9
        return (Float8Tensor(W.to(torch.float8_e4m3fn), sw.to(t.scale.dtype), [1, K], t.mm_config, t.act_quant_kwargs,
                             t.kernel_preference, t.dtype), W, sw.reshape(-1))
    if fmt == "mxfp8":
        Wc = ex.randint(-7, 7, (n, K), g).double() * 2.0**-3
        wb = ex.randint(124, 126, (n, K // 32), g)
        W = Wc * ex.pow2(wb - 127).repeat_interleave(32, 1)
        return (MXTensor(Wc.to(torch.float8_e4m3fn), _blocked_like(t.scale, wb.to(torch.uint8)), t.elem_dtype, t.block_size,
                         t.orig_dtype, t.kernel_preference, t.act_quant_kwargs, t.is_swizzled_scales), W, None)
    win = ex.window("nvfp4w_rowpts", K)
    wc = ex.randint(0, 15, (n, K), g)
    wb = ex.pick(win["wb"], (n, K // 16), g).to(torch.uint8)
    pts = [3, 5, 7][index] * 2.0**-4   # a different per-tensor scale per member
    W = ex.e2m1_value(wc) * ex.e4m3_bytes_value(wb).repeat_interleave(16, 1)
    w = NVFP4Tensor(ex.pack_e2m1(wc), _blocked_like(t.scale, wb), 16, torch.bfloat16,
                    torch.tensor(pts, dtype=torch.float32, device=ex.DEV), None, True, False, t.act_quant_kwargs)
    return w, W, torch.full((n,), pts, dtype=torch.float64, device=ex.DEV)


def _exact_activations(fmt, M, g):
    """bf16 activations [M, HIDDEN] whose per-token quantization (for the dynamic formats) gives small exact codes."""
    K = HIDDEN
    if fmt == "int4":
        return (ex.randint(-8, 8, (M, K), g).double() * 2.0**-3).to(torch.bfloat16)
    if fmt == "int8":
        return torch.randn(M, K, device=ex.DEV, generator=g).to(torch.bfloat16)   # any codes: int8 sums stay exact
    if fmt == "nvfp4":
        return (ex.randint(-1, 1, (M, K), g).double() * 0.5).to(torch.bfloat16)
    X = ex.randint(-7, 7, (M, K), g).double() * 2.0**-2
    step = K if fmt == "fp8" else 32   # +-7/4 in every row (fp8) or 32-block (mxfp8): scale 2^-8, codes 64 c
    X[:, ::step] = ex.pick([-7.0, 7.0], (M, K // step), g) * 2.0**-2
    return X.to(torch.bfloat16)


def _activation_values(fmt, x2):
    """What the kernel multiplies for the activations x2 [M, K]: (values fp64, per-token scale or None).  For the
    dynamic formats the library's quantizer (the one the handler calls) is run, and its codes are checked to be the
    intended small ones by the premise below."""
    o = ex.ops()
    if fmt in ("int4", "nvfp4"):
        return x2.double(), None
    if fmt == "int8":
        q, s = o.int8_quantize_rowwise(x2)
        return q.double(), s.double().reshape(-1)
    if fmt == "fp8":
        q, s = o.fp8_quantize_rowwise(x2)
        return q.double(), s.double().reshape(-1)
    q, s = o.mxfp8_quantize(x2, False)
    return q.double() * ex.pow2(s.view(torch.uint8).long()[:, : x2.shape[1] // 32] - 127).repeat_interleave(32, 1), None


def _reference(fmt, Xv, xs, W, ws, bias):
    """fp64 output of one member, rounded as the kernel's epilogue rounds (bf16)."""
    ex.premise(Xv, W, chunk=fmt == "fp8")
    acc = Xv @ W.t()
    if fmt == "int8":
        t = (acc.float() * xs.float()[:, None]).to(torch.bfloat16).float()
        ex.fp32_exact(t.double() * ws[None, :], "int8: bf16(acc * x_scale) * w_scale")
        return (t * ws.float()[None, :] + bias.float()).to(torch.bfloat16)
    if fmt == "fp8":
        acc = acc * (xs[:, None] * ws[None, :])
    elif ws is not None:
        acc = acc * ws[None, :]
    y = acc + bias.double()
    ex.fp32_exact(y, f"fused {fmt}: the fp64 reference")
    return y.float().to(torch.bfloat16)


@torch.no_grad()
@pytest.mark.parametrize("fmt", FUSED_FORMATS)
def test_fused_projections_equal_separate_and_reference_bit_exact(fmt):
    """Each member of a fused q|k|v and gate|up launch must equal its separate F.linear and the fp64 reference, bit
    for bit, through 3-D inputs [B, S, K] and with bias (no SQNR allowance: the operands make every sum exact)."""
    from ao_b200.fusion import FusedLinearMember, fuse_parallel_linears

    g = ex.gen(50 + FUSED_FORMATS.index(fmt))
    model = nn.Module()
    members = {}
    for group in FUSED_GROUPS.values():
        for i, (name, n) in enumerate(group):
            n = 1000 if fmt == "int4" and name == "k_proj" else n
            w, W, ws = _exact_member(fmt, n, g, i)
            lin = nn.Linear(HIDDEN, n, bias=True, device="meta")
            lin.weight = nn.Parameter(w, requires_grad=False)
            lin.bias = nn.Parameter(torch.zeros(n, dtype=torch.bfloat16, device=ex.DEV), requires_grad=False)
            setattr(model, name, lin)
            members[name] = (W, ws, w)   # w: the separate weight (fusion copies it into the group's storage)
    for B, S in ((1, 1), (2, 16)):
        x = _exact_activations(fmt, B * S, g)
        Xv, xs = _activation_values(fmt, x)
        if fmt in ("fp8", "mxfp8"):   # the quantizer must give the intended codes: 64 c at scale 2^-8
            assert torch.equal(Xv * (xs[:, None] if xs is not None else 1.0), x.double()), f"premise: {fmt} codes"
            assert xs is None or bool((xs == 2.0**-8).all()), f"premise: {fmt} activation scales"
        refs = {}
        for name, (W, ws, _) in members.items():
            lin = getattr(model, name) if not isinstance(getattr(model, name), FusedLinearMember) else None
            probe = _reference(fmt, Xv, xs, W, ws, torch.zeros(W.shape[0], dtype=torch.bfloat16, device=ex.DEV))
            q = ex.lowbit(probe.double()) if fmt != "int8" else 2.0**-8
            bias = (ex.randint(-127, 127, (W.shape[0],), g).double() * q * (16 if fmt != "int8" else 1)).to(torch.bfloat16)
            if lin is not None:
                lin.bias.copy_(bias)
            else:
                getattr(model, name).bias.copy_(bias)   # writes through to the fused storage
            refs[name] = _reference(fmt, Xv, xs, W, ws, bias).reshape(B, S, -1)
        x3 = x.reshape(B, S, HIDDEN)
        if (B, S) == (1, 1):
            sep = {name: getattr(model, name)(x3) for name in members}
            assert fuse_parallel_linears(model) == 2, f"{fmt}: the groups did not fuse"
        else:
            sep = {name: F.linear(x3, members[name][2], getattr(model, name).bias) for name in members}
        outs = {name: getattr(model, name)(x3) for name in members}
        for name in members:
            assert isinstance(getattr(model, name), FusedLinearMember)
            r = refs[name].view(torch.int16)
            assert torch.equal(sep[name].view(torch.int16), r), f"{fmt} {name} [{B}, {S}]: separate F.linear vs reference"
            assert torch.equal(outs[name].view(torch.int16), r), f"{fmt} {name} [{B}, {S}]: fused member vs reference"


# ------------------------------------------------------------------------------------------------ one decode layer
SEVEN = [("q", 4096, 4096), ("k", 1024, 4096), ("v", 1024, 4096), ("o", 4096, 4096), ("gate", 14336, 4096),
         ("up", 14336, 4096), ("down", 4096, 14336)]
LAYER = {"int4": [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336)],
         "fp8": SEVEN, "int8_dyn": SEVEN, "int8wo": SEVEN, "fp8_sparse": SEVEN}


@torch.no_grad()
@pytest.mark.parametrize("op", ["int4", "fp8", "int8_dyn", "int8wo", "fp8_sparse"])
@pytest.mark.parametrize("M", [1, 32])
def test_decode_layer_back_to_back_bit_exact(ops, op, M):
    """The projections of one Llama-3-8B layer launched back to back with PDL (int4 g = 32 with q|k|v and gate|up
    fused, as bench.py runs them; the others as seven launches; int4, int8_dyn, int8wo and fp8_sparse fit two decode
    CTAs per SM, so each GEMM's CTAs share SMs with the next one's), each on its own exact input so that every output
    has a reference: eagerly, then as a CUDA graph replayed twice on new exact inputs copied into the captured buffers.
    A wrong value that the overlapped and the serialized run would share fails here."""
    cases = [ex.served(op, M, N, K, seed=i) for i, (_, N, K) in enumerate(LAYER[op])]
    outs = [c.run() for c in cases]   # no synchronisation between the launches
    torch.cuda.synchronize()
    for (name, _, _), c, y in zip(LAYER[op], cases, outs):
        assert torch.equal(c.bits(y), c.bits(c.ref())), f"eager {name}: {ex.first_mismatch(c, y)}"
    flags = ops.debug_workspace(cases[0].ref_full).view(torch.int32)[:4096]
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for c in cases:   # warm-up on the capture stream: creates its workspace outside the capture
            c.run()
        flags = ops.debug_workspace(cases[0].ref_full).view(torch.int32)[:4096]
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        outs = [c.run() for c in cases]
    for replay in (1, 2):
        fresh = [ex.served(op, M, N, K, seed=i, x_seed=replay) for i, (_, N, K) in enumerate(LAYER[op])]
        for c, f, y in zip(cases, fresh, outs):
            for a, b in zip(c.inputs, f.inputs):
                a.copy_(b)
            c.scrub(y)
        graph.replay()
        torch.cuda.synchronize()
        for (name, _, _), f, y in zip(LAYER[op], fresh, outs):
            assert torch.equal(f.bits(y), f.bits(f.ref())), f"replay {replay} {name}: {ex.first_mismatch(f, y)}"
        assert not bool(flags.ne(0).any()), f"replay {replay}: flags left raised"
        del fresh
