"""Every producer -> consumer handoff between this library's kernels, overlapped by PDL, checked bit for bit against the
same launches run one at a time.

Each kernel here lets the next one on the stream start early (programmatic dependent launch) and waits for its
predecessor before it reads what that predecessor wrote; the dense GEMMs request their first weight tiles before that
wait.  A handoff that breaks the rule only goes wrong while the consumer really runs ahead, which small back-to-back
launches rarely do.  So every chain here starts behind a STALL HEAD: fp8_quantize_rowwise on an unrelated
[8, 2^25] tensor, one CTA per row on 8 SMs, milliseconds long, which triggers its dependents at entry.  Behind it
every kernel of the chain becomes resident, triggers and parks in griddepcontrol.wait, so each consumer's pre-wait
reads happen before its producers have written anything, as far as the chain fits on the SMs the head leaves free
(test_stall_head_opens_the_window checks under torch.profiler, on a CUDA graph replay, that the consumers start before
the head ends).

The kernels are deterministic (stream-K adds partials in a fixed order), so the oracle is the same launches on the same
inputs with torch.cuda.synchronize() between them.  Every buffer a chain writes is filled with 0xFF bytes (NaN in bf16,
f32, e4m3 and e8m0) before either run, so a read that came too early shows up as a NaN or a wrong byte rather than as a
value left over from the other run.  The chains call the C ABI through ctypes on the current stream with their own
workspaces, and launch nothing else between their calls.  Each chain runs once eagerly and once as a CUDA graph
replayed on new inputs copied into its static buffers.
"""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
FENCE = "ao_b200_pdl_fence"

# p: pointer (tensor or None), i: int, f: float, z: size_t
SIGS = {
    FENCE: "p",
    "ao_int8_quantize_rowwise": "piippp", "ao_fp8_quantize_rowwise": "piippp", "ao_fp8_fakequant_rowwise": "piippp",
    "ao_fp8_quantize_rowwise_ld": "piiippp",
    "ao_rmsnorm_quantize_rowwise": "pipfiiippp", "ao_silu_mul_quantize_rowwise": "pipiiiippp",
    "ao_mxfp8_quantize": "piippip", "ao_nvfp4_quantize": "piipppip",
    "ao_int8_dyn_linear": "ppiippipppzp", "ao_int8_mm_i32": "piipippzp", "ao_fp8_rowwise_linear": "ppiippipppzp",
    "ao_mxfp8_linear": "ppiippipppzp", "ao_nvfp4_linear": "pppiipppipppzp",
    "ao_nvfp4_weight_linear_ex": "pipiipppiipppzp",
    "ao_int4_pack_tile4d": "ppiiip", "ao_int4_hqq_quantize": "piiippppzp",
    "ao_int4_tilepacked_linear_strided": "piiippiippipzip",
    "ao_fp8_rowwise_grouped_mm": "ppiippiipppzp", "ao_nvfp4_fakequant_grouped": "piiipipppp",
    "ao_nvfp4_grouped_mm": "ppiipppiipppzp",
}
_CT = {"p": ctypes.c_void_p, "i": ctypes.c_int, "f": ctypes.c_float, "z": ctypes.c_size_t}


@pytest.fixture(scope="module")
def lib():
    import ao_b200  # noqa: F401

    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_b200_last_error.restype = ctypes.c_char_p
    lib.ao_b200_workspace_bytes.restype = ctypes.c_size_t
    lib.ao_int4_hqq_workspace_bytes.restype = ctypes.c_size_t
    for name, sig in SIGS.items():
        getattr(lib, name).argtypes = [_CT[c] for c in sig]
    return lib


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Chain:
    """A sequence of library calls on explicit buffers.  in_(t): an input (kept); out(shape, dtype): a buffer the chain
    writes (poisoned before every run); call(name, *args): one C-ABI call (tensors become their device pointers, the
    stream is appended); torch(fn): a torch launch in the chain."""

    def __init__(self, lib, name):
        self.lib, self.name = lib, name
        self.inputs, self.outs, self.steps = [], [], []
        self.finite = []   # float outputs that must be finite when the chain is right

    def in_(self, t):
        t = t.contiguous()
        self.inputs.append(t)
        return t

    def out(self, shape, dtype, finite=False):
        t = torch.empty(shape, dtype=dtype, device=DEV)
        if finite:
            self.finite.append(len(self.outs))
        self.outs.append(t)
        return t

    def workspace(self, nbytes=None):
        return torch.zeros(int(nbytes or self.lib.ao_b200_workspace_bytes(0, 0)), dtype=torch.uint8, device=DEV)

    def call(self, name, *args):
        self.steps.append((name, args))

    def fence(self):
        self.steps.append((FENCE, ()))

    def torch(self, fn):
        self.steps.append((fn, ()))

    def poison(self):
        for t in self.outs:
            t.view(torch.uint8).fill_(0xFF)

    def launch(self, name, args):
        if callable(name):
            name()
            return
        st = torch.cuda.current_stream().cuda_stream
        conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
        rc = getattr(self.lib, name)(*conv, st)
        assert rc == 0, f"{self.name}: {name}: {self.lib.ao_b200_last_error()}"

    def run(self, head=None, sync_each=False, steps=None):
        if head is not None:
            head()
        for name, args in (self.steps if steps is None else steps):
            self.launch(name, args)
            if sync_each:
                torch.cuda.synchronize()


class Head:
    """The stall head: fp8_quantize_rowwise on [8, 2^25] bf16 rows, one CTA per row (K > 16384) on 8 SMs.  A row of
    2^18 takes one CTA about 126 us (H100 80GB HBM3), shorter than the host needs to launch a chain through ctypes;
    rows 128 times longer keep the window open for milliseconds."""

    M, K = 8, 1 << 25

    def __init__(self, lib):
        self.lib = lib
        g = torch.Generator(device=DEV).manual_seed(99)
        self.x = torch.randn(self.M, self.K, device=DEV, generator=g).to(torch.bfloat16)
        self.q = torch.empty(self.M, self.K, dtype=torch.uint8, device=DEV)
        self.s = torch.empty(self.M, dtype=torch.float32, device=DEV)

    def __call__(self):
        st = torch.cuda.current_stream().cuda_stream
        assert self.lib.ao_fp8_quantize_rowwise(self.x.data_ptr(), self.M, self.K, self.q.data_ptr(), self.s.data_ptr(), st) == 0


@pytest.fixture(scope="module")
def head(lib):
    return Head(lib)


# ---------------------------------------------------------------------------------------------------- operands
def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _bf16(shape, g, scale=1.0):
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


def _blocked_bytes(rows, cols_of_scales):
    return (-(-rows // 128) * 32, -(-cols_of_scales // 4) * 16)


def _rand_int4(N, K, g):
    qd = torch.randint(-2**31, 2**31 - 1, (N // 8, K // 128, 32, 4), device=DEV, dtype=torch.int32, generator=g)
    sz = ((torch.rand(K // 32, N, 2, device=DEV, generator=g) - 0.5) * 0.02).to(torch.bfloat16)
    return qd, sz


def _rand_nvfp4(N, K, g):
    wq = torch.randint(0, 256, (N, K // 2), device=DEV, dtype=torch.uint8, generator=g)
    ws = torch.randint(0x28, 0x30, _blocked_bytes(N, K // 16), device=DEV, dtype=torch.uint8, generator=g)
    return wq, ws


def _pts(t):
    return (t.float().abs().amax() / (448.0 * 6.0)).reshape(1)


# ---------------------------------------------------------------------------------------------------- chains
# Each builder returns a Chain; `x` and the weights are inputs, everything the library writes is an output.

def weight_chain(lib, fmt, via_act, M=32, N=256, K=4096):
    """A weight quantized by this library, then the linear that reads it as weights (directly, or with the activation
    quantizer between them).  The GEMM requests its first weight stages before it waits, so the fence is what orders
    the two."""
    c = Chain(lib, f"{fmt} weight -> {'act quant -> ' if via_act else ''}linear M={M}")
    g = _g(len(fmt) * 10 + via_act + M)
    w, x = c.in_(_bf16((N, K), g, 0.05)), c.in_(_bf16((M, K), g))
    ws = c.workspace()
    y = c.out((M, N), torch.bfloat16, finite=True)
    if fmt in ("int8", "fp8"):
        dt = torch.int8 if fmt == "int8" else torch.uint8
        quant = f"ao_{fmt}_quantize_rowwise"
        wq, wsc = c.out((N, K), dt), c.out((N,), torch.float32)
        if via_act:
            xq, xs = c.out((M, K), dt), c.out((M,), torch.float32)
        else:   # activations quantized before the chain
            xq, xs = c.in_(torch.zeros(M, K, dtype=dt, device=DEV)), c.in_(torch.zeros(M, dtype=torch.float32, device=DEV))
            c.launch(quant, (x, M, K, xq, xs))
            torch.cuda.synchronize()
        c.call(quant, w, N, K, wq, wsc)
        c.fence()
        if via_act:
            c.call(quant, x, M, K, xq, xs)
        lin = "ao_int8_dyn_linear" if fmt == "int8" else "ao_fp8_rowwise_linear"
        c.call(lin, xq, xs, M, K, wq, wsc, N, None, y, ws, ws.numel())
        if fmt == "int8":
            acc = c.out((M, N), torch.int32)
            c.call("ao_int8_mm_i32", xq, M, K, wq, N, acc, ws, ws.numel())
        return c
    if fmt == "mxfp8":
        wq, wsc = c.out((N, K), torch.uint8), c.out(_blocked_bytes(N, K // 32), torch.uint8)
        if via_act:
            xq, xs = c.out((M, K), torch.uint8), c.out(_blocked_bytes(M, K // 32), torch.uint8)
        else:
            xq = c.in_(torch.zeros(M, K, dtype=torch.uint8, device=DEV))
            xs = c.in_(torch.zeros(_blocked_bytes(M, K // 32), dtype=torch.uint8, device=DEV))
            c.launch("ao_mxfp8_quantize", (x, M, K, xq, xs, 1))
            torch.cuda.synchronize()
        c.call("ao_mxfp8_quantize", w, N, K, wq, wsc, 1)
        c.fence()
        if via_act:
            c.call("ao_mxfp8_quantize", x, M, K, xq, xs, 1)
        c.call("ao_mxfp8_linear", xq, xs, M, K, wq, wsc, N, None, y, ws, ws.numel())
        return c
    assert fmt in ("nvfp4", "nvfp4w")
    w_pts, a_pts = c.in_(_pts(w)), c.in_(_pts(x))
    wq, wsc = c.out((N, K // 2), torch.uint8), c.out(_blocked_bytes(N, K // 16), torch.uint8)
    c.call("ao_nvfp4_quantize", w, N, K, w_pts, wq, wsc, 1)
    c.fence()
    if fmt == "nvfp4":
        xq, xs = c.out((M, K // 2), torch.uint8), c.out(_blocked_bytes(M, K // 16), torch.uint8)
        if via_act:
            c.call("ao_nvfp4_quantize", x, M, K, a_pts, xq, xs, 1)
        else:   # the activation quantizer runs before the weight's: its output is complete when the chain's GEMM waits
            c.steps.insert(0, ("ao_nvfp4_quantize", (x, M, K, a_pts, xq, xs, 1)))
        c.call("ao_nvfp4_linear", xq, xs, a_pts, M, K, wq, wsc, w_pts, N, None, y, ws, ws.numel())
    else:
        if via_act:
            xh, xs = c.out((M, K), torch.bfloat16), c.out((M,), torch.float32)
            c.call("ao_fp8_fakequant_rowwise", x, M, K, xh, xs)
            c.call("ao_nvfp4_weight_linear_ex", xh, K, xs, M, K, wq, wsc, w_pts, 0, N, None, y, ws, ws.numel())
        else:
            c.call("ao_nvfp4_weight_linear_ex", x, K, None, M, K, wq, wsc, w_pts, 0, N, None, y, ws, ws.numel())
    return c


def act_chain(lib, kind, M, N=256):
    """An activation quantizer (or a fused RMSNorm / SiLU-mul one), then the GEMMs that read its output."""
    K = {"reg": 4096, "cta": 16400}.get(kind, 4096)
    c = Chain(lib, f"{kind} activations -> linears M={M} K={K}")
    g = _g(7 + M + K)
    x = c.in_(_bf16((M, K), g))
    ws = c.workspace()
    if kind in ("reg", "cta", "rmsnorm", "silu"):
        for fmt in ("int8", "fp8"):
            dt = torch.int8 if fmt == "int8" else torch.uint8
            wq = c.in_(torch.randint(-100, 100, (N, K), device=DEV, generator=g).to(torch.int8)) if fmt == "int8" else \
                c.in_(_bf16((N, K), g).to(torch.float8_e4m3fn).view(torch.uint8))
            wsc = c.in_(torch.rand(N, device=DEV, generator=g) * 1e-3)
            xq, xs = c.out((M, K), dt), c.out((M,), torch.float32)
            if kind in ("reg", "cta"):
                c.call(f"ao_{fmt}_quantize_rowwise", x, M, K, xq, xs)
            elif kind == "rmsnorm":
                c.call("ao_rmsnorm_quantize_rowwise", x, K, c.in_(_bf16((K,), g)), 1e-5, M, K, int(fmt == "fp8"), xq, xs)
            else:
                c.call("ao_silu_mul_quantize_rowwise", x, K, c.in_(_bf16((M, K), g)), K, M, K, int(fmt == "fp8"), xq, xs)
            y = c.out((M, N), torch.bfloat16, finite=True)
            lin = "ao_int8_dyn_linear" if fmt == "int8" else "ao_fp8_rowwise_linear"
            c.call(lin, xq, xs, M, K, wq, wsc, N, None, y, ws, ws.numel())
            if fmt == "int8":
                c.call("ao_int8_mm_i32", xq, M, K, wq, N, c.out((M, N), torch.int32), ws, ws.numel())
        return c
    if kind == "fakequant":
        wq, wsc = _rand_nvfp4(N, K, g)
        xh, xs = c.out((M, K), torch.bfloat16), c.out((M,), torch.float32)
        c.call("ao_fp8_fakequant_rowwise", x, M, K, xh, xs)
        c.call("ao_nvfp4_weight_linear_ex", xh, K, xs, M, K, c.in_(wq), c.in_(wsc), c.in_(torch.tensor([0.5], device=DEV)),
               0, N, None, c.out((M, N), torch.bfloat16, finite=True), ws, ws.numel())
        return c
    # block-scaled activations through a workspace that holds 37 rows of the bf16 slab: several dequant -> GEMM rounds
    act_off = (64 * 1024 + _sm_count() * 128 * 128 * 4 + (1 << 20) - 1) & ~((1 << 20) - 1)
    ws = c.workspace(act_off + 37 * K * 2)
    if kind == "mxfp8":
        wq = c.in_(_bf16((N, K), g).to(torch.float8_e4m3fn).view(torch.uint8))
        wsc = c.in_(torch.randint(120, 130, _blocked_bytes(N, K // 32), device=DEV, dtype=torch.uint8, generator=g))
        xq, xs = c.out((M, K), torch.uint8), c.out(_blocked_bytes(M, K // 32), torch.uint8)
        c.call("ao_mxfp8_quantize", x, M, K, xq, xs, 1)
        c.call("ao_mxfp8_linear", xq, xs, M, K, wq, wsc, N, None, c.out((M, N), torch.bfloat16, finite=True), ws, ws.numel())
        return c
    assert kind == "nvfp4"
    wq, wsc = _rand_nvfp4(N, K, g)
    a_pts = c.in_(_pts(x))
    xq, xs = c.out((M, K // 2), torch.uint8), c.out(_blocked_bytes(M, K // 16), torch.uint8)
    c.call("ao_nvfp4_quantize", x, M, K, a_pts, xq, xs, 1)
    c.call("ao_nvfp4_linear", xq, xs, a_pts, M, K, c.in_(wq), c.in_(wsc), c.in_(torch.tensor([0.5], device=DEV)), N, None,
           c.out((M, N), torch.bfloat16, finite=True), ws, ws.numel())
    return c


def gemm_out_chain(lib, M):
    """GEMM outputs read by the next kernel: column slices of a fused q|k|v (int4) and gate|up (nvfp4 weight-only)
    output feed the next GEMM and the next quantizer without a copy."""
    c = Chain(lib, f"gemm output -> next kernel M={M}")
    g = _g(11 + M)
    D = 1024
    x = c.in_(_bf16((M, D), g))
    ws = c.workspace()
    qkv_q, qkv_sz = (c.in_(t) for t in _rand_int4(3 * D, D, g))
    qkv = c.out((M, 3 * D), torch.bfloat16, finite=True)
    c.call("ao_int4_tilepacked_linear_strided", x, D, M, D, qkv_q, qkv_sz, 32, 3 * D, None, qkv, 3 * D, ws, ws.numel(), 1)
    o_q, o_sz = (c.in_(t) for t in _rand_int4(256, D, g))
    k_slice = qkv[:, D:]   # a column slice: row pitch 3D
    c.call("ao_int4_tilepacked_linear_strided", k_slice, 3 * D, M, D, o_q, o_sz, 32, 256, None,
           c.out((M, 256), torch.bfloat16, finite=True), 256, ws, ws.numel(), 1)
    vq, vs = c.out((M, D), torch.uint8), c.out((M,), torch.float32)
    c.call("ao_fp8_quantize_rowwise_ld", qkv[:, 2 * D:], 3 * D, M, D, vq, vs)
    c.call("ao_fp8_rowwise_linear", vq, vs, M, D, c.in_(_bf16((256, D), g, 0.1).to(torch.float8_e4m3fn).view(torch.uint8)),
           c.in_(torch.rand(256, device=DEV, generator=g)), 256, None, c.out((M, 256), torch.bfloat16, finite=True), ws, ws.numel())
    gu_q, gu_s = (c.in_(t) for t in _rand_nvfp4(2 * D, D, g))
    gu = c.out((M, 2 * D), torch.bfloat16, finite=True)
    pts = c.in_(torch.tensor([0.25], device=DEV))
    c.call("ao_nvfp4_weight_linear_ex", x, D, None, M, D, gu_q, gu_s, pts, 0, 2 * D, None, gu, ws, ws.numel())
    d_q, d_s = (c.in_(t) for t in _rand_nvfp4(256, D, g))
    c.call("ao_nvfp4_weight_linear_ex", gu[:, D:], 2 * D, None, M, D, d_q, d_s, pts, 0, 256, None,
           c.out((M, 256), torch.bfloat16, finite=True), ws, ws.numel())
    return c


def grouped_chain(lib, fmt, quantize_weights, M=300, E=4, N=256, K=1024):
    """Routed rows: offs from a torch cumsum, the grouped activation prologue, and (quantize_weights) the 3-D expert
    weights quantized in the chain.  The grouped GEMMs read no weight before their wait, so no fence is needed."""
    c = Chain(lib, f"grouped {fmt}{' + 3-D weight quant' if quantize_weights else ''}")
    g = _g(13 + quantize_weights)
    x = c.in_(_bf16((M, K), g))
    counts = c.in_(torch.tensor([100, 0, 150, 50], dtype=torch.int32, device=DEV))
    ws = c.workspace()
    offs = c.out((E,), torch.int32)
    c.torch(lambda: torch.cumsum(counts, 0, dtype=torch.int32, out=offs))
    w = c.in_(_bf16((E * N, K), g, 0.05))
    y = c.out((M, N), torch.bfloat16, finite=True)
    if fmt == "fp8":
        if quantize_weights:
            wq, wsc = c.out((E * N, K), torch.uint8), c.out((E * N,), torch.float32)
            c.call("ao_fp8_quantize_rowwise", w, E * N, K, wq, wsc)
        else:
            wq = c.in_(w.to(torch.float8_e4m3fn).view(torch.uint8))
            wsc = c.in_(torch.rand(E * N, device=DEV, generator=g))
        xq, xs = c.out((M, K), torch.uint8), c.out((M,), torch.float32)
        c.call("ao_fp8_quantize_rowwise", x, M, K, xq, xs)
        c.call("ao_fp8_rowwise_grouped_mm", xq, xs, M, K, wq, wsc, E, N, offs, y, ws, ws.numel())
        return c
    per = (N // 128) * 32 * (K // 64) * 16   # one expert's blocked scale bytes
    w_pts = c.in_(torch.stack([_pts(w[e * N:(e + 1) * N]) for e in range(E)]).reshape(E))
    if quantize_weights:
        wq, wsc = c.out((E * N, K // 2), torch.uint8), c.out((E * per,), torch.uint8)
        for e in range(E):
            c.call("ao_nvfp4_quantize", w[e * N:(e + 1) * N], N, K, w_pts[e:e + 1], wq[e * N:(e + 1) * N],
                   wsc[e * per:(e + 1) * per], 1)
    else:
        q, s = _rand_nvfp4(E * N, K, g)
        wq, wsc = c.in_(q), c.in_(s)
    xh, xs, amax = c.out((M, K), torch.bfloat16), c.out((M,), torch.float32), c.out((M,), torch.float32)
    c.call("ao_nvfp4_fakequant_grouped", x, K, M, K, offs, E, xh, xs, amax)
    c.call("ao_nvfp4_grouped_mm", xh, xs, M, K, wq, wsc, w_pts, E, N, offs, y, ws, ws.numel())
    return c


def int4_weight_chain(lib, M=32, N=256, K=2048):
    """int4 weights written in the chain: the packer, the HQQ solver (neither launched with PDL) and torch copy_ / cat
    into the packed weights, each read by the int4 linear."""
    c = Chain(lib, "int4 weights written in the chain")
    g = _g(17)
    x = c.in_(_bf16((M, K), g))
    ws = c.workspace()
    q_u8 = c.in_(torch.randint(0, 256, (N, K // 2), device=DEV, dtype=torch.uint8, generator=g))
    _, sz = _rand_int4(N, K, g)
    sz = c.in_(sz)
    qd = c.out((N // 8, K // 128, 32, 4), torch.int32)
    c.call("ao_int4_pack_tile4d", q_u8, qd, N, K, 8)
    c.call("ao_int4_tilepacked_linear_strided", x, K, M, K, qd, sz, 32, N, None, c.out((M, N), torch.bfloat16, finite=True),
           N, ws, ws.numel(), 1)
    # HQQ codes, packed and with scale_and_zero assembled by torch ops, then the linear
    w = c.in_(_bf16((N, K), g, 0.05))
    hq, hs, hz = c.out((N, K), torch.uint8), c.out((N, K // 32), torch.bfloat16), c.out((N, K // 32), torch.bfloat16)
    hws = c.workspace(lib.ao_int4_hqq_workspace_bytes(N, K, 32))
    c.call("ao_int4_hqq_quantize", w, N, K, 32, hq, hs, hz, hws, hws.numel())
    hu8, hqd, hsz = c.out((N, K // 2), torch.uint8), c.out((N // 8, K // 128, 32, 4), torch.int32), c.out((K // 32, N, 2), torch.bfloat16)
    c.torch(lambda: torch.bitwise_or(hq[:, 0::2] << 4, hq[:, 1::2], out=hu8))
    c.torch(lambda: hsz.copy_(torch.stack([hs, hz], -1).transpose(0, 1)))
    c.call("ao_int4_pack_tile4d", hu8, hqd, N, K, 8)
    c.call("ao_int4_tilepacked_linear_strided", x, K, M, K, hqd, hsz, 32, N, None, c.out((M, N), torch.bfloat16, finite=True),
           N, ws, ws.numel(), 1)
    # torch copy_ / cat into packed weights (a loader), then the linear
    src_a, src_b = (c.in_(t) for t in _rand_int4(N, K, g)[0].split(N // 16))
    cq = c.out((N // 8, K // 128, 32, 4), torch.int32)
    c.torch(lambda: cq[: N // 16].copy_(src_a))
    c.torch(lambda: torch.cat([src_b[:8], src_b[8:]], out=cq[N // 16:]))
    c.call("ao_int4_tilepacked_linear_strided", x, K, M, K, cq, sz, 32, N, None, c.out((M, N), torch.bfloat16, finite=True),
           N, ws, ws.numel(), 1)
    return c


CHAINS = (
    [(f"weight-{fmt}-{'act' if via else 'direct'}", (lambda lib, f=fmt, v=via: weight_chain(lib, f, v)))
     for fmt in ("int8", "fp8", "mxfp8", "nvfp4", "nvfp4w") for via in (False, True)]
    + [(f"act-{kind}-M{M}", (lambda lib, k=kind, m=M: act_chain(lib, k, m)))
       for kind in ("reg", "cta", "rmsnorm", "silu", "fakequant", "mxfp8", "nvfp4") for M in (1, 300)]
    + [(f"gemm-out-M{M}", (lambda lib, m=M: gemm_out_chain(lib, m))) for M in (1, 16, 32, 300)]
    + [(f"grouped-{fmt}-{'wquant' if qw else 'static'}", (lambda lib, f=fmt, q=qw: grouped_chain(lib, f, q)))
       for fmt in ("fp8", "nvfp4") for qw in (False, True)]
    + [("int4-weights", int4_weight_chain)]
)


def _snapshot(c):
    torch.cuda.synchronize()
    return [t.clone() for t in c.outs]


def _check(c, got, want, mode):
    for i, (a, b) in enumerate(zip(got, want)):
        ab, bb = a.view(torch.uint8).reshape(-1), b.view(torch.uint8).reshape(-1)
        if not torch.equal(ab, bb):
            bad = (ab != bb).nonzero().flatten()
            j = int(bad[0])
            pytest.fail(f"{c.name} [{mode}]: output {i} {tuple(a.shape)} {a.dtype}: {bad.numel()} bytes differ from the "
                        f"serialized run, first at byte {j}: {int(ab[j]):#04x} vs {int(bb[j]):#04x}")


def _serialized(c):
    c.poison()
    torch.cuda.synchronize()
    c.run(sync_each=True)
    want = _snapshot(c)
    for i in c.finite:   # the serialized run wrote every output (no poison NaN left)
        assert bool(torch.isfinite(want[i].float()).all()), f"{c.name}: serialized output {i} not finite"
    return want


def _new_inputs(c, seed):
    g = _g(seed)
    for t in c.inputs:
        if t.dtype in (torch.bfloat16, torch.float32) and t.numel() > 4:   # data, not scalars, counts or scales
            t.copy_((torch.randn(t.shape, device=DEV, generator=g) * t.float().std()).to(t.dtype))


@pytest.mark.parametrize("name,make", CHAINS, ids=[n for n, _ in CHAINS])
def test_overlapped_equals_serialized(lib, head, name, make):
    c = make(lib)
    want = _serialized(c)
    c.poison()
    torch.cuda.synchronize()
    c.run(head=head)
    _check(c, _snapshot(c), want, "eager")

    # the same chain captured behind the head in a CUDA graph, replayed on new inputs
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        c.run(head=head)
    torch.cuda.synchronize()
    _new_inputs(c, 1234)
    torch.cuda.synchronize()
    want = _serialized(c)
    c.poison()
    torch.cuda.synchronize()
    graph.replay()
    _check(c, _snapshot(c), want, "graph replay")


def _kernel_spans(fn):
    """(name, start_us, end_us) of every CUDA kernel fn launches, in start order (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    spans = [(e.name, e.time_range.start, e.time_range.end) for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
             and "memset" not in e.name.lower()]
    return sorted(spans, key=lambda s: s[1])


# Chains whose every kernel fits on the SMs the head leaves free.  In the others a later kernel becomes resident only
# as earlier ones exit: a register-A GEMM (mxfp8, nvfp4: one CTA per SM, the whole register file) needs an SM no
# parked producer CTA occupies, and a prefill-tile GEMM's ring leaves no room for the next one.  Those chains overlap
# as far as they fit and are still compared with their serialized run.
PREMISE_CHAINS = ([f"weight-{f}-{v}" for f in ("int8", "fp8") for v in ("direct", "act")]
                  + [f"act-{k}-M1" for k in ("reg", "rmsnorm", "silu", "fakequant", "mxfp8", "nvfp4")] + ["gemm-out-M32"])


@pytest.mark.parametrize("name", PREMISE_CHAINS)
def test_stall_head_opens_the_window(lib, head, name):
    """Premise of the module: behind the head, every kernel of these chains starts before the head ends, so its
    pre-wait reads happen while its producers are still parked.  The weight chains run here WITHOUT their fence, to
    show the window the fence closes: the linear is running, and requesting its weights, before the weight quantizer
    ahead of it has written anything.  (Their outputs are not looked at.)
    Measured on a replay of the head and the chain captured in one CUDA graph: the graph hands every launch to the
    device at once, so whether a kernel starts inside the window depends on PDL alone.  Launched eagerly, a kernel
    the host enqueues after the head has ended (a host thread descheduled for the head's ~16 ms on a loaded machine)
    would start late without anything on the device being wrong."""
    c = dict(CHAINS)[name](lib)
    c.poison()
    steps = [s for s in c.steps if s[0] != FENCE]
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        c.run(head=head, steps=steps)
    graph.replay()   # the first replay uploads the graph
    torch.cuda.synchronize()
    spans = _kernel_spans(graph.replay)
    assert spans and "rowwise_cta_kernel" in spans[0][0], spans[:3]
    head_end = spans[0][2]
    assert len(spans) >= 1 + len(steps), [s[0] for s in spans]   # the head, then at least one kernel per call
    late = [(n[:60], round(s - head_end, 1)) for n, s, _ in spans[1:] if s >= head_end]
    assert not late, f"head ran {head_end - spans[0][1]:.1f} us; these kernels started after it ended: {late}"


# ---------------------------------------------------------------------------------------------------- public API
def _configs():
    from ao_b200.prototype.mx_formats import (MXDynamicActivationMXWeightConfig, NVFP4DynamicActivationNVFP4WeightConfig,
                                              NVFP4WeightFloat8ActivationConfig, NVFP4WeightOnlyConfig)
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Int4WeightOnlyConfig,
                                      Int8DynamicActivationInt8WeightConfig, PerRow)

    return {"int8": Int8DynamicActivationInt8WeightConfig(), "fp8": Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()),
            "mxfp8": MXDynamicActivationMXWeightConfig(), "nvfp4": NVFP4DynamicActivationNVFP4WeightConfig(),
            "nvfp4w": NVFP4WeightOnlyConfig(), "nvfp4w_fp8a": NVFP4WeightFloat8ActivationConfig(),
            "int4": Int4WeightOnlyConfig(group_size=32, int4_packing_format="tile_packed_to_4d")}


@pytest.mark.parametrize("fmt", ["int8", "fp8", "mxfp8", "nvfp4", "nvfp4w", "nvfp4w_fp8a", "int4"])
def test_quantize_then_forward_at_once(fmt):
    """quantize_(lin, cfg) followed at once by lin(x), x created before quantize_, against the same with a sync
    between them.  int8 / fp8 with K = 2^20 and 16 output rows: the weight quantizer is one long CTA per row, its own
    stall head for the activation quantizer and the GEMM behind it."""
    from ao_b200.quantization import quantize_

    K = 1 << 20 if fmt in ("int8", "fp8") else 4096
    g = _g(21)
    lin_a = nn.Linear(K, 16 if fmt in ("int8", "fp8") else 256, bias=True, device=DEV, dtype=torch.bfloat16)
    lin_b = nn.Linear(K, lin_a.out_features, bias=True, device=DEV, dtype=torch.bfloat16)
    lin_b.load_state_dict(lin_a.state_dict())
    x = _bf16((32, K), g)
    torch.cuda.synchronize()
    with torch.no_grad():
        quantize_(lin_b, _configs()[fmt])
        torch.cuda.synchronize()
        want = lin_b(x)
        torch.cuda.synchronize()
        quantize_(lin_a, _configs()[fmt])
        got = lin_a(x)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{fmt}: quantize_ -> forward differs from the synced run"


@pytest.mark.parametrize("fmt", ["int4", "fp8"])
@pytest.mark.parametrize("fused", [False, True])
def test_llama_stack_overlapped_equals_synced(fmt, fused):
    """The bench model (fused or not) at M = 1, 32 and 300 against the same forward with a torch.cuda.synchronize()
    after every linear, then a CUDA graph of it replayed on a new input."""
    from ao_b200.fusion import fuse_parallel_linears
    from ao_b200.models import LlamaLinearStack, LlamaShape
    from ao_b200.quantization import quantize_

    m = LlamaLinearStack(LlamaShape("tiny", 1024, 3072, 256, 2), device=DEV, seed=0, init_scale=0.05)
    quantize_(m, _configs()[fmt])
    if fused:
        assert fuse_parallel_linears(m) == 4

    def synced(x):
        hooks = [mod.register_forward_hook(lambda *_: torch.cuda.synchronize()) for mod in m.modules()
                 if isinstance(mod, nn.Linear)]
        try:
            torch.cuda.synchronize()
            return m(x)
        finally:
            for h in hooks:
                h.remove()

    g = _g(23)
    with torch.no_grad():
        for M in (1, 32, 300):
            x = _bf16((M, 1024), g)
            want = synced(x)
            torch.cuda.synchronize()
            got = m(x)
            torch.cuda.synchronize()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"M={M}: overlapped forward differs"
        x = _bf16((32, 1024), g)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            m(x)   # the capture stream's workspace, outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=st):
            y = m(x)
        x.copy_(_bf16((32, 1024), g))
        torch.cuda.synchronize()
        want = synced(x)
        y.fill_(float("nan"))
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), "graph replay differs from the synced forward"
