#!/usr/bin/env python
"""Outputs and times of the per-token activation quantizers, for comparing two builds of the package.

  python scripts/measure_rowwise_quant.py run OUT.pt [--tree DIR] [--check] [--time]
  python scripts/measure_rowwise_quant.py compare A.pt B.pt [A2.pt B2.pt ...]

`run` imports ao_b200 from DIR (default: this checkout) and writes OUT.pt with
  * `--check`: for the seven quantizer ops (int8 / fp8 / fakequant rowwise, RMSNorm- and SiLU-mul-fused int8 / fp8)
    at M in {1, 7, 32, 300, 2048} x K in {1024, 4096, 14336, 16384, 16392, 28672, 32768}, a SHA-256 of the codes and
    scales on seeded finite inputs without -0.0 (each op also checked in-process to give the same result on a
    row-strided input, ldx = K + 64, as on a dense one), and the full outputs on inputs with -0.0, NaN, +-inf and
    subnormal rows at M = 7;
  * `--time`: the time of each op, CUDA events around CUDA-graph replays, at M in {1, 32, 256, 2048} x
    K in {4096, 14336, 28672};
  * the card's name and power limit.
`compare` takes files in (A, B) pairs: the digests of A and B must agree; of the special-value outputs it counts
the codes that differ, and which of them are the int8 NaN-quotient change (-128 -> 0) or the e4m3 negative-zero change
(0x00 -> 0x80); it prints the times of A and B side by side (median of the runs, min-max in brackets).  Two builds
cannot share a process (both register torch.ops.ao_b200), hence one `run` per build, alternated by the caller.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import statistics
import subprocess
import sys

CHECK_M = [1, 7, 32, 300, 2048]
CHECK_K = [1024, 4096, 14336, 16384, 16392, 28672, 32768]
TIME_M = [1, 32, 256, 2048]
TIME_K = [4096, 14336, 28672]
OPS = ["int8", "fp8", "fakequant", "rmsnorm_int8", "rmsnorm_fp8", "silu_int8", "silu_fp8"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip()


def inputs(M, K, seed, special=False):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = torch.logspace(-3, 3, M, device="cuda").unsqueeze(1)
    xw = (torch.randn(M, K + 64, device="cuda", generator=g) * scale).to(torch.bfloat16)
    gu = (torch.randn(M, 2 * K, device="cuda", generator=g) * 2).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(K, device="cuda", generator=g)).to(torch.bfloat16)
    if special:
        for t in (xw, gu):
            t[:, 1::97] = -0.0
            t[1, 3] = float("nan")
            t[2, 5] = float("inf")
            t[3, 7] = float("-inf")
            t[4, ::3] = 2.0 ** -130
            t[5] = 0
        xw[6] = 2.0 ** -133   # a row of subnormals only: its bf16 scale rounds to 0
    return xw[:, :K], gu[:, :K], gu[:, K:], w


def call(ops, name, x, gate, up, w):
    if name == "int8":
        return ops.int8_quantize_rowwise(x)
    if name == "fp8":
        return ops.fp8_quantize_rowwise(x)
    if name == "fakequant":
        return ops.fp8_fakequant_rowwise(x)
    fmt = 0 if name.endswith("int8") else 1
    if name.startswith("rmsnorm"):
        return ops.rmsnorm_quantize_rowwise(x, w, 1e-5, fmt)
    return ops.silu_mul_quantize_rowwise(gate, up, fmt)


def as_bytes(t):
    import torch

    return t.contiguous().view(torch.uint8)


def digest(q, s):
    h = hashlib.sha256()
    h.update(as_bytes(q).cpu().numpy().tobytes())
    h.update(as_bytes(s).cpu().numpy().tobytes())
    return h.hexdigest()


def check(ops):
    import torch

    digests, special = {}, {}
    for M in CHECK_M:
        for K in CHECK_K:
            x, gate, up, w = inputs(M, K, seed=M * 100003 + K)
            for name in OPS:
                q, s = call(ops, name, x, gate, up, w)
                qc, sc = call(ops, name, x.contiguous(), gate.contiguous(), up.contiguous(), w)
                assert torch.equal(as_bytes(q), as_bytes(qc)) and torch.equal(s, sc), f"{name} {M}x{K}: strided != dense"
                digests[f"{name} {M}x{K}"] = digest(q, s)
    for K in [4096, 16384, 16392, 28672]:
        x, gate, up, w = inputs(7, K, seed=K, special=True)
        for name in OPS:
            q, s = call(ops, name, x, gate, up, w)
            special[f"{name} 7x{K}"] = (as_bytes(q).cpu(), as_bytes(s).cpu())
    return digests, special


def time_ops(ops):
    """Median per-call time over 5 timed replays of a CUDA graph of `iters` back-to-back calls: GPU time, not the
    host's dispatch overhead, which dominates eager calls at small M."""
    import torch

    out = {}
    for M in TIME_M:
        for K in TIME_K:
            x, gate, up, w = inputs(M, K, seed=1)
            x = x.contiguous()
            iters = 100 if M * K <= 256 * 28672 else 20
            for name in OPS:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for _ in range(3):
                        call(ops, name, x, gate, up, w)
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    for _ in range(iters):
                        call(ops, name, x, gate, up, w)
                for _ in range(3):
                    graph.replay()
                ts = []
                for _ in range(5):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(10):
                        graph.replay()
                    b.record()
                    b.synchronize()
                    ts.append(a.elapsed_time(b) * 1e3 / (10 * iters))
                out[f"{name} {M}x{K}"] = statistics.median(ts)
                del graph
            torch.cuda.empty_cache()
    return out


def run(args):
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch

    import ao_b200  # noqa: F401

    assert torch.cuda.is_available(), "needs a CUDA device"
    ops = torch.ops.ao_b200
    res = {"card": card(), "tree": os.path.abspath(args.tree)}
    if args.check:
        res["digests"], res["special"] = check(ops)
    if args.time:
        res["time_us"] = time_ops(ops)
    torch.save(res, args.out)
    print(f"wrote {args.out} ({res['card']})")


def classify(name, qa, qb):
    import torch

    diff = qa != qb
    if name in ("int8", "rmsnorm_int8", "silu_int8"):
        allowed = diff & (qa == 0x80) & (qb == 0)          # int8 -128 -> 0
    elif name == "fakequant":
        allowed = torch.zeros_like(diff)
    else:
        allowed = diff & (qa == 0x00) & (qb == 0x80)       # e4m3 +0 -> -0
    return int(diff.sum()), int(allowed.sum())


def compare(files):
    import torch

    runs = [(torch.load(a, weights_only=False), torch.load(b, weights_only=False)) for a, b in zip(files[::2], files[1::2])]
    ok = True
    print("card:", runs[0][0]["card"])
    for a, b in runs:
        if "digests" not in a:
            continue
        bad = [k for k in a["digests"] if a["digests"][k] != b["digests"].get(k)]
        print(f"finite inputs: {len(a['digests']) - len(bad)}/{len(a['digests'])} outputs identical", bad[:10])
        ok &= not bad
        for k in a["special"]:
            (qa, sa), (qb, sb) = a["special"][k], b["special"][k]
            n, allowed = classify(k.split()[0], qa, qb)
            same_s = torch.equal(sa, sb)
            print(f"special {k:24s} scales {'equal' if same_s else 'DIFFER'}; codes differing {n}, of them intended {allowed}")
            ok &= same_s and n == allowed
    timed = [(a["time_us"], b["time_us"]) for a, b in runs if "time_us" in a]
    if timed:
        print(f"{'op':28s} {'A us':>22s} {'B us':>22s}   B/A")
        for k in timed[0][0]:
            ta = [t[0][k] for t in timed]
            tb = [t[1][k] for t in timed]
            ma, mb = statistics.median(ta), statistics.median(tb)
            print(f"{k:28s} {ma:8.2f} [{min(ta):5.2f}-{max(ta):5.2f}] {mb:8.2f} [{min(tb):5.2f}-{max(tb):5.2f}]  {mb / ma:5.3f}")
    print("RESULT", "OK" if ok else "MISMATCH")
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("out")
    r.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    r.add_argument("--check", action="store_true")
    r.add_argument("--time", action="store_true")
    c = sub.add_parser("compare")
    c.add_argument("files", nargs="+")
    args = ap.parse_args()
    if args.cmd == "run":
        run(args)
        return 0
    return compare(args.files)


if __name__ == "__main__":
    sys.exit(main())
