#!/usr/bin/env python
"""Times the fp8 rowwise grouped GEMM (torch.ops.ao_b200.fp8_rowwise_grouped_mm) against torch's rowwise
F.scaled_grouped_mm on identical operands, for MoE expert shapes; with --fmt nvfp4, the NVFP4 expert path (the
per-expert activation quantizer nvfp4_fakequant_grouped plus nvfp4_grouped_mm) against the fp8 path with its
quantizer (fp8_quantize_rowwise plus fp8_rowwise_grouped_mm) and bf16 torch._grouped_mm on the unquantized weights.

  python scripts/measure_grouped_mm.py [--fmt fp8|nvfp4] [--replays 20] [--out FILE]

  * shapes: Mixtral-8x7B experts (E=8, 4096 -> 14336 and 14336 -> 4096, top-2) and Qwen3-30B-A3B experts (E=128,
    2048 -> 768 and 768 -> 2048, top-8);
  * 1, 8, 32 and 128 decode tokens and one 2048-token prefill, each with a seeded balanced routing (every token picks
    top-k distinct experts uniformly) and a seeded skewed one (expert e drawn with weight 1 / (e + 1)^1.2);
  * each op runs from CUDA-graph replays that cycle through enough weight copies that the active experts' weights
    are never in the 50 MB L2 when they are read again; µs per call = event time / calls.
Reported per case: µs, the output's SQNR against torch's on the written rows ("identical" when every bit agrees),
GB/s over the bytes the GEMM needs (weights and scales of experts with at least one row,
activations, their scales, outputs, offs), and which data-sheet roofline term bounds it (H100 SXM: 3.35 TB/s HBM3,
1979 TFLOP/s dense fp8; figures for a 700 W card) with the time that term gives.  One JSON line per case, then one with
the card's name, power limit and maximum SM clock.  --fmt nvfp4 reports µs and GB/s of the three paths over the bytes
the NVFP4 path needs (0.5625 bytes per weight of the active experts, the bf16 activations read once, the outputs) and
the output's SQNR against bf16 torch._grouped_mm; its roofline term is the HBM time of those bytes (the bf16 wgmma
roofline, 989 TFLOP/s, is never the bound at these shapes up to 128 tokens).
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L2_BYTES = 50 * 2**20
HBM_BPS = 3.35e12
FP8_FLOPS = 1979e12
SHAPES = [("mixtral-8x7b w1/w3", 8, 14336, 4096, 2), ("mixtral-8x7b w2", 8, 4096, 14336, 2),
          ("qwen3-30b-a3b gate/up", 128, 768, 2048, 8), ("qwen3-30b-a3b down", 128, 2048, 768, 8)]
TOKENS = [1, 8, 32, 128, 2048]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip()


def routing(T, E, topk, skewed, seed):
    """Rows per expert for T tokens routed to top-k distinct experts each."""
    import torch

    g = torch.Generator().manual_seed(seed)
    w = torch.tensor([1.0 / (e + 1) ** 1.2 for e in range(E)]) if skewed else torch.ones(E)
    picks = torch.multinomial(w.expand(T, E), topk, replacement=False, generator=g)
    return torch.bincount(picks.reshape(-1), minlength=E).tolist()


def time_graph(fn_of_copy, copies, replays):
    """µs per call of fn_of_copy(c) from a CUDA graph that calls it once for every weight copy c, several rounds."""
    import torch

    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for c in range(copies):   # warm-up outside the capture (workspaces, module loads)
            fn_of_copy(c)
    torch.cuda.synchronize()
    rounds = max(1, 64 // copies)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for _ in range(rounds):
            for c in range(copies):
                fn_of_copy(c)
    g.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(replays):
        g.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / (replays * rounds * copies)


def sqnr_db(ref, out):
    import torch

    d = (out.double() - ref.double()).norm()
    return round(float(20 * torch.log10(ref.double().norm() / d)), 1) if d > 0 else "identical"


def measure_nvfp4(a, ops, dev, lines):
    """The NVFP4 expert path (prologue + GEMM) against fp8 (prologue + GEMM) and bf16 torch._grouped_mm."""
    import torch

    from ao_b200.prototype.mx_formats import per_tensor_amax_to_scale

    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        bf16_expert = N * K * 2
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 0.5625)) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * bf16_expert)) + 1)
        w4, s4, p4, w8, s8, wb = [], [], [], [], [], []
        for c in range(max(copies, copies_bf16)):
            w = (torch.randn(E, N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            if c < copies:
                pts = per_tensor_amax_to_scale(torch.amax(torch.abs(w), dim=(1, 2)))
                qs = [ops.nvfp4_quantize(w[e], pts[e].reshape(1), True) for e in range(E)]
                w4.append(torch.stack([q for q, _ in qs]))
                s4.append(torch.stack([s for _, s in qs]))
                p4.append(pts)
                q, s = ops.fp8_quantize_rowwise(w.reshape(E * N, K))
                w8.append(q.reshape(E, N, K))
                s8.append(s.reshape(E, N))
            if c < copies_bf16:
                wb.append(w)
            del w
        for T in TOKENS:
            for skewed in (False, True):
                rows = routing(T, E, topk, skewed, seed=T * 131 + E + skewed)
                M = sum(rows)
                offs = torch.tensor(rows, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)
                x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
                active = sum(1 for r in rows if r)
                need = int(active * N * K * 0.5625) + M * K * 2 + M * N * 2 + E * 8
                rec = dict(fmt="nvfp4", shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))

                def ours(c):
                    xhat, xs = ops.nvfp4_fakequant_grouped(x, offs)
                    return ops.nvfp4_grouped_mm(xhat, xs, w4[c], s4[c], p4[c], offs)

                def fp8(c):
                    xq, sx = ops.fp8_quantize_rowwise(x)
                    return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), w8[c], s8[c], offs)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                n = int(offs[-1])
                y_ref = bf16(0)
                rec["sqnr_vs_bf16_db"] = sqnr_db(y_ref[:n], ours(0)[:n])
                for key, fn, cp in (("ours", ours, copies), ("fp8", fp8, copies), ("bf16", bf16, copies_bf16)):
                    us = time_graph(fn, cp, a.replays)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del w4, s4, p4, w8, s8, wb
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fmt", choices=["fp8", "nvfp4"], default="fp8")
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    import ao_b200  # noqa: F401

    assert torch.cuda.is_available(), "needs a CUDA device"
    ops = torch.ops.ao_b200
    dev = torch.device("cuda", 0)
    lines = []
    for name, E, N, K, topk in (SHAPES if a.fmt == "fp8" else []):
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        w_bytes_expert = N * K + N * 4
        min_active = min(topk, E) * w_bytes_expert
        copies = max(2, math.ceil(2 * L2_BYTES / min_active) + 1)
        wq, sw = [], []
        for _ in range(copies):
            w = (torch.randn(E * N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            q, s = ops.fp8_quantize_rowwise(w)
            wq.append(q.reshape(E, N, K))
            sw.append(s.reshape(E, N))
            del w
        for T in TOKENS:
            for skewed in (False, True):
                rows = routing(T, E, topk, skewed, seed=T * 131 + E + skewed)
                M = sum(rows)
                offs = torch.tensor(rows, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)
                x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
                xq, sx = ops.fp8_quantize_rowwise(x)
                sx = sx.reshape(-1)
                active = sum(1 for r in rows if r)
                need = active * w_bytes_expert + M * K + M * 4 + M * N * 2 + E * 4
                t_mem, t_fp = need / HBM_BPS * 1e6, 2.0 * M * N * K / FP8_FLOPS * 1e6
                rec = dict(shape=name, E=E, N=N, K=K, topk=topk, tokens=T, routing="skewed" if skewed else "balanced",
                           rows=M, active_experts=active, bytes=need, weight_copies=copies,
                           bound="memory" if t_mem >= t_fp else "compute", roofline_us=round(max(t_mem, t_fp), 2))
                ours = lambda c: ops.fp8_rowwise_grouped_mm(xq, sx, wq[c], sw[c], offs)
                us = time_graph(ours, copies, a.replays)
                rec["ours_us"] = round(us, 2)
                rec["ours_GBps"] = round(need / us * 1e-3, 1)

                def theirs(c):
                    return F.scaled_grouped_mm(xq, wq[c].transpose(-2, -1), scale_a=sx, scale_recipe_a=F.ScalingType.RowWise,
                                               scale_b=sw[c], scale_recipe_b=F.ScalingType.RowWise, offs=offs,
                                               output_dtype=torch.bfloat16)
                try:
                    y_t = theirs(0)
                    y = ours(0)
                    n = int(offs[-1])
                    d = (y[:n].double() - y_t[:n].double()).norm()
                    rec["sqnr_vs_torch_db"] = (round(float(20 * torch.log10(y_t[:n].double().norm() / d)), 1) if d > 0
                                               else "identical")
                    us_t = time_graph(theirs, copies, a.replays)
                    rec["torch_us"] = round(us_t, 2)
                    rec["torch_GBps"] = round(need / us_t * 1e-3, 1)
                except (RuntimeError, NotImplementedError) as e:
                    rec["torch_us"] = f"unavailable: {str(e).splitlines()[0][:160]}"
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del wq, sw
        torch.cuda.empty_cache()
    if a.fmt == "nvfp4":
        measure_nvfp4(a, ops, dev, lines)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(info=info, cases=lines), f, indent=1)


if __name__ == "__main__":
    main()
