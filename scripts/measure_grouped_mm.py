#!/usr/bin/env python
"""Times the fp8 rowwise grouped GEMM (torch.ops.ao_b200.fp8_rowwise_grouped_mm) against torch's rowwise
F.scaled_grouped_mm on identical operands, for MoE expert shapes.

  python scripts/measure_grouped_mm.py [--replays 20] [--out FILE]

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
the card's name, power limit and maximum SM clock.
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


def main():
    ap = argparse.ArgumentParser()
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
    for name, E, N, K, topk in SHAPES:
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
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(info=info, cases=lines), f, indent=1)


if __name__ == "__main__":
    main()
