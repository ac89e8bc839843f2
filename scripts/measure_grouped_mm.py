#!/usr/bin/env python
"""Times the fp8 rowwise grouped GEMM (torch.ops.ao_b200.fp8_rowwise_grouped_mm) against torch's rowwise
F.scaled_grouped_mm on identical operands, for MoE expert shapes; with --fmt nvfp4, the NVFP4 expert path (the
per-expert activation quantizer nvfp4_fakequant_grouped plus nvfp4_grouped_mm) against the fp8 path with its
quantizer (fp8_quantize_rowwise plus fp8_rowwise_grouped_mm) and bf16 torch._grouped_mm on the unquantized weights.

  python scripts/measure_grouped_mm.py [--fmt fp8|nvfp4|int4|fp8wo|int8wo|int8|fp8_blockwise|mxfp8|mxfp4] [--group-size 32]
                                       [--replays 20] [--prologue]
                                       [--out FILE]

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
roofline, 989 TFLOP/s, is never the bound at these shapes up to 128 tokens).  --fmt int4 --group-size {32,128}: the
int4 expert GEMM (int4_tilepacked_grouped_mm on 3-D Int4TilePackedTo4dTensor weights) against the dense int4 linear of
each active expert (the select loop, captured with the routing fixed, without its host syncs), the fp8 path with its
quantizer and bf16 torch._grouped_mm; bytes are the int4 path's (0.5 + 4 / g bytes per weight of the active experts,
K and N as padded, the bf16 activations read once, the outputs).  --fmt fp8wo: the weight-only e4m3 expert GEMM
(torch._grouped_mm on 3-D Float8Tensor weights of Float8WeightOnlyConfig) against the reference's recipe (torch._grouped_mm
on W.dequantize(), all E experts dequantized on every call), bf16 torch._grouped_mm and the fp8 dynamic path with its
quantizer; bytes are the weight-only path's (1 byte per weight and 4 per row scale of the active experts, the bf16
activations read once, the outputs, offs) and its roofline term the HBM time of those bytes.  --fmt int8wo / int8:
the int8 expert GEMM (torch._grouped_mm on 3-D Int8Tensor weights; int8: dynamic PerRow activations, quantizer
included) against this engine's dense int8 op per active expert (the select loop, captured with the routing fixed),
the reference's per-expert recipe restated in torch (int8wo: torch.mm on qdata.to(bf16) times the bf16 scale; int8:
per-row quantization, torch._int_mm and the pointwise epilogue), bf16 torch._grouped_mm and the fp8 counterpart (fp8
weight-only, or fp8 rowwise with its quantizer); bytes are the int8 path's (1 byte per weight and 4 per row scale of
the active experts, the activations as the GEMM reads them, the outputs, offs), its roofline term their HBM time, and
vs_select_linear compares the output with select + F.linear on every active expert.  --fmt fp8_blockwise: the blockwise
e4m3 expert path (torch._grouped_mm on 3-D Float8Tensor weights with [1, 128, 128] blocks: the 1x128 quantizer plus
fp8_blockwise_grouped_mm) against the eager loop of select + the dense blockwise linear on each active expert (its
quantizer and GEMM, captured with the routing fixed, without the host sync that reads offs), the rowwise fp8 grouped
op with its quantizer on the same codes, and bf16 torch._grouped_mm, on the shapes above plus DeepSeek-V3's experts
(E=256, 7168 -> 4096 gate|up and 2048 -> 7168 down, top-8); bytes are the blockwise path's (1 byte per weight and 4 per
128x128 block scale of the active experts, the e4m3 activations and their 1x128 scales, the outputs, offs), its
roofline term their HBM time, and vs_select_linear compares the output with the loop's.  Torch's blockwise
F.scaled_grouped_mm is tried and reported as unavailable when this torch build lacks it (it needs torch built for
CUDA 12.9 or later).  --fmt mxfp8 / mxfp4: the MX expert path (torch._grouped_mm on 3-D MXTensor weights:
mx*_fakequant plus mx*_grouped_mm) against the eager loop of select + the dense MX linear on each active expert (its
quantizer and GEMM, captured with the routing fixed), the fp8 rowwise path with its quantizer and bf16
torch._grouped_mm; bytes are the MX path's (1 or 0.5 bytes per weight and 1 per 32-weight scale of the active experts,
the bf16 activations read once, the outputs, offs) and its roofline term their HBM time; vs_select_linear compares the
output with the loop's.  With --prologue it gives instead the kernel time of the one-launch prologue (mx*_fakequant)
and of the two launches it replaces (mx*_quantize, then the dense linear's dequant_act_kernel), alternated in one
torch.profiler run with PDL off.  Prefill (2048-token) cases time one round of weight copies per replay.
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
DEEPSEEK_SHAPES = [("deepseek-v3 gate|up", 256, 4096, 7168, 8), ("deepseek-v3 down", 256, 7168, 2048, 8)]


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


def time_graph(fn_of_copy, copies, replays, rounds=None):
    """µs per call of fn_of_copy(c) from a CUDA graph that calls it once for every weight copy c, several rounds."""
    import torch

    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for c in range(copies):   # warm-up outside the capture (workspaces, module loads)
            fn_of_copy(c)
    torch.cuda.synchronize()
    rounds = rounds or max(1, 64 // copies)
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


def measure_int4(a, ops, dev, lines):
    """The int4 expert GEMM against the per-expert dense int4 linears, fp8 (prologue + GEMM) and bf16."""
    import torch

    from ao_b200.quantization import Int4TilePackedTo4dTensor

    gs = a.group_size
    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        Np, Kp = -(-N // 8) * 8, -(-K // 1024) * 1024
        per_weight = 0.5 + 4.0 / gs
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * Np * Kp * per_weight)) + 1)
        copies8 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K)) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 2)) + 1)
        w4, w8, s8, wb = [], [], [], []
        for c in range(max(copies, copies8, copies_bf16)):
            w = (torch.randn(E, N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            if c < copies:
                w4.append(Int4TilePackedTo4dTensor.from_hp(w, [1, 1, gs]))
            if c < copies8:
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
                xp = torch.nn.functional.pad(x, (0, Kp - K)).contiguous()
                active = sum(1 for r in rows if r)
                need = int(active * Np * Kp * per_weight) + M * Kp * 2 + M * N * 2 + E * 4
                rec = dict(fmt=f"int4 g{gs}", shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))
                spans, start = [], 0
                for e, r in enumerate(rows):
                    if r:
                        spans.append((e, start, start + r))
                    start += r

                def ours(c):
                    return torch._grouped_mm(x, w4[c].transpose(-2, -1), offs=offs)

                def loop(c):
                    w = w4[c]
                    for e, s0, s1 in spans:
                        ops.int4_tilepacked_linear(xp[s0:s1], w.qdata[e], gs, w.scale_and_zero[e], None, N, 0)

                def fp8(c):
                    xq, sx = ops.fp8_quantize_rowwise(x)
                    return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), w8[c], s8[c], offs)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                n = int(offs[-1])
                rec["sqnr_vs_bf16_db"] = sqnr_db(bf16(0)[:n], ours(0)[:n])
                for key, fn, cp in (("ours", ours, copies), ("expert_loop", loop, copies), ("fp8", fp8, copies8),
                                    ("bf16", bf16, copies_bf16)):
                    us = time_graph(fn, cp, a.replays)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del w4, w8, s8, wb
        torch.cuda.empty_cache()


def measure_fp8wo(a, ops, dev, lines):
    """The weight-only e4m3 expert GEMM (torch._grouped_mm on a 3-D Float8Tensor without act_quant_kwargs) against
    the reference's recipe (torch._grouped_mm on W.dequantize(), every expert dequantized in eager torch on each call),
    bf16 torch._grouped_mm and the fp8 dynamic path with its quantizer."""
    import torch

    from ao_b200.quantization import Float8Tensor, PerRow

    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * (N * K + N * 4))) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 2)) + 1)
        wo, w8, s8, wb = [], [], [], []
        for c in range(max(copies, copies_bf16)):
            w = (torch.randn(E, N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            if c < copies:
                t = Float8Tensor.from_hp(w, torch.float8_e4m3fn, PerRow())
                wo.append(t)
                w8.append(t.qdata)
                s8.append(t.scale.reshape(E, N))
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
                need = active * (N * K + N * 4) + M * K * 2 + M * N * 2 + E * 4
                rec = dict(fmt="fp8wo", shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))

                def ours(c):
                    return torch._grouped_mm(x, wo[c].transpose(-2, -1), offs=offs)

                def recipe(c):
                    return torch._grouped_mm(x, wo[c].dequantize().transpose(-2, -1), offs=offs)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                def fp8(c):
                    xq, sx = ops.fp8_quantize_rowwise(x)
                    return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), w8[c], s8[c], offs)

                n = int(offs[-1])
                y = ours(0)[:n]
                rec["sqnr_vs_recipe_db"] = sqnr_db(recipe(0)[:n], y)
                rec["sqnr_vs_bf16_db"] = sqnr_db(bf16(0)[:n], y)
                # the recipe allocates a bf16 copy of all E experts per call: one round of copies per replay
                for key, fn, cp, rounds in (("ours", ours, copies, None), ("recipe", recipe, copies, 1),
                                            ("bf16", bf16, copies_bf16, None), ("fp8", fp8, copies, None)):
                    us = time_graph(fn, cp, a.replays, rounds)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del wo, w8, s8, wb
        torch.cuda.empty_cache()


def measure_int8(a, ops, dev, lines):
    """The int8 expert GEMM (torch._grouped_mm on a 3-D Int8Tensor; --fmt int8wo weight-only, --fmt int8 dynamic PerRow
    activations with their quantizer) against this engine's dense int8 op on each active expert (the select loop,
    captured with the routing fixed, without its host syncs), the reference's per-expert recipe restated in torch,
    bf16 torch._grouped_mm, and this engine's fp8 counterpart (fp8 weight-only, or fp8 rowwise with its quantizer)."""
    import torch

    from ao_b200.quantization import Float8Tensor, Int8Tensor, PerRow, QuantizeTensorToInt8Kwargs

    dyn = a.fmt == "int8"
    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * (N * K + N * 4))) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 2)) + 1)
        w8, f8, wb = [], [], []
        kw = dict(act_quant_kwargs=QuantizeTensorToInt8Kwargs(granularity=PerRow())) if dyn else {}
        for c in range(max(copies, copies_bf16)):
            w = (torch.randn(E, N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            if c < copies:
                w8.append(Int8Tensor.from_hp(w, PerRow(), **kw))
                f8.append(Float8Tensor.from_hp(w, torch.float8_e4m3fn, PerRow()))
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
                act_bytes = M * K + M * 4 if dyn else M * K * 2
                need = active * (N * K + N * 4) + act_bytes + M * N * 2 + E * 4
                rec = dict(fmt=a.fmt, shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))
                spans, start = [], 0
                for e, r in enumerate(rows):
                    if r:
                        spans.append((e, start, start + r))
                    start += r
                ws = [t.scale.reshape(E, N).float() for t in w8]

                def ours(c):
                    return torch._grouped_mm(x, w8[c].transpose(-2, -1), offs=offs)

                def loop(c):
                    w = w8[c]
                    if dyn:
                        xq, sx = ops.int8_quantize_rowwise(x)
                        for e, s0, s1 in spans:
                            ops.int8_dyn_linear(xq[s0:s1], sx.reshape(-1)[s0:s1], w.qdata[e], ws[c][e], None)
                    else:
                        for e, s0, s1 in spans:
                            ops.int8_weight_linear(x[s0:s1], w.qdata[e], ws[c][e], None)

                def recipe(c):
                    # per expert, in torch: weight-only torch.mm on qdata.to(bf16) times the bf16 scale; dynamic
                    # per-row quantization, torch._int_mm (rows padded to 17, its minimum on CUDA) and the epilogue
                    w = w8[c]
                    for e, s0, s1 in spans:
                        xe = x[s0:s1]
                        if dyn:
                            sx = (xe.float().abs().amax(dim=1, keepdim=True) / 127).clamp(min=torch.finfo(torch.float32).eps)
                            xq = torch.clamp(torch.round(xe.float() / sx), -128, 127).to(torch.int8)
                            xq = torch.nn.functional.pad(xq, (0, 0, 0, max(0, 17 - xq.shape[0])))
                            acc = torch._int_mm(xq, w.qdata[e].t())[: s1 - s0]
                            (acc * sx).to(torch.bfloat16) * ws[c][e]
                        else:
                            torch.mm(xe, w.qdata[e].to(torch.bfloat16).t()) * ws[c][e].to(torch.bfloat16)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                if dyn:
                    def fp8(c):
                        xq, sx = ops.fp8_quantize_rowwise(x)
                        return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), f8[c].qdata, f8[c].scale.reshape(E, N), offs)
                else:
                    def fp8(c):
                        return torch._grouped_mm(x, f8[c].transpose(-2, -1), offs=offs)

                n = int(offs[-1])
                y = ours(0)[:n]
                y_loop = torch.cat([torch.nn.functional.linear(x[s0:s1], w8[0][e]) for e, s0, s1 in spans])
                rec["vs_select_linear"] = "identical" if torch.equal(y.view(torch.int16), y_loop.view(torch.int16)) \
                    else sqnr_db(y_loop, y)
                rec["sqnr_vs_bf16_db"] = sqnr_db(bf16(0)[:n], y)
                for key, fn, cp in (("ours", ours, copies), ("expert_loop", loop, copies), ("recipe", recipe, copies),
                                    ("bf16", bf16, copies_bf16), ("fp8" if dyn else "fp8wo", fp8, copies)):
                    us = time_graph(fn, cp, a.replays)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del w8, f8, wb
        torch.cuda.empty_cache()


def measure_fp8_blockwise(a, ops, dev, lines):
    """The blockwise e4m3 expert path (quantizer + grouped GEMM) against the eager select + dense blockwise loop, the
    rowwise fp8 grouped op (quantizer + GEMM) on the same codes, and bf16 torch._grouped_mm.  DeepSeek-V3's gate|up is
    7.5 GB of e4m3 (15 GB of bf16) for all 256 experts: its weights are made and quantized 16 experts at a time, and one
    copy of its active experts' weights is already far past L2."""
    import torch
    import torch.nn.functional as F

    from ao_b200.quantization import Float8Tensor, PerBlock, QuantizeTensorToFloat8Kwargs

    act = QuantizeTensorToFloat8Kwargs(granularity=PerBlock([1, 128]))
    for name, E, N, K, topk in SHAPES + DEEPSEEK_SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        w_bytes_expert = N * K + (N // 128) * (K // 128) * 4
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * w_bytes_expert)) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 2)) + 1)
        wt, wb = [], []
        for c in range(max(copies, copies_bf16)):
            w = torch.randn(E, N, K, device=dev, generator=g, dtype=torch.bfloat16).mul_(0.05)
            if c < copies:
                parts = [Float8Tensor.from_hp(w[e0:e0 + 16], granularity=PerBlock([128, 128])) for e0 in range(0, E, 16)]
                wt.append(Float8Tensor(torch.cat([p.qdata for p in parts]), torch.cat([p.scale for p in parts]),
                                       [1, 128, 128], parts[0].mm_config, act, dtype=torch.bfloat16))
                del parts
            if c < copies_bf16:
                wb.append(w)
            del w
        ones = torch.ones(E, N, device=dev)   # the rowwise op's scales: only its time is compared
        for T in TOKENS:
            for skewed in (False, True):
                rows = routing(T, E, topk, skewed, seed=T * 131 + E + skewed)
                M = sum(rows)
                offs = torch.tensor(rows, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)
                x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
                active = sum(1 for r in rows if r)
                need = active * w_bytes_expert + M * K + M * (K // 128) * 4 + M * N * 2 + E * 4
                rec = dict(fmt="fp8_blockwise", shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))
                spans, start = [], 0
                for e, r in enumerate(rows):
                    if r:
                        spans.append((e, start, start + r))
                    start += r

                def ours(c):
                    return torch._grouped_mm(x, wt[c].transpose(-2, -1), offs=offs)

                def loop(c, out=None):
                    w = wt[c]
                    for e, s0, s1 in spans:
                        q, s = ops.fp8_quantize_1x128(x[s0:s1])
                        y = ops.fp8_blockwise_linear(q, s, w.qdata[e], w.scale[e], None)
                        if out is not None:
                            out.append(y)

                def rowwise(c):
                    xq, sx = ops.fp8_quantize_rowwise(x)
                    return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), wt[c].qdata, ones, offs)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                n = int(offs[-1])
                y = ours(0)[:n]
                y_loop = []
                loop(0, y_loop)
                y_loop = torch.cat(y_loop)
                rec["vs_select_linear"] = "identical" if torch.equal(y.view(torch.int16), y_loop.view(torch.int16)) \
                    else sqnr_db(y_loop, y)
                rec["sqnr_vs_bf16_db"] = sqnr_db(bf16(0)[:n], y)
                rounds = 1 if T >= 2048 else None
                for key, fn, cp in (("ours", ours, copies), ("expert_loop", loop, copies), ("fp8_rowwise", rowwise, copies),
                                    ("bf16", bf16, copies_bf16)):
                    us = time_graph(fn, cp, a.replays, rounds)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                try:
                    xq, xs = ops.fp8_quantize_1x128(x)
                    F.scaled_grouped_mm(xq, wt[0].qdata.transpose(-2, -1), scale_a=xs[:, :M].t().contiguous(),
                                        scale_recipe_a=F.ScalingType.BlockWise1x128, scale_b=wt[0].scale,
                                        scale_recipe_b=F.ScalingType.BlockWise128x128, offs=offs,
                                        output_dtype=torch.bfloat16)
                    rec["torch_scaled_grouped_mm"] = "ran (not timed)"
                except Exception as e:   # the blockwise recipes need torch built for CUDA 12.9 or later
                    rec["torch_scaled_grouped_mm"] = (f"unavailable in torch {torch.__version__} (CUDA {torch.version.cuda}): "
                                                      f"{str(e).splitlines()[0][:160]}")
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del wt, wb, ones
        torch.cuda.empty_cache()


def measure_mx_prologue(a, ops, dev, lines):
    """Kernel time per call of the one-launch MX prologue (mx*_fakequant) and of the two launches it replaces:
    mx*_quantize with blocked scales, then the dequant_act_kernel of the dense MX linear (run on a 128-row weight; its
    GEMM is not counted), on the activations of every case of measure_mx, the two alternated call by call in one
    torch.profiler run.  main() turns PDL off for this mode (AO_B200_NO_PDL=1): a PDL kernel starts while the one
    before it still runs, and its time would include that wait."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from ao_b200.prototype.mx_formats import MXTensor

    fp4 = a.fmt == "mxfp4"
    elem = torch.float4_e2m1fn_x2 if fp4 else torch.float8_e4m3fn
    fq = ops.mxfp4_fakequant if fp4 else ops.mxfp8_fakequant
    quant, lin = (ops.mxfp4_quantize, ops.mxfp4_linear) if fp4 else (ops.mxfp8_quantize, ops.mxfp8_linear)
    reps = 20
    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        w = MXTensor.to_mx(torch.randn(128, K, device=dev, generator=g).to(torch.bfloat16), elem, 32,
                           is_swizzled_scales=True)
        w128, s128 = w.qdata, w.scale.view(torch.uint8)
        for T in TOKENS:
            for skewed in (False, True):
                M = sum(routing(T, E, topk, skewed, seed=T * 131 + E + skewed))
                x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
                for _ in range(2):   # warm-up outside the profile
                    fq(x)
                    lin(*quant(x, True), w128, s128, None)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        fq(x)
                        lin(*quant(x, True), w128, s128, None)
                    torch.cuda.synchronize()
                us = {"mx_fakequant_kernel": 0.0, "_quant_kernel": 0.0, "dequant_act_kernel": 0.0}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None)
                    t = e.cuda_time_total if t is None else t
                    for k in us:
                        if k in e.key:
                            us[k] += t / reps
                rec = dict(fmt=a.fmt, shape=name, K=K, tokens=T, routing="skewed" if skewed else "balanced", rows=M,
                           prologue_us=round(us["mx_fakequant_kernel"], 2), quantize_us=round(us["_quant_kernel"], 2),
                           dequant_us=round(us["dequant_act_kernel"], 2),
                           composition_us=round(us["_quant_kernel"] + us["dequant_act_kernel"], 2))
                print(json.dumps(rec), flush=True)
                lines.append(rec)


def measure_mx(a, ops, dev, lines):
    """The MX expert path (mx*_fakequant + mx*_grouped_mm) against the eager select + dense MX linear loop, the fp8
    rowwise path with its quantizer and bf16 torch._grouped_mm."""
    import torch

    from ao_b200.prototype.mx_formats import MXTensor

    fp4 = a.fmt == "mxfp4"
    elem = torch.float4_e2m1fn_x2 if fp4 else torch.float8_e4m3fn
    fq, gmm = (ops.mxfp4_fakequant, ops.mxfp4_grouped_mm) if fp4 else (ops.mxfp8_fakequant, ops.mxfp8_grouped_mm)
    quant, lin = (ops.mxfp4_quantize, ops.mxfp4_linear) if fp4 else (ops.mxfp8_quantize, ops.mxfp8_linear)
    for name, E, N, K, topk in SHAPES:
        g = torch.Generator(device=dev).manual_seed(E * N + K)
        w_bytes_expert = N * K // (2 if fp4 else 1) + N * K // 32
        copies = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * w_bytes_expert)) + 1)
        copies_bf16 = max(2, math.ceil(2 * L2_BYTES / (min(topk, E) * N * K * 2)) + 1)
        wm, ws, w8, s8, wb = [], [], [], [], []
        for c in range(max(copies, copies_bf16)):
            w = (torch.randn(E, N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
            if c < copies:
                t = MXTensor.to_mx(w, elem, 32, is_swizzled_scales=True)
                wm.append(t.qdata)
                ws.append(t.scale.view(torch.uint8))
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
                need = active * w_bytes_expert + M * K * 2 + M * N * 2 + E * 4
                rec = dict(fmt=a.fmt, shape=name, E=E, N=N, K=K, topk=topk, tokens=T,
                           routing="skewed" if skewed else "balanced", rows=M, active_experts=active, bytes=need,
                           weight_copies=copies, roofline_us=round(need / HBM_BPS * 1e6, 2))
                spans, start = [], 0
                for e, r in enumerate(rows):
                    if r:
                        spans.append((e, start, start + r))
                    start += r

                def ours(c):
                    return gmm(fq(x), wm[c], ws[c], offs)

                def loop(c, out=None):
                    for e, s0, s1 in spans:
                        q, s = quant(x[s0:s1], True)
                        y = lin(q, s, wm[c][e], ws[c][e], None)
                        if out is not None:
                            out.append(y)

                def fp8(c):
                    xq, sx = ops.fp8_quantize_rowwise(x)
                    return ops.fp8_rowwise_grouped_mm(xq, sx.reshape(-1), w8[c], s8[c], offs)

                def bf16(c):
                    return torch._grouped_mm(x, wb[c].transpose(-2, -1), offs=offs)

                n = int(offs[-1])
                y = ours(0)[:n]
                y_loop = []
                loop(0, y_loop)
                y_loop = torch.cat(y_loop)
                rec["vs_select_linear"] = "identical" if torch.equal(y.view(torch.int16), y_loop.view(torch.int16)) \
                    else sqnr_db(y_loop, y)
                rec["sqnr_vs_bf16_db"] = sqnr_db(bf16(0)[:n], y)
                rounds = 1 if T >= 2048 else None
                for key, fn, cp in (("ours", ours, copies), ("expert_loop", loop, copies), ("fp8", fp8, copies),
                                    ("bf16", bf16, copies_bf16)):
                    us = time_graph(fn, cp, a.replays, rounds)
                    rec[f"{key}_us"] = round(us, 2)
                    rec[f"{key}_GBps"] = round(need / us * 1e-3, 1)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
        del wm, ws, w8, s8, wb
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fmt", choices=["fp8", "nvfp4", "int4", "fp8wo", "int8wo", "int8", "fp8_blockwise", "mxfp8", "mxfp4"],
                    default="fp8")
    ap.add_argument("--group-size", type=int, choices=[32, 64, 128, 256], default=32)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--prologue", action="store_true", help="mxfp8 / mxfp4: the activation prologue alone (PDL off)")
    a = ap.parse_args()
    if a.prologue:
        os.environ["AO_B200_NO_PDL"] = "1"   # read once, when the library first launches
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
    if a.fmt == "int4":
        measure_int4(a, ops, dev, lines)
    if a.fmt == "fp8wo":
        measure_fp8wo(a, ops, dev, lines)
    if a.fmt in ("int8wo", "int8"):
        measure_int8(a, ops, dev, lines)
    if a.fmt == "fp8_blockwise":
        measure_fp8_blockwise(a, ops, dev, lines)
    if a.fmt in ("mxfp8", "mxfp4"):
        (measure_mx_prologue if a.prologue else measure_mx)(a, ops, dev, lines)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(info=info, cases=lines), f, indent=1)


if __name__ == "__main__":
    main()
