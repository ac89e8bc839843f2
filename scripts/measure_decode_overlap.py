#!/usr/bin/env python
"""Where the int4 decode step's time goes between consecutive GEMMs.

  python scripts/measure_decode_overlap.py [--runs 3] [--steps 200] [--out DIR]

Prints one JSON line with
  * `chain`: ms/step of the Llama-3-8B int4 g=32 stack (bench.build_stack, CUDA-graph replays as bench.py times them)
    at bs=1 and bs=32, with programmatic dependent launch (PDL) on and off (AO_B200_NO_PDL=1, read once per process),
    in alternating subprocesses;
  * `sweep`: single int4 GEMMs (the four fused projections and a K sweep at N=4096) at M in {1, 16, 32}, launched
    back to back from a CUDA graph on weight copies rotated past the L2, and per M the least-squares fit
    t = F + c * chunks_per_CTA (F: the fixed cost of one GEMM; c: the time of one 128-k chunk of a CTA's range);
  * `trace`: from a torch.profiler trace of one bs=1 replay (a run of its own), the start-to-start interval and the
    gap between the end of one `ts_gemm_kernel` and the start of the next (negative when the next one became
    resident under the previous one);
  * the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GROUP = 32
L2_BYTES = 50 * 2**20
SHAPES = [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336)]
K_SWEEP = [1024, 2048, 8192, 14336]   # N = 4096; K = 4096 is o


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip()


def chain_child(steps):
    import torch

    import bench
    from ao_b200.quantization import Int4WeightOnlyConfig

    dev = torch.device("cuda", 0)
    cfg = Int4WeightOnlyConfig(group_size=GROUP, int4_packing_format="tile_packed_to_4d")
    model = bench.build_stack("llama-3-8b", cfg, 32, dev)
    out = {}
    for bs in (1, 32):
        x = torch.randn(bs, 4096, device=dev, generator=torch.Generator(device=dev).manual_seed(1)).to(torch.bfloat16)
        graph, _, launches = bench.graph_of(model, x)
        out[f"bs{bs}"] = bench.time_replays(graph, steps, 20, torch.cuda.synchronize)
        out["launches"] = launches
    return out


def trace_child():
    import torch

    import bench
    from ao_b200.quantization import Int4WeightOnlyConfig

    dev = torch.device("cuda", 0)
    cfg = Int4WeightOnlyConfig(group_size=GROUP, int4_packing_format="tile_packed_to_4d")
    model = bench.build_stack("llama-3-8b", cfg, 32, dev)
    x = torch.randn(1, 4096, device=dev).to(torch.bfloat16)
    graph, _, _ = bench.graph_of(model, x)
    for _ in range(10):
        graph.replay()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        graph.replay()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if "ts_gemm_kernel" in e.name and e.device_type.name == "CUDA"),
                key=lambda e: e.time_range.start)
    starts = [e.time_range.start for e in ev]
    ends = [e.time_range.end for e in ev]
    step = [b - a for a, b in zip(starts, starts[1:])]
    gap = [b - a for a, b in zip(ends, starts[1:])]
    dur = [b - a for a, b in zip(starts, ends)]

    def summ(v):
        return {"median": statistics.median(v), "min": min(v), "max": max(v)} if v else None

    return {"kernels": len(ev), "start_to_start_us": summ(step), "end_to_start_gap_us": summ(gap),
            "duration_us": summ(dur), "span_us": (ends[-1] - starts[0]) if ev else None}


def sweep(iters):
    import torch

    import bench

    ops = torch.ops.ao_b200
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = [(name, n, k) for name, n, k in SHAPES] + [(f"k{k}", 4096, k) for k in K_SWEEP]
    out = {"cases": {}, "fit": {}}
    for M in (1, 16, 32):
        pts = []
        for name, N, K in cases:
            wbytes = N * K // 2 + (K // GROUP) * N * 4
            copies = max(2, -(-3 * L2_BYTES // wbytes))
            ws = [(torch.randint(-2**31, 2**31 - 1, (N // 8, K // 128, 32, 4), device=dev, dtype=torch.int32),
                   ((torch.rand(K // GROUP, N, 2, device=dev) - 0.5) * 0.004).to(torch.bfloat16)) for _ in range(copies)]
            x = torch.randn(M, K, device=dev).to(torch.bfloat16)
            launches = copies * max(1, 32 // copies)

            def run():
                for i in range(launches):
                    qd, sz = ws[i % copies]
                    ops.int4_tilepacked_linear(x, qd, GROUP, sz, None, N, 1)

            graph, _, _ = bench.graph_of(lambda _x: run(), x)
            us = bench.time_replays(graph, iters, 5, torch.cuda.synchronize) * 1e3 / launches
            units = (N // 128) * (K // 128)
            grid = min(sms, max(1, units // 4))
            cpc = units / grid
            pts.append((cpc, us))
            out["cases"][f"M{M}_{name}"] = {"us": us, "chunks_per_cta": cpc, "grid": grid}
            del ws, graph
            torch.cuda.empty_cache()
        n = len(pts)
        mx = sum(p[0] for p in pts) / n
        my = sum(p[1] for p in pts) / n
        c = sum((p[0] - mx) * (p[1] - my) for p in pts) / sum((p[0] - mx) ** 2 for p in pts)
        out["fit"][f"M{M}"] = {"F_us": my - c * mx, "c_us_per_chunk": c}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: stdout only)")
    ap.add_argument("--child", choices=["chain", "trace"], default=None)
    args = ap.parse_args()
    if args.child:
        import ao_b200  # noqa: F401
        print(json.dumps(chain_child(args.steps) if args.child == "chain" else trace_child()))
        return

    def child(kind, no_pdl):
        env = dict(os.environ)
        env.pop("AO_B200_NO_PDL", None)
        if no_pdl:
            env["AO_B200_NO_PDL"] = "1"
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", kind, "--steps", str(args.steps)],
                           env=env, stdout=subprocess.PIPE, text=True, check=True)
        return json.loads(r.stdout.strip().splitlines()[-1])

    res = {"card": card(), "chain": {"pdl": [], "no_pdl": []}}
    for _ in range(args.runs):
        res["chain"]["pdl"].append(child("chain", False))
        res["chain"]["no_pdl"].append(child("chain", True))
    res["trace"] = child("trace", False)
    import ao_b200  # noqa: F401
    res["sweep"] = sweep(args.steps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "decode_overlap.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
