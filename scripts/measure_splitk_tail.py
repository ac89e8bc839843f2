#!/usr/bin/env python
"""How much of the int4 decode GEMM's fixed cost comes from splitting tiles over CTAs (the owner's gather).

  python scripts/measure_splitk_tail.py [--steps 200] [--out DIR]

Single int4 GEMMs (g=32) at M in {1, 16, 32}, launched back to back from a CUDA graph on weight copies rotated past
the L2 (as scripts/measure_decode_overlap.py does), under three grids:
  * `normal`: the grid launch_gemm picks (132 CTAs on an H100 SXM for every Llama-3-8B projection);
  * `unsplit`: forced (ao_b200_debug_set_streamk_ctas) to n_tiles CTAs: every CTA computes one whole tile, no tile is
    split, nobody publishes or gathers a partial;
  * `split2`: forced to 2 x n_tiles: every tile is split in two, each owner gathers one contributor's partial.
Per grid and M, the least-squares fit t = F + c * chunks_per_CTA over a K sweep at N = 4096 (K = 1024 .. 14336; o is
K = 4096, down K = 14336) gives F, the fixed cost of one GEMM.  If F's growth from M = 1 to M = 32 is mostly a cost of
split tiles, it shows under `normal` and `split2` and not under `unsplit`.

Prints one JSON line: the card's name and power limit, per case the time and chunks per CTA, per grid and M the fit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_decode_overlap import GROUP, L2_BYTES, card  # noqa: E402

N_SWEEP = 4096
K_SWEEP = [1024, 2048, 4096, 8192, 14336]   # o = 4096 x 4096, down = 4096 x 14336
NAMED = [("qkv", 6144, 4096), ("gate_up", 28672, 4096)]   # their normal grid; qkv also unsplit (48 CTAs)
MS = (1, 16, 32)


def time_gemm(M, N, K, ctas, iters):
    """us per GEMM of [M, K] x [N, K]^T at grid `ctas` (0: the heuristic); returns (us, grid, chunks per CTA)"""
    import torch

    import bench

    ops = torch.ops.ao_b200
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
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

    units = (N // 128) * (K // 128)
    # the grid launch_gemm takes (ts_gemm.cuh): heuristic, or the forced count capped at units and the SM count
    grid = min(ctas, units, sms) if ctas else min(sms, max(1, units // 4))
    ops.debug_set_streamk_ctas(ctas)
    try:
        graph, _, _ = bench.graph_of(lambda _x: run(), x)
    finally:
        ops.debug_set_streamk_ctas(0)
    us = bench.time_replays(graph, iters, 5, torch.cuda.synchronize) * 1e3 / launches
    del ws, graph
    torch.cuda.empty_cache()
    return us, grid, units / grid


def fit(pts):
    n = len(pts)
    mx = sum(p[0] for p in pts) / n
    my = sum(p[1] for p in pts) / n
    c = sum((p[0] - mx) * (p[1] - my) for p in pts) / sum((p[0] - mx) ** 2 for p in pts)
    return {"F_us": my - c * mx, "c_us_per_chunk": c}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: stdout only)")
    args = ap.parse_args()

    import ao_b200  # noqa: F401

    n_tiles = N_SWEEP // 128
    grids = {"normal": 0, "unsplit": n_tiles, "split2": 2 * n_tiles}
    res = {"card": card(), "cases": {}, "fit": {}}
    for M in MS:
        for gname, ctas in grids.items():
            pts = []
            for K in K_SWEEP:
                us, grid, cpc = time_gemm(M, N_SWEEP, K, ctas, args.steps)
                res["cases"][f"M{M}_{gname}_{N_SWEEP}x{K}"] = {"us": us, "grid": grid, "chunks_per_cta": cpc}
                pts.append((cpc, us))
            res["fit"][f"M{M}_{gname}"] = fit(pts)
        for name, N, K in NAMED:
            for gname, ctas in [("normal", 0)] + ([("unsplit", N // 128)] if name == "qkv" else []):
                us, grid, cpc = time_gemm(M, N, K, ctas, args.steps)
                res["cases"][f"M{M}_{gname}_{name}"] = {"us": us, "grid": grid, "chunks_per_cta": cpc}
    line = json.dumps(res)
    print(line)
    for g in grids:
        f = [res["fit"][f"M{M}_{g}"] for M in MS]
        print(f"{g:8s} F(M=1/16/32) = " + " / ".join(f"{v['F_us']:.2f}" for v in f) + " us   c = "
              + " / ".join(f"{v['c_us_per_chunk']:.3f}" for v in f) + " us/chunk", file=sys.stderr)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "splitk_tail.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
