"""Per-linear time of NF4 weights (one launch: bf16 activations on NF4 codes, the double-quantized scalers decoded and
every weight dequantized in the kernel) against the reference's eager recipe (F.linear(x, t.get_original_weight()) + b),
the bf16 F.linear and int4 weight-only tile-packed g=64 (the nearest bytes per weight in this engine), on the
Llama-3-8B projections with bias, all from the same bf16 weights.

Each measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every call streams
its weights from HBM rather than the 50 MB L2; the formats alternate within one run.  Achieved GB/s counts the
algorithmic bytes (codes, scalers and factors, bias, activations in and out once); the bound is the larger of those bytes at
3.35 TB/s and the bf16 FLOPs at 989 TFLOP/s (H100 SXM data sheet, 700 W).  Changes no device setting; the card, its
power limit and its SM clocks are read in the same run and printed with the table.

    python scripts/measure_nf4.py [--reps 20] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}
TOKENS = (1, 32, 512, 4096)
L2_BYTES = 50 * 2**20
HBM_BPS, BF16_FLOPS = 3.35e12, 989e12
FMTS = ("nf4", "ref_eager", "bf16", "int4_g64")
# per weight: NF4 0.5 byte of code + 1/64 of an int8 scaler (+ a bf16 factor per 256 scalers); int4 g=64 0.5 + a bf16
# scale and zero per 64
BYTES_PER_PARAM = {"nf4": 0.5 + 1 / 64 + 2 / (64 * 256), "ref_eager": 0.5 + 1 / 64 + 2 / (64 * 256), "bf16": 2,
                   "int4_g64": 0.5 + 4 / 64}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power, sm, sm_max = (f.strip() for f in q.stdout.strip().splitlines()[0].split(","))
        return f"{name}, power limit {power}, SM clock {sm} (max {sm_max})"
    return torch.cuda.get_device_name(0)


def linear_of(w, b, fmt):
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import Int4PackingFormat, Int4WeightOnlyConfig, quantize_

    lin = nn.Linear(w.shape[1], w.shape[0], bias=True, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
        lin.bias.copy_(b)
    if fmt == "bf16":
        return lin
    config = {"nf4": NF4WeightOnlyConfig(), "ref_eager": NF4WeightOnlyConfig(),
              "int4_g64": Int4WeightOnlyConfig(group_size=64, int4_packing_format=Int4PackingFormat.TILE_PACKED_TO_4D)}[fmt]
    quantize_(lin, config)
    if fmt != "ref_eager":
        return lin
    t, bias = lin.weight, lin.bias

    def recipe(x):   # the reference's forward, op for op: the whole bf16 weight rebuilt, F.linear, then + bias
        return F.linear(x, t.get_original_weight()) + bias
    return recipe


def graph_of(fns, x):
    for f in fns:
        f(x)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for f in fns:
            f(x)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the rows as JSON to this file")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--tokens", default=",".join(map(str, TOKENS)))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_nf4.py needs a CUDA device"
    import ao_b200  # noqa: F401

    info = card()
    rows = []
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        torch.manual_seed(0)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        b = (torch.randn(N, device="cuda") * 0.02).to(torch.bfloat16)
        lins = {}
        for fmt in FMTS:
            copies = max(2, int(-(-2 * L2_BYTES // (N * K * BYTES_PER_PARAM[fmt]))) + 1)
            lins[fmt] = [linear_of(w, b, fmt) for _ in range(copies)]
        del w, b
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                graphs = {f: graph_of(lins[f], x) for f in FMTS}
                for g in graphs.values():
                    g.replay()
                torch.cuda.synchronize()
                times = {f: [] for f in FMTS}
                for _ in range(args.reps):
                    for f in FMTS:   # alternate the formats
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        graphs[f].replay()
                        b.record()
                        b.synchronize()
                        times[f].append(a.elapsed_time(b) * 1e-3 / len(lins[f]))
            for f in FMTS:
                ts = sorted(times[f])
                t = ts[len(ts) // 2]
                nbytes = N * K * BYTES_PER_PARAM[f] + N * 2 + M * K * 2 + M * N * 2
                t_hbm, t_flop = nbytes / HBM_BPS, 2.0 * M * N * K / BF16_FLOPS
                rows.append({"proj": name, "N": N, "K": K, "M": M, "fmt": f, "us": t * 1e6, "us_min": ts[0] * 1e6,
                             "us_max": ts[-1] * 1e6, "GB/s": nbytes / t / 1e9, "bound_us": max(t_hbm, t_flop) * 1e6,
                             "bound": "HBM" if t_hbm >= t_flop else "bf16 FLOP", "of_bound": max(t_hbm, t_flop) / t})
            del graphs
        del lins
        torch.cuda.empty_cache()
    print(f"# {info}")
    print(f"{'proj':8} {'M':>5} " + " ".join(f"{f:>22}" for f in FMTS) + "   (us, GB/s)   bound of nf4")
    for name in args.shapes.split(","):
        for M in map(int, args.tokens.split(",")):
            r = {x["fmt"]: x for x in rows if x["proj"] == name and x["M"] == M}
            print(f"{name:8} {M:5d} " + " ".join(f"{r[f]['us']:10.1f} {r[f]['GB/s']:9.0f}  " for f in FMTS)
                  + f"  {r['nf4']['bound_us']:.1f} us ({r['nf4']['bound']}), reached {100 * r['nf4']['of_bound']:.0f} %"
                  + f"  spread {max((x['us_max'] - x['us_min']) / x['us'] for x in r.values()) * 100:.0f} %")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
