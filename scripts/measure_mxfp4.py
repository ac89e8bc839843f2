"""Per-GEMM time of the mxfp4 linear against mxfp8 and nvfp4 of this library and against the reference's only Hopper
path for mxfp4 (dequantize() both operands in eager torch, then a bf16 F.linear), on the Llama-3-8B projections.

Each format runs the whole dynamic-activation linear (activation quantizer + GEMM) on the same bf16 weights.  Each
measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every call streams
its weights from HBM rather than the 50 MB L2; the formats alternate within one run.  Achieved GB/s counts the
algorithmic bytes (weights with their scales, activations in and out once); the bound term is the larger of those bytes
at 3.35 TB/s and the bf16 FLOPs at 989 TFLOP/s (H100 SXM data sheet, 700 W).

    python scripts/measure_mxfp4.py [--reps 20] [--out results.json]
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
# weight bytes per parameter: codes plus scales
BYTES_PER_PARAM = {"mxfp4": 0.5 + 1 / 32, "mxfp8": 1 + 1 / 32, "nvfp4": 0.5 + 1 / 16, "ref_dequant_bf16": 0.5 + 1 / 32}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def quantized(w, fmt):
    from ao_b200.prototype.mx_formats import MXDynamicActivationMXWeightConfig, NVFP4DynamicActivationNVFP4WeightConfig
    from ao_b200.quantization import quantize_

    lin = nn.Linear(w.shape[1], w.shape[0], bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
    fp4 = torch.float4_e2m1fn_x2
    cfg = {"mxfp4": MXDynamicActivationMXWeightConfig(activation_dtype=fp4, weight_dtype=fp4),
           "ref_dequant_bf16": MXDynamicActivationMXWeightConfig(activation_dtype=fp4, weight_dtype=fp4),
           "mxfp8": MXDynamicActivationMXWeightConfig(),
           "nvfp4": NVFP4DynamicActivationNVFP4WeightConfig()}[fmt]
    quantize_(lin, cfg)
    if fmt != "ref_dequant_bf16":
        return lin
    from ao_b200.prototype.mx_formats import MXTensor

    wq = lin.weight

    def emulated(x):   # the reference's KernelPreference.EMULATED: both operands dequantized, bf16 matmul
        xq = MXTensor.to_mx(x, fp4)
        return F.linear(xq.dequantize(torch.bfloat16), wq.dequantize(torch.bfloat16))
    return emulated


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
    assert torch.cuda.is_available(), "measure_mxfp4.py needs a CUDA device"
    import ao_b200  # noqa: F401

    info = card()
    rows = []
    fmts = ("mxfp4", "mxfp8", "nvfp4", "ref_dequant_bf16")
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        torch.manual_seed(0)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        lins = {}
        for fmt in fmts:
            copies = max(2, -(-2 * L2_BYTES // int(N * K * BYTES_PER_PARAM[fmt])) + 1)
            lins[fmt] = [quantized(w, fmt) for _ in range(copies)]
        del w
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                graphs = {f: graph_of(lins[f], x) for f in fmts}
                for g in graphs.values():
                    g.replay()
                torch.cuda.synchronize()
                times = {f: [] for f in fmts}
                for _ in range(args.reps):
                    for f in fmts:   # alternate the formats
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        graphs[f].replay()
                        b.record()
                        b.synchronize()
                        times[f].append(a.elapsed_time(b) * 1e-3 / len(lins[f]))
            for f in fmts:
                t = sorted(times[f])[len(times[f]) // 2]
                nbytes = N * K * BYTES_PER_PARAM[f] + M * K * 2 + M * N * 2
                bound = max(nbytes / HBM_BPS, 2.0 * M * N * K / BF16_FLOPS)
                rows.append({"proj": name, "N": N, "K": K, "M": M, "fmt": f, "us": t * 1e6, "GB/s": nbytes / t / 1e9,
                             "bound_us": bound * 1e6, "bound": "HBM" if nbytes / HBM_BPS >= 2.0 * M * N * K / BF16_FLOPS else "bf16 FLOP",
                             "of_bound": bound / t})
            del graphs
        del lins
        torch.cuda.empty_cache()
    print(f"# {info}")
    print(f"{'proj':8} {'M':>5} " + " ".join(f"{f:>22}" for f in fmts) + "   (us, GB/s)")
    for name in args.shapes.split(","):
        for M in map(int, args.tokens.split(",")):
            r = {x["fmt"]: x for x in rows if x["proj"] == name and x["M"] == M}
            print(f"{name:8} {M:5d} " + " ".join(f"{r[f]['us']:10.1f} {r[f]['GB/s']:9.0f}  " for f in fmts)
                  + f"  bound {r['mxfp4']['bound_us']:.1f} us ({r['mxfp4']['bound']})")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
