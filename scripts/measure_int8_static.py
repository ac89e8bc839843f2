"""Per-linear time of static int8 activations (Int8StaticActivationInt8WeightConfig: one quantizer launch that applies the
pre-scale and the calibrated scale, then the int8 GEMM) with and without a bf16 ``act_pre_scale``, against the dynamic
int8 linear (per-token quantizer + the same GEMM) and the torch route a static Int8Tensor took before the quantizer
existed (x * act_pre_scale, Int8Tensor.from_hp with the static scale in eager torch, an expand().contiguous() of the
scale, then the same GEMM), on the Llama-3-8B projections, all from the same bf16 weights (PerRow weights, a PerTensor
activation scale).  The static quantizer alone is timed as well, and the static outputs are compared bit for bit with
the torch route's in the same run.

Each measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every call streams
its weights from HBM rather than the 50 MB L2; the formats alternate within one run.  Changes no device setting; the
card, its power limit and its SM clocks are read in the same run and printed with the table.

    python scripts/measure_int8_static.py [--reps 20] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}
TOKENS = (1, 32, 512)
L2_BYTES = 50 * 2**20
FMTS = ("static", "static_pre", "dynamic", "torch", "torch_pre", "quant_pre")
ACT_SCALE = 0.02


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power, sm, sm_max = (f.strip() for f in q.stdout.strip().splitlines()[0].split(","))
        return f"{name}, power limit {power}, SM clock {sm} (max {sm_max})"
    return torch.cuda.get_device_name(0)


def torch_route(w):
    """The torch route of a static symmetric Int8Tensor before the static quantizer, op for op."""
    from ao_b200.quantization import Int8Tensor

    def run(x):
        out_dtype, N, K = x.dtype, w.qdata.shape[0], w.qdata.shape[1]
        if w.act_pre_scale is not None:
            x = x * w.act_pre_scale
        x2 = x.reshape(-1, K)
        kw = w.act_quant_kwargs
        xt = Int8Tensor.from_hp(x2, kw.granularity, mapping_type=kw.mapping_type, scale=w.act_quant_scale,
                                zero_point=w.act_quant_zero_point, reduce_range=kw.reduce_range)
        xs = xt.scale.reshape(-1).float().expand(x2.shape[0])
        y = torch.ops.ao_b200.int8_dyn_linear(xt.qdata.contiguous(), xs.contiguous(), w.qdata.contiguous(),
                                              w.scale.reshape(-1).float().contiguous(), None)
        return y.reshape(*x.shape[:-1], N).to(out_dtype)
    return run


def linear_of(w, fmt, pre):
    from ao_b200.quantization import (Int8DynamicActivationInt8WeightConfig, Int8StaticActivationInt8WeightConfig,
                                      PerRow, PerTensor, quantize_)

    lin = nn.Linear(w.shape[1], w.shape[0], bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
    if fmt == "dynamic":
        quantize_(lin, Int8DynamicActivationInt8WeightConfig())
        return lin
    quantize_(lin, Int8StaticActivationInt8WeightConfig(act_quant_scale=torch.tensor([[ACT_SCALE]], device="cuda"),
                                                        granularity=[PerTensor(), PerRow()]))
    if fmt.endswith("_pre"):
        lin.weight.act_pre_scale = pre
    if fmt.startswith("torch"):
        return torch_route(lin.weight)
    if fmt == "quant_pre":
        q = lin.weight
        return lambda x: torch.ops.ao_b200.int8_quantize_static(x, q.act_quant_scale, None, q.act_pre_scale, -128, 127)
    return lin


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
    assert torch.cuda.is_available(), "measure_int8_static.py needs a CUDA device"
    import ao_b200  # noqa: F401

    info = card()
    rows, exact = [], []
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        torch.manual_seed(0)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        pre = (torch.rand(K, device="cuda") + 0.5).to(torch.bfloat16)   # 1 / smoothing factor
        copies = max(2, -(-2 * L2_BYTES // (N * K)) + 1)
        lins = {f: [linear_of(w, f, pre) for _ in range(copies if f != "quant_pre" else 8)] for f in FMTS}
        del w
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                for a, b in (("static", "torch"), ("static_pre", "torch_pre")):
                    same = torch.equal(lins[a][0](x).view(torch.int16), lins[b][0](x).view(torch.int16))
                    exact.append({"proj": name, "M": M, "pair": f"{a} == {b}", "bit_exact": same})
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
                rows.append({"proj": name, "N": N, "K": K, "M": M, "fmt": f, "us": ts[len(ts) // 2] * 1e6,
                             "us_min": ts[0] * 1e6, "us_max": ts[-1] * 1e6})
            del graphs
        del lins
        torch.cuda.empty_cache()
    print(f"# {info}")
    print(f"{'proj':8} {'M':>5} " + " ".join(f"{f:>11}" for f in FMTS) + "   (us per linear, median)")
    for name in args.shapes.split(","):
        for M in map(int, args.tokens.split(",")):
            r = {x["fmt"]: x for x in rows if x["proj"] == name and x["M"] == M}
            print(f"{name:8} {M:5d} " + " ".join(f"{r[f]['us']:11.2f}" for f in FMTS))
    bad = [e for e in exact if not e["bit_exact"]]
    print(f"# static vs torch route: {len(exact) - len(bad)} / {len(exact)} comparisons bit-exact", bad or "")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows, "bit_exact": exact}, fh, indent=1)
    return 0 if not bad else 1


if __name__ == "__main__":
    sys.exit(main())
