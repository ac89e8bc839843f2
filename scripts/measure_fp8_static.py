"""Per-linear time of static e4m3 activations (Float8StaticActivationFloat8WeightConfig, PerTensor: one quantizer launch
with the calibrated scale, then the e4m3 GEMM), with and without the output fake-quant fused into the GEMM's epilogue,
against the dynamic fp8 linears of this engine (Float8DynamicActivationFloat8WeightConfig, PerTensor and PerRow) and the
reference's recipe on the same codes (the torch quantize ops, torch._scaled_mm, then the torch ops of the output
fake-quant), on the Llama-3-8B projections, all from the same bf16 weights.  The static quantizer alone is timed as
well.

In the same run, before timing each token count, the static weights are given the dynamic per-tensor quantizer's own
scale for that input, and the outputs are compared bit for bit: static with dynamic PerTensor, and static with the
output fake-quant with the reference's fake-quant ops applied to the static output.  The reference recipe's largest
difference from the static fake-quant output is reported (torch._scaled_mm sums in its own order).

Each measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every call streams
its weights from HBM rather than the 50 MB L2; the columns alternate within one run.  Changes no device setting; the
card, its power limit and its SM clocks are read in the same run and printed with the table.

    python scripts/measure_fp8_static.py [--reps 20] [--out results.json]
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
FMTS = ("static", "static_qdq", "dyn_tensor", "dyn_row", "reference", "quant")
E4M3 = torch.float8_e4m3fn


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power, sm, sm_max = (f.strip() for f in q.stdout.strip().splitlines()[0].split(","))
        return f"{name}, power limit {power}, SM clock {sm} (max {sm_max})"
    return torch.cuda.get_device_name(0)


def ref_qdq(y, so):
    return ((y.float() / so).clamp(-448.0, 448.0).to(E4M3).float() * so).to(y.dtype)


def reference_recipe(w):
    """The reference's PerTensor recipe op for op (prototype_float8_tensor.py:329-474) on the static weight's codes."""
    def run(x):
        s = w.act_quant_scale
        xq = (x.float() / s).clamp(-448.0, 448.0).to(E4M3)
        y = torch._scaled_mm(xq, w.qdata.t(), s.reshape(()), w.scale.reshape(()), out_dtype=torch.bfloat16,
                             use_fast_accum=True)
        return ref_qdq(y, w.output_act_quant_scale)
    return run


def linear_of(w, fmt, act_scale, out_scale):
    from ao_b200.quantization import (Float8DynamicActivationFloat8WeightConfig, Float8StaticActivationFloat8WeightConfig,
                                      PerRow, PerTensor, quantize_)

    lin = nn.Linear(w.shape[1], w.shape[0], bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
    if fmt.startswith("dyn"):
        quantize_(lin, Float8DynamicActivationFloat8WeightConfig(granularity=PerTensor() if fmt == "dyn_tensor"
                                                                 else PerRow()))
        return lin
    # every static copy shares the calibrated scale tensors, so that one copy_ sets them all
    quantize_(lin, Float8StaticActivationFloat8WeightConfig(
        act_quant_scale=act_scale, output_act_quant_scale=out_scale if fmt in ("static_qdq", "reference") else None))
    lin.weight.act_quant_scale = act_scale
    if lin.weight.output_act_quant_scale is not None:
        lin.weight.output_act_quant_scale = out_scale
    if fmt == "reference":
        return reference_recipe(lin.weight)
    if fmt == "quant":
        return lambda x: torch.ops.ao_b200.fp8_quantize_static(x, act_scale)
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
    assert torch.cuda.is_available(), "measure_fp8_static.py needs a CUDA device"
    import ao_b200  # noqa: F401
    from ao_b200.quantization import Float8Tensor, PerTensor

    info = card()
    rows, exact = [], []
    act_scale = torch.tensor([[0.01]], device="cuda")
    out_scale = torch.tensor([[0.5 / 448]], device="cuda")
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        torch.manual_seed(0)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        copies = max(2, -(-2 * L2_BYTES // (N * K)) + 1)
        lins = {f: [linear_of(w, f, act_scale, out_scale) for _ in range(copies if f != "quant" else 8)] for f in FMTS}
        del w
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                act_scale.copy_(Float8Tensor.from_hp(x, E4M3, PerTensor()).scale.reshape(1, 1))
                st, sq, dt = lins["static"][0](x), lins["static_qdq"][0](x), lins["dyn_tensor"][0](x)
                rf = lins["reference"][0](x)
                exact.append({"proj": name, "M": M, "pair": "static == dyn_tensor",
                              "bit_exact": torch.equal(st.view(torch.int16), dt.view(torch.int16))})
                exact.append({"proj": name, "M": M, "pair": "static_qdq == ref_qdq(static)",
                              "bit_exact": torch.equal(sq.view(torch.int16), ref_qdq(st, out_scale).view(torch.int16))})
                ref_diff = float((rf.float() - sq.float()).abs().max())
                graphs = {f: graph_of(lins[f], x) for f in FMTS}
                for g in graphs.values():
                    g.replay()
                torch.cuda.synchronize()
                times = {f: [] for f in FMTS}
                for _ in range(args.reps):
                    for f in FMTS:   # alternate the columns
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        graphs[f].replay()
                        b.record()
                        b.synchronize()
                        times[f].append(a.elapsed_time(b) * 1e-3 / len(lins[f]))
            for f in FMTS:
                ts = sorted(times[f])
                rows.append({"proj": name, "N": N, "K": K, "M": M, "fmt": f, "us": ts[len(ts) // 2] * 1e6,
                             "us_min": ts[0] * 1e6, "us_max": ts[-1] * 1e6, "ref_max_abs_diff": ref_diff})
            del graphs
        del lins
        torch.cuda.empty_cache()
    print(f"# {info}")
    print(f"{'proj':8} {'M':>5} " + " ".join(f"{f:>11}" for f in FMTS) + "   (us per linear, median)  ref-vs-qdq max|d|")
    for name in args.shapes.split(","):
        for M in map(int, args.tokens.split(",")):
            r = {x["fmt"]: x for x in rows if x["proj"] == name and x["M"] == M}
            print(f"{name:8} {M:5d} " + " ".join(f"{r[f]['us']:11.2f}" for f in FMTS)
                  + f"   {r['static']['ref_max_abs_diff']:.3g}")
    bad = [e for e in exact if not e["bit_exact"]]
    print(f"# bit-exact pairs: {len(exact) - len(bad)} / {len(exact)}", bad or "")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows, "bit_exact": exact}, fh, indent=1)
    return 0 if not bad else 1


if __name__ == "__main__":
    sys.exit(main())
