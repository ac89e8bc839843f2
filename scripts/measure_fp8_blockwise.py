"""Per-linear time of blockwise fp8 (Float8DynamicActivationFloat8WeightConfig with [PerBlock([1, 128]),
PerBlock([128, 128])]: the 1x128 quantizer + the blockwise e4m3 GEMM) against this engine's rowwise fp8 linear on the
same weights (per-token quantizer + the rowwise e4m3 GEMM: the same weight bytes, N x K / 16384 fewer scales), the
bf16 F.linear, and torch._scaled_mm with blockwise scales where the installed torch accepts it on this GPU (probed
once), on the Llama-3-8B projections and the DeepSeek-V3 dense-MLP shapes; then a Llama-3-8B linear-stack step
(q|k|v, o, gate|up, down of 32 layers) as a CUDA graph at batch 32 and 1, blockwise against rowwise.

Each per-linear measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every
call streams its weights from HBM rather than the 50 MB L2; CUDA events time --reps replays (each one launch per
copy) after a warm-up, and the arms alternate within the run.  Outputs are compared at every timed size: the
quantized arms against bf16 (SQNR, dB) and blockwise against rowwise and against torch._scaled_mm.  Changes no device
setting; the card and its power limit are read in the same run and printed with the table.

    python scripts/measure_fp8_blockwise.py [--reps 200] [--out results.json]
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

SHAPES = {"l3_qkv": (6144, 4096), "l3_o": (4096, 4096), "l3_gate_up": (28672, 4096), "l3_down": (4096, 14336),
          "dsv3_gate_up": (36864, 7168), "dsv3_down": (7168, 18432)}
TOKENS = (1, 4, 16, 32, 128, 512, 4096)
L2_BYTES = 50 * 2**20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power, sm_max = (f.strip() for f in q.stdout.strip().splitlines()[0].split(","))
        return f"{name}, power limit {power}, max SM clock {sm_max}"
    return torch.cuda.get_device_name(0)


def config(fmt):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerBlock, PerRow

    if fmt == "blockwise":
        return Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])])
    return Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())


def linear_of(w, fmt):
    from ao_b200.quantization import quantize_

    lin = nn.Linear(w.shape[1], w.shape[0], bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
    if fmt != "bf16":
        quantize_(lin, config(fmt))
    return lin


def scaled_mm_blockwise(lin):
    """torch._scaled_mm on the blockwise weight's codes and scales with the activations' 1x128 codes and scales, or None
    when the installed torch rejects blockwise scales on this GPU"""
    w = lin.weight
    from ao_b200.quantization import Float8Tensor, PerBlock

    def run(x):
        xt = Float8Tensor.from_hp(x, granularity=PerBlock([1, 128]))
        # scale_a outer-dim-major [M, K/128], scale_b [K/128, N/128] transposed views, as torch's blockwise path takes
        return torch._scaled_mm(xt.qdata, w.qdata.t(), xt.scale.t().contiguous().t(), w.scale.t(),
                                out_dtype=torch.bfloat16)
    try:
        y = run(torch.randn(256, w.shape[1], device="cuda", dtype=torch.bfloat16))
        torch.cuda.synchronize()
        return run if y.shape == (256, w.shape[0]) else None
    except Exception as e:   # noqa: BLE001  (the probe: any rejection means "not available")
        print(f"# torch._scaled_mm with blockwise scales: not available ({type(e).__name__}: {str(e).splitlines()[0][:160]})")
        return None


def graph_of(fns, x):
    for f in fns:
        f(x)   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = [f(x) for f in fns]
    return g, outs[0]


def time_alternating(graphs, reps, per):
    """median seconds per call of each graph (alternating), over reps replays after two warm-up replays"""
    for g in graphs.values():
        g.replay()
        g.replay()
    torch.cuda.synchronize()
    times = {k: [] for k in graphs}
    for _ in range(reps):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) * 1e-3 / per[k])
    out = {}
    for k, ts in times.items():
        ts = sorted(ts)
        out[k] = (ts[len(ts) // 2], ts[0], ts[-1])
    return out


def sqnr(ref, y):
    ref, y = ref.float(), y.float()
    return float(20 * torch.log10(ref.norm() / (ref - y).norm().clamp_min(1e-30)))


def per_linear(args, rows):
    probe_done, smm_ok = False, False
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        torch.manual_seed(0)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        lins = {}
        for fmt, nbytes in (("blockwise", 1), ("rowwise", 1), ("bf16", 2)):
            copies = max(2, -(-2 * L2_BYTES // (N * K * nbytes)) + 1)
            lins[fmt] = [linear_of(w, fmt) for _ in range(copies)]
        del w
        fns = {k: v for k, v in lins.items()}
        if not probe_done:
            smm_ok, probe_done = scaled_mm_blockwise(lins["blockwise"][0]) is not None, True
        if smm_ok:
            fns["scaled_mm"] = [scaled_mm_blockwise(l) for l in lins["blockwise"]]
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                built = {k: graph_of(v, x) for k, v in fns.items()}
                t = time_alternating({k: g for k, (g, _) in built.items()}, args.reps, {k: len(v) for k, v in fns.items()})
                y = {k: o for k, (_, o) in built.items()}
                r = {"shape": name, "N": N, "K": K, "M": M, "us": {k: v[0] * 1e6 for k, v in t.items()},
                     "spread": {k: (v[2] - v[1]) / v[0] for k, v in t.items()},
                     "sqnr_vs_bf16": {k: sqnr(y["bf16"], y[k]) for k in y if k != "bf16"},
                     "sqnr_blockwise_vs_rowwise": sqnr(y["rowwise"], y["blockwise"])}
                if "scaled_mm" in y:
                    r["max_abs_blockwise_vs_scaled_mm"] = float((y["blockwise"].float() - y["scaled_mm"].float()).abs().max())
                rows.append(r)
            del built, y
        del lins, fns
        torch.cuda.empty_cache()
    if not smm_ok:
        print("# torch._scaled_mm with blockwise scales: not available")


def stack_step(args):
    """Llama-3-8B's linears of 32 layers (q|k|v and gate|up fused) as one CUDA graph per format, alternating"""
    layers = {"blockwise": [], "rowwise": []}
    torch.manual_seed(1)
    for _ in range(32):
        ws = [(torch.randn(n, k, device="cuda") * 0.02).to(torch.bfloat16) for n, k in
              ((6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336))]
        for fmt in layers:
            layers[fmt].append([linear_of(w, fmt) for w in ws])
        del ws

    def step(ls):
        def f(h):
            for qkv, o, gu, down in ls:
                a = o(qkv(h)[:, :4096])
                g = gu(a)
                h = down(F.silu(g[:, :14336]) * g[:, 14336:])
                h = h * torch.rsqrt(h.float().pow(2).mean(-1, keepdim=True) + 1e-6).to(h.dtype)   # keeps 32 layers finite
            return h
        return f
    out = []
    for bs in (32, 1):
        x = (torch.randn(bs, 4096, device="cuda") * 0.5).to(torch.bfloat16)
        with torch.no_grad():
            built = {k: graph_of([step(v)], x) for k, v in layers.items()}
            t = time_alternating({k: g for k, (g, _) in built.items()}, args.reps, {k: 1 for k in built})
            y = {k: o for k, (_, o) in built.items()}
        out.append({"bs": bs, "ms": {k: v[0] * 1e3 for k, v in t.items()}, "spread": {k: (v[2] - v[1]) / v[0] for k, v in t.items()},
                    "sqnr_blockwise_vs_rowwise": sqnr(y["rowwise"], y["blockwise"])})
        del built
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--tokens", default=",".join(map(str, TOKENS)))
    ap.add_argument("--no-stack", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_fp8_blockwise.py needs a CUDA device"
    import ao_b200  # noqa: F401

    info = card()
    print(f"# {info}")
    rows = []
    per_linear(args, rows)
    arms = [a for a in ("blockwise", "rowwise", "bf16", "scaled_mm") if a in rows[0]["us"]]
    print(f"{'shape':13} {'M':>5} " + " ".join(f"{a:>10}" for a in arms)
          + "   (us per linear)  blockwise/rowwise  SQNR vs bf16: blockwise rowwise (dB)  max spread")
    for r in rows:
        print(f"{r['shape']:13} {r['M']:5d} " + " ".join(f"{r['us'][a]:10.1f}" for a in arms)
              + f"   {r['us']['blockwise'] / r['us']['rowwise']:17.3f}  {r['sqnr_vs_bf16']['blockwise']:10.1f}"
              f" {r['sqnr_vs_bf16']['rowwise']:7.1f}   {100 * max(r['spread'].values()):5.0f} %")
    stack = [] if args.no_stack else stack_step(args)
    for s in stack:
        print(f"# Llama-3-8B 32-layer linear stack, bs={s['bs']}: blockwise {s['ms']['blockwise']:.3f} ms, rowwise "
              f"{s['ms']['rowwise']:.3f} ms (x{s['ms']['blockwise'] / s['ms']['rowwise']:.3f}), SQNR blockwise vs "
              f"rowwise {s['sqnr_blockwise_vs_rowwise']:.1f} dB, spread {100 * max(s['spread'].values()):.0f} %")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows, "stack": stack}, fh, indent=1)


if __name__ == "__main__":
    main()
