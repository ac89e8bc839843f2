"""Time torch.bmm on rowwise e4m3 expert weights at Llama-4-Scout expert shapes (E = 16, D = 5120, F = 8192:
w1 / w3 [16, 5120, 8192], w2 [16, 8192, 5120]) for M tokens per expert, four ways:

  bnk    this engine, w the transposed view of a stored [B, N, K] weight (grouped e4m3 kernel)
  bkn    this engine, w stored [B, K, N] (N-major kernel: each weight tile transposed on chip)
  torch  the reference's recipe in torch ops: the rowwise activation quantizer, the transposed copy
         w.transpose(-2, -1).contiguous() of the [B, K, N] codes, then F.scaled_grouped_mm
  bf16   torch.bmm on the bf16 weights

Each path runs as a CUDA graph of `reps` calls, timed with CUDA events over `iters` replays after a warm-up.  One fp8
weight set is 671 MB and one bf16 set 1.3 GB, over 13x the 50 MB L2, so every call streams its weights from HBM.
Prints the card's name and power limit, then one JSON line per (shape, M).

    python scripts/measure_fp8_bmm.py [--iters 20] [--reps 5] [--out fp8_bmm.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"w1/w3": (5120, 8192), "w2": (8192, 5120)}   # (K, N)
E = 16
TOKENS = [1, 8, 32, 128, 2048]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "power limit unknown"
    return name, q


def timed(fn, iters, reps):
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for _ in range(reps):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (iters * reps)   # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_fp8_bmm.py needs a CUDA device"
    import ao_b200  # noqa: F401
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow, quantize_

    ops = torch.ops.ao_b200
    name, limit = card()
    print(f"card: {name} ({limit})")
    rows = []
    for label, (K, N) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(K)
        w_bf16 = (torch.randn(E, K, N, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)

        class Holder(torch.nn.Module):
            def __init__(self, w):
                super().__init__()
                self.weight = torch.nn.Parameter(w, requires_grad=False)

        kn = Holder(w_bf16.clone())
        quantize_(kn, Float8DynamicActivationFloat8WeightConfig(granularity=[PerRow(), PerRow(1)]),
                  filter_fn=lambda *_: True)
        w_kn = kn.weight                                   # stored [E, K, N]
        nk = Holder(w_bf16.transpose(-2, -1).contiguous())
        quantize_(nk, Float8DynamicActivationFloat8WeightConfig(granularity=PerRow()), filter_fn=lambda *_: True)
        w_nk = nk.weight.transpose(-2, -1)                 # view of a stored [E, N, K]
        sw = w_kn.scale.reshape(E, N).float().contiguous()
        for M in TOKENS:
            x = torch.randn(E, M, K, device="cuda", generator=g).to(torch.bfloat16)
            offs = torch.arange(M, M * (E + 1), M, device="cuda", dtype=torch.int32)

            def torch_recipe():
                xq, sx = ops.fp8_quantize_rowwise(x.reshape(E * M, K))
                wt = w_kn.qdata.transpose(-2, -1).contiguous()   # the reference's transposed copy, [E, N, K]
                return F.scaled_grouped_mm(xq, wt.transpose(-2, -1), scale_a=sx.reshape(-1),
                                           scale_recipe_a=F.ScalingType.RowWise, scale_b=sw,
                                           scale_recipe_b=F.ScalingType.RowWise, offs=offs,
                                           output_dtype=torch.bfloat16)

            paths = {"bnk": lambda: torch.bmm(x, w_nk), "bkn": lambda: torch.bmm(x, w_kn), "torch": torch_recipe,
                     "bf16": lambda: torch.bmm(x, w_bf16)}
            y_kn, y_nk = paths["bkn"](), paths["bnk"]()
            assert torch.equal(y_kn.view(torch.int16), y_nk.view(torch.int16)), (label, M)
            res = {"shape": label, "E": E, "M": M, "K": K, "N": N, "card": name, "power": limit}
            for p, fn in paths.items():
                try:
                    res[f"{p}_us"] = round(timed(fn, args.iters, args.reps), 2)
                except (RuntimeError, NotImplementedError) as e:
                    res[f"{p}_us"] = None
                    res[f"{p}_error"] = str(e).splitlines()[0][:160]
            if res["bnk_us"] and res["bkn_us"]:
                res["bkn_over_bnk"] = round(res["bkn_us"] / res["bnk_us"], 3)
                res["fp8_weight_GBps_bkn"] = round(E * K * N / (res["bkn_us"] * 1e3), 1)
            print(json.dumps(res), flush=True)
            rows.append(res)
            del x
        del w_bf16, kn, nk, w_kn, w_nk
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
