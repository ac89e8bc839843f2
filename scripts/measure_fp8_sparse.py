"""Per-linear time of 2:4-sparse fp8 (Float8DynamicActivationFloat8WeightConfig, packing_format
SPARSE_2D_DATA_2D_METADATA: the per-token quantizer + the sparse e4m3 GEMM) against this engine's dense rowwise fp8
linear on the same pruned weights (the same quantizer + the dense e4m3 GEMM), the bf16 F.linear, and the reference's
own CUTLASS sparse GEMM (oracle/_ref, built by oracle/ref_sparse.py; skipped with a note when it is not built) fed
the same codes, on the Llama-3-8B projections at 1, 4, 16, 32, 128, 512 and 4096 tokens.

Each measurement is a CUDA graph that runs the linear once on each of several weight copies, so that every call
streams its weights from HBM rather than the 50 MB L2; CUDA events time --reps replays after a warm-up, and the arms
alternate within the run (helpers of measure_fp8_blockwise.py).  Outputs are compared at every timed size: SQNR of
each quantized arm against bf16 on the pruned weights, and the largest |sparse - reference GEMM|.  Changes no device
setting; the card and its power limit are read in the same run and printed with the table.

    python scripts/measure_fp8_sparse.py [--reps 100] [--out results.json]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_fp8_blockwise import L2_BYTES, card, graph_of, sqnr, time_alternating  # noqa: E402

SHAPES = {"l3_qkv": (6144, 4096), "l3_o": (4096, 4096), "l3_gate_up": (28672, 4096), "l3_down": (4096, 14336)}
TOKENS = (1, 4, 16, 32, 128, 512, 4096)


def config(fmt):
    from ao_b200.quantization import Float8DynamicActivationFloat8WeightConfig, Float8PackingFormat, PerRow

    if fmt == "sparse":
        return Float8DynamicActivationFloat8WeightConfig(granularity=PerRow(),
                                                         packing_format=Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA)
    return Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())


def linear_of(w, fmt):
    from ao_b200.quantization import quantize_

    lin = nn.Linear(w.shape[1], w.shape[0], bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(w)
    if fmt != "bf16":
        quantize_(lin, config(fmt))
    return lin


def reference_gemm():
    """a function lin -> (x -> y) running the reference's sparse GEMM on the sparse weight, or None"""
    from oracle import ref_sparse

    try:
        ref = ref_sparse.load()
    except FileNotFoundError as e:
        print(f"# reference CUTLASS sparse GEMM: not built ({e})")
        return None
    from ao_b200.quantization import Float8Tensor, PerRow

    def make(lin):
        w = lin.weight

        def run(x):
            xt = Float8Tensor.from_hp(x, granularity=PerRow())
            return ref.rowwise_scaled_linear_sparse_cutlass_f8f8(xt.qdata, xt.scale.reshape(-1), w.qdata,
                                                                  w.sparse_metadata, w.scale.reshape(-1), None,
                                                                  torch.bfloat16)
        return run
    return make


def pruned(N, K, g):
    w = torch.randn(N, K, device="cuda", generator=g) * 0.02
    idx = torch.rand(N, K // 4, 4, device="cuda", generator=g).argsort(-1)[..., :2]
    mask = torch.zeros(N, K // 4, 4, dtype=torch.bool, device="cuda").scatter_(-1, idx, True).reshape(N, K)
    return (w * mask).to(torch.bfloat16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--tokens", default=",".join(map(str, TOKENS)))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import ao_b200  # noqa: F401

    print(f"# {card()}")
    make_ref = reference_gemm()
    rows = []
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        w = pruned(N, K, torch.Generator(device="cuda").manual_seed(0))
        lins = {}
        for fmt, nbytes in (("sparse", 0.625), ("rowwise", 1), ("bf16", 2)):
            copies = max(2, int(-(-2 * L2_BYTES // (N * K * nbytes))) + 1)
            lins[fmt] = [linear_of(w, fmt) for _ in range(copies)]
        del w
        fns = dict(lins)
        if make_ref is not None:
            fns["reference"] = [make_ref(l) for l in lins["sparse"]]
        for M in map(int, args.tokens.split(",")):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            with torch.no_grad():
                built = {k: graph_of(v, x) for k, v in fns.items()}
                t = time_alternating({k: g for k, (g, _) in built.items()}, args.reps,
                                     {k: len(v) for k, v in fns.items()})
                y = {k: o for k, (_, o) in built.items()}
                r = {"shape": name, "N": N, "K": K, "M": M, "us": {k: v[0] * 1e6 for k, v in t.items()},
                     "spread": {k: (v[2] - v[1]) / v[0] for k, v in t.items()},
                     "sqnr_vs_bf16": {k: sqnr(y["bf16"], y[k]) for k in y if k != "bf16"}}
                if "reference" in y:
                    r["max_abs_sparse_vs_reference"] = float((y["sparse"].float() - y["reference"].float()).abs().max())
                rows.append(r)
            del built, y
        del lins, fns
        torch.cuda.empty_cache()
    head = f"{'shape':>11} {'M':>5} {'sparse us':>10} {'rowwise':>8} {'bf16':>8} {'ref':>8} {'sp/row':>7} {'sp/ref':>7} " \
           f"{'SQNR sp':>8} {'SQNR row':>8} {'|sp-ref|':>9}"
    print(head)
    for r in rows:
        us = r["us"]
        ref = us.get("reference", float("nan"))
        print(f"{r['shape']:>11} {r['M']:>5} {us['sparse']:>10.1f} {us['rowwise']:>8.1f} {us['bf16']:>8.1f} {ref:>8.1f} "
              f"{us['sparse'] / us['rowwise']:>7.3f} {us['sparse'] / ref:>7.3f} {r['sqnr_vs_bf16']['sparse']:>8.1f} "
              f"{r['sqnr_vs_bf16']['rowwise']:>8.1f} {r.get('max_abs_sparse_vs_reference', float('nan')):>9.3g}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
