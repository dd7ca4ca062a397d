"""Per-layer conv kernel timing of the benchmark network (YOLOv6-S, bs32, 640x640, bf16 mode) on cuda:0.

    python tools/conv_layers.py --out DIR [--iters 20] [--pair]

Each conv launch of one forward is timed on its own with CUDA events, after a 256 MB write that flushes the L2
(InferEngine.profile_layers), and the median over `--iters` launches is kept.  Also times the back-to-back conv launches of
a whole forward (InferEngine.profile_convs, the figure in bench.py's roofline).  `--pair` repeats both with every launch
asking for CTA pairs (force_pair = 1) -- the planner's default is unchanged.  Writes DIR/conv_layers.json with the GPU name
and power limit, and prints the table.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_info  # noqa: E402
from yolov6_b200.model import build_model  # noqa: E402
from yolov6_b200.synth import randomize_  # noqa: E402

MODEL, BATCH, SIZE = "yolov6s", 32, 640


def plan_str(p):
    """Plan dict (ops.PLAN_KEYS) -> 'BWxBHxBI BN<n> kb<k> st<stages> [halo<h> a<A stages>[ res]] [pair]'."""
    s = f"{p['BW']}x{p['BH']}x{p['BI']} BN{p['BN']} kb{p['KB']} st{p['stages']}"
    if p["halo"]:
        s += f" halo{p['halo']} a{p['a_res'] // 100}" + (" res" if p["a_res"] % 10 else "")
    if (p["a_res"] // 10) % 10:
        s += " pair"
    return s


def measure(eng, x, iters):
    rows = eng.profile_layers(x, iters=iters)
    table = [{"layer": r["name"], "shape": f"{r['cin']}->{r['cout']} k{r['k']}s{r['s']} out {r['hw']}", "plan": plan_str(r["plan"]),
              "median_ms": r["ms"], "tflops": r["tflops"]} for r in rows]
    total_ms, flop, launches = eng.profile_convs(x, steps=10)
    return {"layers": table, "sum_of_layer_medians_ms": sum(r["median_ms"] for r in table),
            "back_to_back_ms": total_ms, "back_to_back_tflops": flop / (total_ms * 1e-3) / 1e12, "launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory for conv_layers.json")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--pair", action="store_true", help="also time every launch with force_pair = 1")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    model = randomize_(build_model(MODEL, 80, dev), seed=0)
    model.eval().set_precision("bf16")
    eng = model.engine()
    x = torch.rand(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(1)).to(dev)
    result = {"workload": f"{MODEL} {SIZE}x{SIZE} bs{BATCH} bf16, conv launches of one forward", "gpu": gpu_info(0),
              "timing": f"median of {args.iters} launches, L2 flushed before each", "default": None}
    with torch.no_grad():
        result["default"] = measure(eng, x, args.iters)
        if args.pair:
            descs = [d for kind, d in eng._plan(BATCH, SIZE, SIZE, torch.float32)["calls"] if kind == "conv"]
            for d in descs:
                d.force_pair = 1
            try:
                result["force_pair"] = measure(eng, x, args.iters)
            finally:
                for d in descs:
                    d.force_pair = 0
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "conv_layers.json"), "w") as f:
        json.dump(result, f, indent=1)
    for key in ("default", "force_pair"):
        if key not in result:
            continue
        r = result[key]
        print(f"== {key}: back-to-back {r['back_to_back_ms']:.3f} ms ({r['back_to_back_tflops']:.0f} TFLOP/s), "
              f"sum of layer medians {r['sum_of_layer_medians_ms']:.3f} ms")
        for row in r["layers"]:
            print(f"{row['layer']:<40} {row['shape']:<32} {row['plan']:<34} {row['median_ms']:8.4f} ms {row['tflops']:6.1f} TFLOP/s")
    print(json.dumps({"gpu": result["gpu"]}))


if __name__ == "__main__":
    main()
