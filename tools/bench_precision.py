"""Speed and accuracy of the bf16 and fp16 inference modes side by side: YOLOv6-S, batch 32, 640 x 640 (bench.py's flagship
shape), steady-state DetectFarm images/s per mode in alternating runs within one process (so both see the same clocks and
neighbours), then each mode's max deviation from the fp32-equivalent mode on the benchmark input: max |a - b| / (1 + |b|) over
the decoded predictions [B, A, 85], the metric of bench.py's precision_check.  Prints one JSON line; writes nothing.

    python tools/bench_precision.py [--rounds 5] [--steps 50] [--warmup 10]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

MODES = ("bf16", "fp16")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov6s")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision: no CUDA device")
    dev = torch.device("cuda:0")
    runs = {m: [] for m in MODES}
    model = x = None
    for r in range(a.rounds):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):      # alternate which mode goes first
            out = bench.bench_infer(a.model, a.batch, a.size, a.steps, a.warmup, 0, 1, dev, precision=m, e2e=False, roofline=False)
            runs[m].append(out["value"])
            model, x = out["_model"], out["_input"]
            del out
            torch.cuda.empty_cache()
    with torch.no_grad():
        pred = {}
        for m in ("fp32",) + MODES:
            model.set_precision(m)
            pred[m] = model.engine().forward(x).clone()
        dev_of = {m: float(((pred[m] - pred["fp32"]).abs() / (1 + pred["fp32"].abs())).max()) for m in MODES}
    props = torch.cuda.get_device_properties(dev)
    line = {"model": a.model, "batch": a.batch, "size": a.size, "pipeline": "DetectFarm", "unit": "images/s", "gpu": props.name,
            "rounds": a.rounds, "steps": a.steps,
            "images_per_s": {m: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for m, v in runs.items()},
            "fp16_over_bf16": statistics.median(runs["fp16"]) / statistics.median(runs["bf16"]),
            "max_rel_dev_vs_fp32": dev_of, "dev_ratio_fp16_over_bf16": dev_of["fp16"] / max(dev_of["bf16"], 1e-30)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
