"""Time the GPU PR metric (yolov6_b200.metrics.PRMetric) on a COCO-val-sized synthetic set: 5000 images, batches of 32,
up to 300 NMS rows per image, 80 classes.

    python tools/bench_metrics.py [--images 5000] [--batch 32] [--repeat 5]

GPU arm: `update` per batch and `result()` timed with CUDA events (the rows are already on the device, as DetectPipeline
leaves them).  CPU arm: the oracle (oracle/metrics.py, numpy; the same per-image matching and ap_per_class) on the host
cores, timed with a wall clock.  The oracle is not the reference's code, so its time is not the reference's time.
Prints the card name and its power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        power = f"unknown ({e.__class__.__name__})"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeat", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py needs a CUDA device")
    from oracle import metrics as om
    from yolov6_b200.metrics import PRMetric
    dev = torch.device("cuda:0")
    batches, nc = om.coco_val_sized(n_images=args.images, B=args.batch)
    staged = []
    for preds, targets, shapes, hw in batches:
        out, count = om.pack(preds, 300)
        staged.append((torch.from_numpy(out).to(dev), torch.from_numpy(count).to(dev), torch.from_numpy(targets), shapes, hw))
    metric = PRMetric(nc, max_images=args.images, device=dev, confusion=True)
    upd, res_ms = [], []
    for rep in range(args.repeat + 1):                       # the first pass warms up
        metric.reset()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in staged:
            metric.update(*s)
        e1.record()
        torch.cuda.synchronize()
        r0 = time.perf_counter()
        res = metric.result()
        r1 = time.perf_counter()
        if rep:
            upd.append(e0.elapsed_time(e1) / len(staged))
            res_ms.append((r1 - r0) * 1e3)
    t0 = time.perf_counter()
    ref = om.evaluate(batches, nc)
    cpu_s = time.perf_counter() - t0
    assert abs(ref["map50"] - res.map50) <= 1e-12 and abs(ref["map"] - res.map) <= 1e-12
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "images": args.images, "batch": args.batch,
                      "rows": int(len(ref["conf"])), "labels": int(len(ref["tcls"])),
                      "gpu_update_ms_per_batch": round(float(np.median(upd)), 4),
                      "gpu_result_ms": round(float(np.median(res_ms)), 3),
                      "cpu_oracle_s": round(cpu_s, 2), "cpu_threads": torch.get_num_threads(),
                      "map50": res.map50, "map": res.map}))


if __name__ == "__main__":
    main()
