"""Time the GPU COCO box evaluation (yolov6_b200.cocoeval.COCOMetric) on a COCO-val-sized fabricated set: 5000 images,
80 categories with non-contiguous ids, about 37k gts (about 1 % crowd, areas over all three ranges), 300 NMS rows per
image (jittered gts and false positives), batches of 32.

    python tools/bench_cocoeval.py [--images 5000] [--batch 32] [--repeat 5]

GPU arm: `update` per batch and `result()` timed with CUDA events around work that ends in a synchronise (the rows are
already on the device, as DetectPipeline leaves them).  If pycocotools imports, it is timed on the same rows
(loadRes + evaluate + accumulate + summarize, host wall clock) and its stats are compared; otherwise the output says so.
The CPU oracle is not timed: it is not pycocotools.  Prints the card name and its power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
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


def time_pycocotools(gt, make_rows):
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
        if not hasattr(COCOeval, "evaluate"):
            raise ImportError
    except ImportError:
        return None, None
    rows = make_rows()
    with tempfile.TemporaryDirectory() as d:
        gpath, rpath = os.path.join(d, "gt.json"), os.path.join(d, "predictions.json")
        with open(gpath, "w") as f:
            json.dump(gt, f)
        with open(rpath, "w") as f:
            json.dump(rows, f)
        coco = COCO(gpath)
        t0 = time.perf_counter()
        ev = COCOeval(coco, coco.loadRes(rpath), "bbox")
        ev.evaluate()
        ev.accumulate()
        ev.summarize()
        return time.perf_counter() - t0, ev.stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeat", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cocoeval.py needs a CUDA device")
    from oracle import cocoeval as oc
    from yolov6_b200.cocoeval import COCOMetric
    dev = torch.device("cuda:0")
    gt, batches, ids = oc.fabricate(2024, args.images, n_cats=80, crowd=0.01, B=args.batch, p_full=1.0)
    staged = [(torch.from_numpy(o).to(dev), torch.from_numpy(c).to(dev), s, i) for o, c, s, i in batches]
    metric = COCOMetric(gt, ids, device=dev)
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
    rows = int(sum(int(b[1].sum()) for b in batches))
    py_s, py_stats = time_pycocotools(gt, lambda: oc.rows_of(batches, ids))
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "images": args.images, "batch": args.batch, "rows": rows,
                      "gts": len(gt["annotations"]), "crowd": int(sum(a["iscrowd"] for a in gt["annotations"])),
                      "gpu_update_ms_per_batch": round(float(np.median(upd)), 4), "gpu_result_ms": round(float(np.median(res_ms)), 3),
                      "gpu_epoch_ms": round(float(np.median(upd)) * len(staged) + float(np.median(res_ms)), 2),
                      "pycocotools_s": round(py_s, 2) if py_s is not None else "pycocotools is not installed: not timed",
                      "pycocotools_stats_equal": bool(np.array_equal(py_stats, res.stats)) if py_stats is not None else None,
                      "AP": float(res.stats[0]), "AP50": float(res.stats[1])}))


if __name__ == "__main__":
    main()
