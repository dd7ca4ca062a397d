"""What loading new weights into captured inference pipelines costs, per detector: the yv6_fold launch alone, the path without
refold (ema_state_dict() into a fresh model, its engine and k rect-canvas pipelines rebuilt and recaptured), load_weights_ on
the captured pipelines, and one whole validation pass each way over a synthetic set with several canvases.

    python tools/bench_refold.py [--models yolov6s yolov6m yolov6l6] [--precision bf16] [--canvases 4] [--batch 32]

Prints one JSON line per detector, with the card name and its power limit (nvidia-smi, read-only query) in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from yolov6_b200 import refold  # noqa: E402
from yolov6_b200.cocoeval import COCOMetric  # noqa: E402
from yolov6_b200.evaluate import EpochEval  # noqa: E402
from yolov6_b200.model import build_model  # noqa: E402
from yolov6_b200.optim import FusedSGDEMA  # noqa: E402
from yolov6_b200.pipeline import DetectPipeline  # noqa: E402
from yolov6_b200.synth import randomize_  # noqa: E402
from yolov6_b200.valdata import ValFeed  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:          # the numbers stay valid; the card is then unknown
        return torch.cuda.get_device_name(0), "unknown"


def synthetic_set(n_canvas, batch, img_size, stride):
    """Sources of n_canvas aspect-ratio groups (one rect canvas each), `batch` images per group, with a few labels each."""
    shapes, frames, labels = [], [], []
    rng = np.random.default_rng(0)
    for g in range(n_canvas):
        h0, w0 = img_size, int(img_size * (0.5 + 0.5 * g / max(n_canvas - 1, 1)))
        for _ in range(batch):
            shapes.append((h0, w0))
            frames.append(rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8))
            labels.append(np.array([[rng.integers(0, 80), 0.5, 0.5, 0.3, 0.4]], np.float32))
    anno = {"images": [{"id": i} for i in range(len(shapes))], "categories": [{"id": j} for j in range(80)],
            "annotations": [{"id": i + 1, "image_id": i, "category_id": int(lab[0, 0]), "bbox": [w0 * 0.35, h0 * 0.3, w0 * 0.3, h0 * 0.4],
                             "area": w0 * h0 * 0.12, "iscrowd": 0} for i, ((h0, w0), lab) in enumerate(zip(shapes, labels))]}
    return shapes, frames, labels, anno


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def bench(name, precision, n_canvas, batch, img_size, reps):
    train = randomize_(build_model(name, 80, DEV), seed=0).train()
    with torch.no_grad():
        for n, p in train.named_parameters():
            if n.endswith("alpha"):
                p.fill_(1.0)
    opt = FusedSGDEMA(train)
    stride = max(32, int(train.stride.max()))
    shapes, frames, labels, anno = synthetic_set(n_canvas, batch, img_size, stride)
    feed = ValFeed(batch, img_size, stride, shapes, device=DEV)
    canvases = sorted({tuple(int(v) for v in c) for c in feed.canvases})
    source = lambda idx: ([frames[i] for i in idx], [labels[i] for i in idx])       # noqa: E731

    ev = EpochEval(build_model(name, 80, DEV).set_precision(precision), feed, source, COCOMetric(anno, list(range(80)), device=DEV))
    ev.run(opt)                                    # builds and captures the pipelines once
    ev.run(opt)                                    # and folds once from the EMA layout (its records on the device)
    eng = ev.model.engine()

    # the fold kernel alone: events around back-to-back launches
    plan = eng._fold_plan(opt.flat.slots)
    tables = plan.dev[id(eng)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(50):
        refold.launch(eng.lib, eng.handle, tables, opt.ema, False, torch.cuda.current_stream())
    e1.record()
    torch.cuda.synchronize()
    fold_ms = e0.elapsed_time(e1) / 50

    def rebuild():                                  # the path without refold
        m = build_model(name, 80, DEV)
        m.load_state_dict(opt.ema_state_dict())
        m.eval().set_precision(precision)
        for H, W in canvases:
            DetectPipeline(m, batch, H, W, host_input=False, multi_label=True, conf_thres=0.03, iou_thres=0.65)

    def host_pass():                               # a whole validation pass the same way
        m = build_model(name, 80, DEV)
        m.load_state_dict(opt.ema_state_dict())
        m.eval().set_precision(precision)
        e = EpochEval(m, feed, source, ev.metric)
        e.run(m.state_dict())

    out = dict(model=name, precision=precision, canvases=len(canvases), batch=batch, img_size=img_size,
               fold_kernel_ms=fold_ms,
               rebuild_ms=timed(rebuild, reps),
               load_weights_ms=timed(lambda: ev.model.load_weights_(opt), reps),
               val_pass_rebuild_ms=timed(host_pass, reps),
               val_pass_refold_ms=timed(lambda: ev.run(opt), reps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["yolov6s", "yolov6m", "yolov6l6"])
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--canvases", type=int, default=4)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--img-size", type=int, default=640)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    name, limit = card()
    for m in a.models:
        r = bench(m, a.precision, a.canvases, a.batch, a.img_size, a.reps)
        r.update(card=name, power_limit=limit)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
