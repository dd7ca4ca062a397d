"""Training on rectangular canvases against the square: YOLOv6-S, batch 32, uint8 images, seeded synthetic weights, images
and targets, one GPU, no optimizer (the step is forward + loss + backward, as tools/bench_train.py).

  alternate: one TrainStep built with shapes=[(384, 640), (640, 384)] around 640 x 640 runs the three shapes in turn,
             step after step (every step switches shape and so clears the shared buffers); a square-only TrainStep runs
             beside it as the baseline.
  epoch:     --rect's batches (augment.rect_batches, stride 32, pad 0) over a seeded list of COCO-like aspect ratios,
             one TrainStep built with every canvas of the schedule, against the same number of 640 x 640 steps.

Per shape it prints ms per step (CUDA events around each run), images/s, the forward conv GFLOP per image of the graph
(tools/bench_models.py), captures and capture time, and the peak device memory each step allocates, measured for each
step built and run alone (no other step alive), with the card's name, power limit and maximum SM clock read in the same run.  One JSON line per run.

    python tools/bench_rect_train.py [--steps 20] [--warmup 3] [--runs 2] [--images 1024]
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(ROOT), ROOT]

from bench import gpu_info  # noqa: E402
from bench_models import conv_gflop_per_image  # noqa: E402
from yolov6_b200.augment import rect_batches  # noqa: E402
from yolov6_b200.loss import ComputeLoss  # noqa: E402
from yolov6_b200.model import build_model  # noqa: E402
from yolov6_b200.step import TrainStep  # noqa: E402
from yolov6_b200.synth import randomize_  # noqa: E402

B, SIZE, MODEL = 32, 640, "yolov6s"
RECTS = [(384, 640), (640, 384)]


def coco_like_shapes(n, seed):
    """(h0, w0) of n images: mostly 640-wide landscape 4:3 and 16:9, some portrait and square, as COCO's mix."""
    r = np.random.RandomState(seed)
    ar = r.choice([4 / 3, 16 / 9, 3 / 2, 1.0, 3 / 4, 2 / 3], n, p=[0.45, 0.1, 0.1, 0.1, 0.15, 0.1]) * r.uniform(0.95, 1.05, n)
    return [(int(round(640 / a)), 640) if a >= 1 else (640, int(round(640 * a))) for a in ar]


def inputs(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).pin_memory()
    n = 8 * B
    t = torch.rand(n, 6, generator=g)
    t[:, 0] = torch.arange(n) % B
    t[:, 1] = (t[:, 1] * 80).floor()
    t[:, 4:] = 0.05 + 0.3 * t[:, 4:]
    t[:, 2:4] = 0.2 + 0.6 * t[:, 2:4]
    return x, t


def make_step(shapes=None):
    m = randomize_(build_model(MODEL, 80, torch.device("cuda:0")), seed=0).train()
    crit = ComputeLoss(num_classes=80, ori_img_size=SIZE, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    return TrainStep(m, crit, B, SIZE, SIZE, in_dtype=torch.uint8, max_gt=64, shapes=shapes)


def timed(step, x, t):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    step.load(x, t)
    a.record()
    step.run()
    b.record()
    return a, b


def first_runs(step, batches):
    """Capture time of each shape: host clock around its first run, device synchronised."""
    out = {}
    for (H, W), (x, t) in batches.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step.load(x, t)
        step.run()
        torch.cuda.synchronize()
        out[f"{H}x{W}"] = round((time.perf_counter() - t0) * 1e3, 1)
    return out


def released():
    """Frees every step dropped so far (model and engine reference each other, so only the cyclic collector frees them)."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def alone(shapes, data):
    """Builds one step, runs each of its shapes once with no other step alive: (capture ms per shape, captures, peak GB of
    device memory allocated while building and running it, above what was allocated before)."""
    released()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step = make_step([s for s in shapes if s != (SIZE, SIZE)] or None)
    cap = first_runs(step, {s: data[s] for s in shapes})
    out = cap, step.captures, round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)
    del step
    released()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--images", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rect_train: no CUDA device")
    g = build_model(MODEL, 80, torch.device("cpu")).graph
    shapes = [(SIZE, SIZE)] + RECTS
    sched = rect_batches(coco_like_shapes(a.images, 7), SIZE, B, 32)
    sched = [(idx, c) for idx, c in sched if len(idx) == B]
    canv = sorted({c for _, c in sched})
    data = {s: inputs(*s, seed=k) for k, s in enumerate(sorted(set(shapes) | set(canv)))}

    # memory and captures: each step alone
    cap_sq, n_sq, peak_sq = alone([(SIZE, SIZE)], data)
    cap_alt, n_alt, peak_alt = alone(shapes, data)
    cap_ep, n_ep, peak_ep = alone(canv, data)

    # timing: the alternating step beside a square-only one, then the epoch step beside the square one
    square = make_step()
    first_runs(square, {(SIZE, SIZE): data[(SIZE, SIZE)]})
    multi = make_step(RECTS)
    first_runs(multi, {s: data[s] for s in shapes})
    arena_gb = round(multi.eng.arena.store.numel() / 2 ** 30, 2)
    z0, z1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    z0.record()
    for _ in range(10):
        multi.eng.arena.store.zero_()
    z1.record()
    torch.cuda.synchronize()
    clear_ms = z0.elapsed_time(z1) / 10
    multi.eng.arena.live = None
    info = gpu_info(0)
    alt = []
    for run in range(a.runs):
        ev = {s: [] for s in shapes}
        ev_sq = []
        for i in range(a.warmup + a.steps):
            for s in shapes:
                e = timed(multi, *data[s])
                if i >= a.warmup:
                    ev[s].append(e)
            e = timed(square, *data[(SIZE, SIZE)])
            if i >= a.warmup:
                ev_sq.append(e)
        torch.cuda.synchronize()
        alt.append(({f"{h}x{w}": float(np.median([x.elapsed_time(y) for x, y in ev[(h, w)]])) for h, w in shapes},
                    float(np.median([x.elapsed_time(y) for x, y in ev_sq]))))
    del multi
    released()
    ep = make_step([c for c in canv if c != (SIZE, SIZE)])
    first_runs(ep, {c: data[c] for c in canv})
    for run in range(a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _, c in sched:
            ep.load(*data[c])
            ep.run()
        torch.cuda.synchronize()
        t_rect = time.perf_counter() - t0
        t0 = time.perf_counter()
        for _ in sched:
            square.load(*data[(SIZE, SIZE)])
            square.run()
        torch.cuda.synchronize()
        t_sq = time.perf_counter() - t0
        ms, ms_sq = alt[run]
        n_img = B * len(sched)
        print(json.dumps({
            "bench": "rect_train", "run": run, "model": MODEL, "batch": B, "gpu": info,
            "alternate_ms_per_step": {k: round(v, 2) for k, v in ms.items()},
            "alternate_images_per_s": {k: round(B * 1e3 / v, 1) for k, v in ms.items()},
            "square_step_ms": round(ms_sq, 2), "square_step_images_per_s": round(B * 1e3 / ms_sq, 1),
            "fwd_conv_gflop_per_image": {f"{h}x{w}": round(conv_gflop_per_image(g, (h, w)), 2) for h, w in shapes},
            "captures": {"square": n_sq, "alternate": n_alt, "epoch": n_ep},
            "capture_ms": {"square": cap_sq, "alternate": cap_alt, "epoch": cap_ep},
            "peak_gb_each_step_alone": {"square": peak_sq, "alternate": peak_alt, "epoch": peak_ep},
            "arena_gb": arena_gb, "arena_clear_ms": round(clear_ms, 3),
            "epoch": {"batches": len(sched), "canvases": {f"{h}x{w}": sum(c == (h, w) for _, c in sched) for h, w in canv},
                      "rect_images_per_s": round(n_img / t_rect, 1), "square_images_per_s": round(n_img / t_sq, 1),
                      "speedup": round(t_sq / t_rect, 3),
                      "rect_fwd_conv_gflop_per_image": round(float(np.mean([conv_gflop_per_image(g, c) for _, c in sched])), 2)},
        }), flush=True)


if __name__ == "__main__":
    main()
