"""Serving 1920x1080 frames on the full square canvas against the minimum-rectangle one: YOLOv6-S bf16 at img_size 640,
batch 32, bench.py's NMS settings, seeded synthetic weights and frames.  The same device-resident 1080p frames (uint8 BGR
HWC, generated from a seed) go through two two-lane DetectFarms with raw_input=True:

  full: auto=False -- every frame letterboxed onto 640 x 640 (the Evaler's canvas);
  rect: auto=True, source_shape=(1080, 1920) -- Inferer.process_image's canvas, padded only to the stride: 384 x 640.

Each timed step submits one batch and collects the previous batch of that lane; the clock (host, after a device
synchronise) stops when every batch is collected.  The two farms alternate within each of `--runs` runs, and each run
prints one JSON line with both rates, their ratio, the conv GFLOP per image of each canvas (2 x MACs, tools/bench_models.py)
and the card's name, power limit and maximum SM clock read in the same run.

    python tools/bench_rect.py [--steps 40] [--warmup 5] [--runs 3] [--batch 32] [--model yolov6s]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import NMS_KW, gpu_info  # noqa: E402
from bench_models import conv_gflop_per_image  # noqa: E402

SOURCE = (1080, 1920)


def run(farm, frames, steps):
    """Images/s of `steps` batches through the farm, every batch collected."""
    L = len(farm.lanes)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for i in range(steps):
        farm.submit(frames[i & 1])
        farm.lanes[i % L].collect()        # the lane's previous batch, post-processed by the step just submitted
    for ln, lane in enumerate(farm.lanes):
        with torch.cuda.stream(farm.streams[ln]):
            lane.drain()
    torch.cuda.synchronize()
    for lane in farm.lanes:
        while lane.collect() is not None:
            pass
    return steps * len(frames[0]) / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--model", default="yolov6s")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rect: needs a CUDA device")
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectFarm
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    B, S = args.batch, args.size
    model = randomize_(build_model(args.model, 80, dev), seed=0)
    model.eval().set_precision("bf16")
    rng = np.random.default_rng(0)
    frames = [[torch.from_numpy(rng.integers(0, 256, (*SOURCE, 3), dtype=np.uint8)).to(dev) for _ in range(B)] for _ in range(2)]
    farms = {"full": DetectFarm(model, B, S, S, lanes=2, raw_input=True, **NMS_KW),
             "rect": DetectFarm(model, B, S, S, lanes=2, raw_input=True, auto=True, source_shape=SOURCE, **NMS_KW)}
    gflop = {k: round(conv_gflop_per_image(model.graph, f.canvas), 3) for k, f in farms.items()}
    for f in farms.values():
        run(f, frames, args.warmup)
    for r in range(args.runs):
        order = list(farms) if r % 2 == 0 else list(farms)[::-1]
        ips = {k: round(run(farms[k], frames, args.steps), 1) for k in order}
        print(json.dumps({"metric": f"images/s 1920x1080 device frames -> detections, {args.model} bf16 img_size {S} bs{B}, "
                                    f"DetectFarm 2 lanes", "full_canvas": list(farms["full"].canvas), "rect_canvas": list(farms["rect"].canvas),
                          "full_images_per_s": ips["full"], "rect_images_per_s": ips["rect"],
                          "rect_over_full": round(ips["rect"] / ips["full"], 3), "full_conv_gflop_per_img": gflop["full"],
                          "rect_conv_gflop_per_img": gflop["rect"], "order": order, "steps": args.steps, "run": r,
                          "gpu": gpu_info(0)}), flush=True)


if __name__ == "__main__":
    main()
