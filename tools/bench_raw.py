"""Serving from decoded frames: 1920x1080 uint8 BGR frames -> detections in source pixels, YOLOv6-S bs32 at 640 (bf16,
seeded synthetic weights, bench.py's NMS settings), one JSON line of frames/s for two ways of feeding the same DetectStream:

  raw:  raw_input=True -- the frames' bytes go to pinned staging and are letterboxed on the GPU (yv6_letterbox), boxes are
        rescaled on the GPU (yv6_rescale_boxes);
  cv2:  the reference's host path -- data_augment.letterbox (cv2.resize + copyMakeBorder, auto=False) + HWC->CHW + BGR->RGB on
        all host cores into the pinned uint8 batch, then the existing pipeline (rescale not included).

Each timed step packs / letterboxes one batch on the host, submits it and collects the previous one; the clock stops after
the last batch is collected.

    python tools/bench_raw.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import NMS_KW, gpu_info, host_cores  # noqa: E402


def cv2_letterbox_chw(im, S):
    """letterbox(im, (S, S), auto=False) (data/data_augment.py:29-58) + transpose / flip of Inferer.process_image, in cv2."""
    import cv2
    h0, w0 = im.shape[:2]
    r = min(S / h0, S / w0)
    nw, nh = int(round(w0 * r)), int(round(h0 * r))
    dw, dh = (S - nw) / 2, (S - nh) / 2
    if (w0, h0) != (nw, nh):
        im = cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR)
    top, bottom, left, right = int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1))
    im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
    return im.transpose(2, 0, 1)[::-1]


def run(ds, feed, steps, warmup):
    """feed(i) prepares batch i on the host and submits it; returns frames/s over `steps` batches."""
    def loop(n):
        for i in range(n):
            feed(i)
            ds.collect()
        ds.drain()
        while ds.collect() is not None:
            pass
    loop(warmup)
    torch.cuda.synchronize()
    t = time.perf_counter()
    loop(steps)
    torch.cuda.synchronize()
    return steps * ds.B / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    args = ap.parse_args()
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectStream
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    B, S = args.batch, args.size
    model = randomize_(build_model("yolov6s", 80, dev), seed=0)
    model.eval().set_precision("bf16")
    rng = np.random.default_rng(0)
    frames = [[rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(B)] for _ in range(2)]
    threads = host_cores()
    pool = ThreadPoolExecutor(threads)

    raw = DetectStream(model, B, S, S, raw_input=True, max_src_bytes=B * 1080 * 1920 * 3, **NMS_KW)
    fps_raw = run(raw, lambda i: raw.submit(frames[i & 1]), args.steps, args.warmup)
    del raw
    torch.cuda.empty_cache()

    host = DetectStream(model, B, S, S, host_input=True, **NMS_KW)
    batch = torch.empty(B, 3, S, S, dtype=torch.uint8)
    view = batch.numpy()

    def feed_cv2(i):
        def one(j):
            view[j] = cv2_letterbox_chw(frames[i & 1][j], S)
        list(pool.map(one, range(B)))
        host.submit(batch)
    fps_cv2 = run(host, feed_cv2, args.steps, args.warmup)
    print(json.dumps({"metric": f"frames/s 1920x1080 BGR -> detections, YOLOv6-S {S} bs{B}", "raw_frames_per_s": round(fps_raw, 1),
                      "cv2_host_frames_per_s": round(fps_cv2, 1), "host_threads": threads, "steps": args.steps,
                      "gpu": gpu_info(0)}), flush=True)


if __name__ == "__main__":
    main()
