"""Validation batches from decoded frames: ValFeed (yv6_letterbox_val) against the reference's host path.

The same seeded decoded frames -- a COCO-like mix of 640x480, 640x427 and 1920x1080 sources plus sizes that are no
integer multiple of the canvas (1000x777, 375x500, 3000x2000) -- are batched as TrainValDataset(augment=False, rect=True,
pad=0.5) batches them at img_size 320 and 640, batch 32, stride 32, and turned into device uint8 canvases three ways:

  host:        the reference's path on one host thread: cv2.resize (INTER_AREA / INTER_LINEAR, load_image) + letterbox
               (cv2.copyMakeBorder) + HWC->CHW + BGR->RGB + torch.from_numpy + stack + copy to the device;
  feed_host:   ValFeed from the same host frames (staged through pinned memory, one launch per batch);
  feed_device: ValFeed from the frames already in device memory (a GPU decoder's case).

Times are host clocks over every batch, ended by a device synchronise; `kernel_ms_per_batch` is yv6_letterbox_val's own
time from torch.profiler in a separate pass over the device frames.  `gb_per_s` is the bytes the kernel must move -- every
source byte read once and every canvas byte written once -- over that kernel time, beside the H100 SXM data-sheet 3.35 TB/s.  The first batch of
each size is checked byte for byte against the host path.  One JSON line per img_size, with the card's name, power limit
and maximum SM clock read in the same run.

    python tools/bench_valdata.py [--images 192] [--repeats 3]
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

from bench import gpu_info  # noqa: E402

# (h0, w0) and weight of each source size
MIX = [((480, 640), 5), ((427, 640), 3), ((640, 480), 2), ((1080, 1920), 2), ((777, 1000), 1), ((375, 500), 1), ((2000, 3000), 1)]
HBM_TBPS = 3.35


def sources(n, seed=0):
    rng = np.random.default_rng(seed)
    sizes = [s for s, w in MIX for _ in range(w)]
    shapes = [sizes[int(rng.integers(len(sizes)))] for _ in range(n)]
    return shapes, [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def host_batch(cv2, frames, H, W, img_size, dev):
    """load_image + letterbox(auto=False, scaleup=False) + CHW RGB + stack + H2D, as the reference's loader does it."""
    out = []
    for im in frames:
        h0, w0 = im.shape[:2]
        r = img_size / max(h0, w0)
        if r != 1:
            im = cv2.resize(im, (int(w0 * r), int(h0 * r)), interpolation=cv2.INTER_AREA if r < 1 else cv2.INTER_LINEAR)
        h, w = im.shape[:2]
        dw, dh = (W - w) / 2, (H - h) / 2
        top, bottom, left, right = int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1))
        im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        out.append(torch.from_numpy(np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])))
    return torch.stack(out, 0).to(dev)


def timed(fn, batches):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for b in batches:
        fn(b)
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=192)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_valdata: needs a CUDA device")
    import cv2
    from yolov6_b200.valdata import ValFeed
    dev = torch.device("cuda:0")
    shapes, frames = sources(args.images)
    dev_frames = [torch.from_numpy(f).to(dev) for f in frames]
    labels = [np.zeros((0, 5), np.float32)] * len(frames)
    B = args.batch
    for S in (320, 640):
        feed = ValFeed(B, S, 32, shapes, max_src_bytes=B * 3000 * 2000 * 3, device=dev)
        batches = [(list(idx), tuple(int(v) for v in feed.canvases[b])) for b, idx in enumerate(feed.batches())]
        n_img = sum(len(i) for i, _ in batches)

        def host(b):
            host_batch(cv2, [frames[i] for i in b[0]], *b[1], S, dev)

        def feed_host(b):
            feed.feed(b[0], [frames[i] for i in b[0]], [labels[i] for i in b[0]])

        def feed_device(b):
            feed.feed(b[0], [dev_frames[i] for i in b[0]], [labels[i] for i in b[0]])

        idx, (H, W) = batches[0]
        got = feed.feed(idx, [dev_frames[i] for i in idx], [labels[i] for i in idx])[0][:len(idx)]
        assert torch.equal(got, host_batch(cv2, [frames[i] for i in idx], H, W, S, dev)), "ValFeed differs from cv2"
        for fn in (host, feed_host, feed_device):
            timed(fn, batches[:2])
        res = {"host": [], "feed_host": [], "feed_device": []}
        for r in range(args.repeats):
            for name, fn in (("host", host), ("feed_host", feed_host), ("feed_device", feed_device)):
                res[name].append(timed(fn, batches))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:      # a run of its own
            timed(feed_device, batches)
        kern = [e for e in prof.key_averages() if "letterbox_val_kernel" in e.key]
        assert len(kern) == 1 and kern[0].count == len(batches), [(e.key, e.count) for e in kern]
        ev = getattr(kern[0], "device_time_total", None) or kern[0].cuda_time_total       # microseconds
        ev /= 1e6
        moved = sum(int(np.prod(shapes[i])) * 3 for idx, _ in batches for i in idx) + sum(B * 3 * H * W for _, (H, W) in batches)
        best = {k: min(v) for k, v in res.items()}
        print(json.dumps({
            "metric": f"validation batches from decoded frames, img_size {S}, rect batches of {B}, stride 32",
            "images": n_img, "batches": len(batches), "canvases": sorted({c for _, c in batches}),
            "host_images_per_s": round(n_img / best["host"], 1), "feed_host_images_per_s": round(n_img / best["feed_host"], 1),
            "feed_device_images_per_s": round(n_img / best["feed_device"], 1),
            "host_ms_per_batch": round(1e3 * best["host"] / len(batches), 3),
            "feed_host_ms_per_batch": round(1e3 * best["feed_host"] / len(batches), 3),
            "feed_device_ms_per_batch": round(1e3 * best["feed_device"] / len(batches), 3),
            "kernel_ms_per_batch": round(1e3 * ev / len(batches), 3),
            "kernel_bytes": moved, "gb_per_s": round(moved / ev / 1e9, 1),
            "share_of_3_35_tb_per_s": round(moved / ev / (HBM_TBPS * 1e12), 4),
            "measured": True, "repeats": args.repeats, "gpu": gpu_info(0)}), flush=True)


if __name__ == "__main__":
    main()
