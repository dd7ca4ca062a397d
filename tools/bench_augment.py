"""Training augmentation on the device: kernel time per batch, and the TrainStep step time preloaded vs fed by AugmentFeed.

    python tools/bench_augment.py [--batch 32] [--size 640] [--iters 20]
    python tools/bench_augment.py --reference-host /path/to/YOLOv6      # host time of the reference's __getitem__ (CPU only)

Sources are COCO-like synthetic frames (640x480 and mixed sizes); hyps are yolov6s and yolov6l6.  Prints one JSON line per
measurement with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def dataset(n, mixed, seed=0):
    rng = np.random.default_rng(seed)
    sizes = [(480, 640)] * n if not mixed else [tuple(int(v) for v in rng.choice([(480, 640), (640, 480), (427, 640), (375, 500), (720, 1280), (333, 500)])) for _ in range(n)]
    src = {i: rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for i, (h, w) in enumerate(sizes)}
    labels = {}
    for i in range(n):
        k = int(rng.integers(1, 14))
        wh = rng.uniform(0.02, 0.5, (k, 2))
        labels[i] = np.concatenate([rng.integers(0, 80, (k, 1)), rng.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32)
    return src, labels


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:        # noqa: BLE001
        return f"unknown ({e})"


def gpu(args):
    import torch
    from oracle import fabricate as fab
    from yolov6_b200.augment import HYP_YOLOV6L6, HYP_YOLOV6S, AugmentFeed, as_source, batch_tables, resize_frames_launch
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.preprocess import check_frame
    from yolov6_b200.step import TrainStep
    dev = torch.device("cuda:0")
    B, S = args.batch, args.size
    info = card()
    n = 4 * B
    for mixed in (False, True):
        src, labels = dataset(n, mixed)
        max_src = 8 * B * max(v.nbytes for v in src.values())
        for hname, hyp in (("yolov6s", HYP_YOLOV6S), ("yolov6l6", HYP_YOLOV6L6)):
            feed = AugmentFeed(B, S, S, hyp, n, max_src, device=dev)
            random.seed(0)
            np.random.seed(0)
            plans = [feed.draw(list(range(j * B % n, j * B % n + B))) for j in range(args.iters + 3)]
            # kernel time: resize + augment on the aug stream, bracketed by events (copies excluded by waiting first)
            times, moved = [], []
            for j, plan in enumerate(plans):
                feed.submit(plan, src, labels)
                torch.cuda.synchronize()
            for plan in plans[3:]:
                srcs = {i: as_source(check_frame(src[i], "bgr_hwc", dev), "bgr_hwc") for i in plan.sources}
                used, total, shapes, loc, jobs1, recs1, jobs2, smp = batch_tables(feed.sampler, B, plan, srcs)
                feed.submit(plan, src, labels)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                slot = feed.slots[feed.turn ^ 1]
                from yolov6_b200 import _lib
                import ctypes as C
                h, L, sp = _lib.handle(0), _lib.lib(), _lib.stream_ptr()
                e0.record()
                if jobs1:
                    resize_frames_launch(dev, slot["recs_dev"].data_ptr(), slot["jobs_dev"][0].data_ptr(), len(jobs1),
                                         max(j[4] * j[5] for j in jobs1), slot["arena"].data_ptr(), None)
                if jobs2:
                    _lib.check(L.yv6_aug_resize(h, C.c_void_p(slot["arena"].data_ptr()), C.c_void_p(slot["jobs_dev"][1].data_ptr()), len(jobs2),
                                                max(j[4] * j[5] for j in jobs2), sp))
                _lib.check(L.yv6_augment(h, C.c_void_p(slot["arena"].data_ptr()), C.c_void_p(slot["samples_dev"].data_ptr()), B, S, S,
                                         C.c_void_p(feed.images.data_ptr()), sp))
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                # bytes the kernels must move: each resize reads its source and writes its result; augment writes B x 3 x S x S
                # and reads at least the canvas pixels it samples (bounded below by the output size per canvas)
                rb = sum(j[1] * j[2] * 3 + j[4] * j[5] * 3 for j in jobs1 + jobs2)
                ncanvas = sum(len(p.canvases) for p in plan.samples)
                moved.append(rb + B * 3 * S * S + ncanvas * 3 * S * S)
            t = float(np.median(times)) * 1e-3
            b = float(np.median(moved))
            print(json.dumps(dict(what="augment_kernels", hyp=hname, mixed_sizes=mixed, batch=B, size=S, ms=t * 1e3,
                                  bytes=b, GBps=b / t / 1e9, hbm_fraction=b / t / 3.35e12, card=info)), flush=True)
    # step time: preloaded vs fed, alternating in one process
    src, labels = dataset(n, True)
    max_src = 8 * B * max(v.nbytes for v in src.values())
    sd = fab.fabricate_state_dict(_keys("yolov6s"), seed=0)
    m = build_model("yolov6s", 80, dev)
    m.load_state_dict(sd)
    crit = ComputeLoss(num_classes=80, ori_img_size=S, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    step = TrainStep(m.train(), crit, B, S, S, in_dtype=torch.uint8)
    feed = AugmentFeed(B, S, S, HYP_YOLOV6S, n, max_src, step=step)
    random.seed(1)
    np.random.seed(1)
    plan = feed.draw(list(range(B)))
    tg = feed.submit(plan, src, labels)
    feed.wait()
    pre_imgs = step.images.clone()
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
    res = {"preloaded": [], "fed": []}
    for it in range(args.iters):
        for mode in ("preloaded", "fed"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(5):
                if mode == "preloaded":
                    step.load(pre_imgs, tg)
                    step.run()
                else:
                    feed.wait()
                    step.run()
                    nxt = feed.draw(list(range((j + 1) * B % n, (j + 1) * B % n + B)))
                    feed.submit(nxt, src, labels)
            torch.cuda.synchronize()
            res[mode].append((time.perf_counter() - t0) / 5 * 1e3)
    print(json.dumps(dict(what="trainstep_ms", model="yolov6s", batch=B, size=S, preloaded=float(np.median(res["preloaded"])),
                          fed=float(np.median(res["fed"])), preloaded_min=min(res["preloaded"]), fed_min=min(res["fed"]), card=info)), flush=True)


def _keys(name):
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(here, "tests", "golden", f"keys_{name}.json")) as f:
        return [(k, tuple(s)) for k, s in json.load(f)]


def reference_host(path, args):
    """Host time of the reference's __getitem__ per sample on one core (the stand-in dataset of make_golden_augment)."""
    import tempfile
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(here, "tests", "golden", "refshim"), path]
    import cv2
    cv2.setNumThreads(1)
    from yolov6.data.datasets import TrainValDataset
    from yolov6_b200.augment import HYP_YOLOV6L6, HYP_YOLOV6S
    n = 64
    src, labels = dataset(n, True)
    for hname, hyp in (("yolov6s", HYP_YOLOV6S), ("yolov6l6", HYP_YOLOV6L6)):
        d = TrainValDataset.__new__(TrainValDataset)
        d.augment, d.hyp, d.img_size, d.specific_shape, d.rect, d.cache_ram = True, hyp, args.size, False, False, False
        d.target_height = d.target_width = args.size
        with tempfile.TemporaryDirectory() as tmp:
            d.img_paths = []
            for i in range(n):
                p = os.path.join(tmp, f"{i}.png")
                cv2.imwrite(p, src[i])
                d.img_paths.append(p)
            d.labels = [labels[i] for i in range(n)]
            loaded = [d.load_image(i) for i in range(n)]
        d.imgs, d.imgs_hw0, d.imgs_hw = [x[0] for x in loaded], [x[1] for x in loaded], [x[2] for x in loaded]
        d.cache_ram = True
        random.seed(0)
        np.random.seed(0)
        t0 = time.perf_counter()
        for i in range(n):
            d[i]
        dt = (time.perf_counter() - t0) / n
        print(json.dumps(dict(what="reference_getitem_ms_per_sample", hyp=hname, size=args.size, ms=dt * 1e3, cores=1,
                              note="RAM-cached sources, excludes decoding")), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reference-host", default=None)
    a = ap.parse_args()
    if a.reference_host:
        reference_host(a.reference_host, a)
    else:
        gpu(a)
