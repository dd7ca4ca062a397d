"""Training from frames in GPU memory: a YOLOv6-S TrainStep fed by AugmentFeed from host frames, from CUDA frames uploaded
once, from JPEGs decoded on the GPU on a side stream (`ready=`) by torchvision's nvJPEG ("decode") and by this project's
decoder from a JpegStore ("gpujpeg"), and from a FrameCache, against the same step preloaded.

    python tools/bench_augment_frames.py [--batch 32] [--size 640] [--steps 10] [--reps 3]

Sources are synthetic photographs -- smooth gradients and blobs with mild grain, so they compress like photos rather
than like noise -- at COCO-like sizes, encoded as JPEG (quality 90) for the decode feed.  The feeds alternate in one
process, `reps` rounds of `steps` steps each.  Prints one JSON line per measurement with the card name and power limit
read in the same run:
  - trainstep_ms: median ms per step of each feed and of the preloaded step;
  - submit_cpu_ms: mean host process time per `submit` (and process and wall time per GPU decode call);
  - resize_frames_ms: the first-pass yv6_aug_resize_frames launch of one batch, timed with CUDA events, per feed;
  - jpeg: the sources' mean JPEG size in MB per frame;
  - jpeg_decode_ms: this project's decode of one batch's sources from the device store: its device work alone (CUDA
    events, the stream held until the call has enqueued everything) as ms, images/s, compressed MB/s and output GB/s, and
    the host time of the call.
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

from bench_augment import _keys, card  # noqa: E402

SIZES = [(480, 640), (640, 480), (427, 640), (375, 500), (720, 1280), (333, 500)]


def photo(h, w, rng):
    """A smooth synthetic photograph (uint8 HWC BGR): per-channel low-frequency waves, a few soft blobs, mild grain."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.empty((h, w, 3), np.float32)
    for c in range(3):
        fy, fx = rng.uniform(0.5, 3, 2) * np.pi / np.array([h, w])
        img[..., c] = 128 + 60 * np.sin(y * fy + x * fx + rng.uniform(0, 2 * np.pi))
    for _ in range(6):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0.05, 0.3) * max(h, w)
        img += rng.uniform(-80, 80, 3) * np.exp(-((y - cy) ** 2 + (x - cx) ** 2) / (2 * r * r))[..., None]
    img += rng.normal(0, 3, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def dataset(n, seed=0):
    rng = np.random.default_rng(seed)
    sizes = [SIZES[int(k)] for k in rng.integers(0, len(SIZES), n)]
    src = {i: photo(h, w, rng) for i, (h, w) in enumerate(sizes)}
    labels = {}
    for i in range(n):
        k = int(rng.integers(1, 14))
        wh = rng.uniform(0.02, 0.5, (k, 2))
        labels[i] = np.concatenate([rng.integers(0, 80, (k, 1)), rng.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32)
    return src, labels


def main(args):
    import torch
    from torchvision.io import decode_jpeg, encode_jpeg

    from oracle import fabricate as fab
    from yolov6_b200.jpeg import JpegDecoder, JpegStore
    from yolov6_b200.augment import HYP_YOLOV6S, AugmentFeed, FrameCache, as_source, batch_tables, resize_frames_launch
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.preprocess import check_frame
    from yolov6_b200.step import TrainStep
    dev = torch.device("cuda:0")
    B, S = args.batch, args.size
    info = card()
    n = 4 * B
    src, labels = dataset(n)
    jpegs = {i: encode_jpeg(torch.from_numpy(np.ascontiguousarray(src[i][..., ::-1].transpose(2, 0, 1))), quality=90)
             for i in src}
    print(json.dumps(dict(what="jpeg", frames=n, mb_per_frame=float(np.mean([j.numel() for j in jpegs.values()])) / 1e6,
                          raw_mb_per_frame=float(np.mean([s.nbytes for s in src.values()])) / 1e6, quality=90, card=info)), flush=True)
    max_src = 8 * B * max(v.nbytes for v in src.values())

    sd = fab.fabricate_state_dict(_keys("yolov6s"), seed=0)
    m = build_model("yolov6s", 80, dev)
    m.load_state_dict(sd)
    crit = ComputeLoss(num_classes=80, ori_img_size=S, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    step = TrainStep(m.train(), crit, B, S, S, in_dtype=torch.uint8)
    feeds = {k: AugmentFeed(B, S, S, HYP_YOLOV6S, n, max_src, step=step) for k in ("host", "device", "decode", "gpujpeg")}
    store = JpegStore([jpegs[i].numpy().tobytes() for i in range(n)], device=dev)     # every source's JPEG resident on the card
    gdec = JpegDecoder(dev)
    cache = FrameCache([s.shape[:2] for s in src.values()], feeds["host"].sampler, 4 << 30)
    cache.put(src)
    feeds["cache"] = AugmentFeed(B, S, S, HYP_YOLOV6S, n, max_src, step=step, cache=cache)
    dev_frames = {i: torch.from_numpy(s).to(dev) for i, s in src.items()}
    side = torch.cuda.Stream(dev)
    cpu = {k: [] for k in feeds}
    decode_cpu, gdec_cpu = [], []

    def submit(mode, plan):
        feed = feeds[mode]
        ready = None
        if mode == "host":
            frames = src
        elif mode == "device":
            frames = dev_frames
        elif mode == "cache":
            frames = {}
        elif mode == "gpujpeg":    # yolov6_b200.jpeg from the device store on a side stream
            c0, w0 = time.process_time(), time.perf_counter()
            frames, ready = gdec.decode({i: i for i in plan.sources}, stream=side, store=store)
            gdec_cpu.append(((time.process_time() - c0) * 1e3, (time.perf_counter() - w0) * 1e3, len(plan.sources)))
        else:                      # nvJPEG on a side stream: the step on the current stream keeps running meanwhile
            c0, w0 = time.process_time(), time.perf_counter()
            with torch.cuda.stream(side):
                out = decode_jpeg([jpegs[i] for i in plan.sources], device=dev)
                ready = torch.cuda.Event()
                ready.record(side)
            decode_cpu.append(((time.process_time() - c0) * 1e3, (time.perf_counter() - w0) * 1e3, len(plan.sources)))
            frames = dict(zip(plan.sources, out))
        c0 = time.process_time()
        feed.submit(plan, frames, labels, layout="rgb_chw" if mode == "decode" else "bgr_hwc", ready=ready)
        cpu[mode].append((time.process_time() - c0) * 1e3)
        return frames

    def indices(j):
        return list(range(j * B % n, j * B % n + B))

    # first-pass resize launch of one batch per feed, CUDA events around the launch alone
    random.seed(2)
    np.random.seed(2)
    plan = feeds["host"].draw(indices(1))
    for mode, feed in feeds.items():
        times = []
        for _ in range(args.steps):
            frames = submit(mode, plan)
            torch.cuda.synchronize()
            if mode == "cache":
                srcs = {i: cache.source(i) for i in plan.sources}
            else:
                lay = "rgb_chw" if mode == "decode" else "bgr_hwc"
                srcs = {i: as_source(check_frame(frames[i], lay, dev), lay) for i in plan.sources}
            _, _, _, _, jobs1, _, _, _ = batch_tables(feed.sampler, B, plan, srcs)
            slot = feed.slots[feed.turn ^ 1]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            resize_frames_launch(dev, slot["recs_dev"].data_ptr(), slot["jobs_dev"][0].data_ptr(), len(jobs1),
                                 max(j[4] * j[5] for j in jobs1), slot["arena"].data_ptr(), None)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        moved = sum(j[1] * j[2] * 3 + j[4] * j[5] * 3 for j in jobs1)
        t = float(np.median(times))
        print(json.dumps(dict(what="resize_frames_ms", feed=mode, batch=B, size=S, jobs=len(jobs1), ms=t, min_ms=min(times),
                              bytes=moved, GBps=moved / (t * 1e-3) / 1e9, card=info)), flush=True)
    for k in cpu:
        cpu[k].clear()
    decode_cpu.clear()
    gdec_cpu.clear()

    # the GPU decode of one batch's sources alone.  The stream is held behind a sleep kernel while decode() does its host
    # work (tables, records, staging), so the events bracket the device work only: the H2D copy of the records and the
    # three kernels.  The host time of the call is reported beside it.
    srcs = {i: i for i in plan.sources}
    cbytes = sum(jpegs[i].numel() for i in srcs)
    obytes = sum(src[i].nbytes for i in srcs)
    times, call_wall, call_cpu = [], [], []
    for r in range(args.steps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)
        e0.record(side)
        c0, w0 = time.process_time(), time.perf_counter()
        gdec.decode(srcs, stream=side, store=store)
        w1, c1 = time.perf_counter(), time.process_time()
        e1.record(side)
        assert not e0.query(), "the sleep ended before decode() had enqueued its work: the events would include host time"
        e1.synchronize()
        if r >= 2:
            times.append(e0.elapsed_time(e1))
            call_wall.append((w1 - w0) * 1e3)
            call_cpu.append((c1 - c0) * 1e3)
    gdec.check()
    t = float(np.median(times))
    print(json.dumps(dict(what="jpeg_decode_ms", images=len(srcs), device_ms=t, device_min_ms=min(times), device_max_ms=max(times),
                          images_per_s=len(srcs) / (t * 1e-3), compressed_MBps=cbytes / (t * 1e-3) / 1e6,
                          output_GBps=obytes / (t * 1e-3) / 1e9, compressed_mb=cbytes / 1e6,
                          call_wall_ms=float(np.median(call_wall)), call_cpu_ms=float(np.mean(call_cpu)),
                          note="device_ms: CUDA events around the decode's device work alone (record copy + 3 kernels); "
                               "call_*: host time of the decode() call", card=info)), flush=True)

    # step time: preloaded, then each feed, alternating in rounds
    random.seed(1)
    np.random.seed(1)
    plan = feeds["host"].draw(indices(0))
    tg = feeds["host"].submit(plan, src, labels)
    feeds["host"].wait()
    pre_imgs = step.images.clone()
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
    modes = ["preloaded"] + list(feeds)
    res = {k: [] for k in modes}
    for rep in range(args.reps + 1):                      # round 0 warms every feed up and is not kept
        for mode in modes:
            if mode != "preloaded":
                submit(mode, feeds[mode].draw(indices(0)))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(args.steps):
                if mode == "preloaded":
                    step.load(pre_imgs, tg)
                    step.run()
                else:
                    feeds[mode].wait()
                    step.run()
                    submit(mode, feeds[mode].draw(indices(j + 1)))
            torch.cuda.synchronize()
            if rep:
                res[mode].append((time.perf_counter() - t0) / args.steps * 1e3)
        if rep == 0:
            for k in cpu:
                cpu[k].clear()
            decode_cpu.clear()
            gdec_cpu.clear()
    gdec.check()
    print(json.dumps(dict(what="trainstep_ms", model="yolov6s", batch=B, size=S, steps=args.steps, reps=args.reps,
                          **{k: float(np.median(v)) for k, v in res.items()}, **{f"{k}_min": min(v) for k, v in res.items()},
                          **{f"{k}_max": max(v) for k, v in res.items()}, card=info)), flush=True)
    dc = np.array(decode_cpu)
    print(json.dumps(dict(what="submit_cpu_ms", batch=B, **{k: float(np.mean(v)) for k, v in cpu.items()},
                          calls={k: len(v) for k, v in cpu.items()}, decode_call_cpu=float(dc[:, 0].mean()),
                          decode_call_wall=float(dc[:, 1].mean()), decode_frames_per_call=float(dc[:, 2].mean()),
                          gpujpeg_call_cpu=float(np.mean([g[0] for g in gdec_cpu])), gpujpeg_call_wall=float(np.mean([g[1] for g in gdec_cpu])),
                          note="process time of all threads, mean over the calls (the clock may tick in 10 ms steps); "
                               "decode_call_*: torchvision decode_jpeg(device='cuda') of a batch's sources; "
                               "gpujpeg_call_*: yolov6_b200.jpeg's decode of the same sources from the device store",
                          card=info)), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    main(ap.parse_args())
