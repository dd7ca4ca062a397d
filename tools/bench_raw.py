"""Serving from decoded frames: 1920x1080 uint8 frames -> detections in source pixels, YOLOv6-S bs32 at 640 (bf16,
seeded synthetic weights, bench.py's NMS settings), frames/s for several ways of feeding the same DetectStream settings:

  raw:  raw_input=True -- host BGR frames: their bytes go to pinned staging and are letterboxed on the GPU
        (yv6_letterbox_frames), boxes are rescaled on the GPU (yv6_rescale_boxes);
  dev:  raw_input=True -- the same frames uploaded to the GPU once and submitted as CUDA tensors, letterboxed in place;
  jpeg: (--jpeg) raw_input=True -- the same frames encoded once with cv2.imencode; each step decodes its batch on the GPU
        (torchvision.io.decode_jpeg(..., device="cuda"), RGB CHW) and submits the decoder's tensors with layout="rgb_chw",
        so no raw pixel touches the host.  Uniform noise is JPEG's worst case: large files, slow entropy decoding;
  gpujpeg: (--jpeg) the same JPEG bytes decoded by yolov6_b200.jpeg (cv2.imread's pixels, BGR HWC), staged from the host,
        and submitted with the decode's `ready` event; its decode of one batch alone is timed as device work (CUDA
        events) and as host time of the call;
  cv2:  the reference's host path -- data_augment.letterbox (cv2.resize + copyMakeBorder, auto=False) + HWC->CHW + BGR->RGB on
        all host cores into the pinned uint8 batch, then the existing pipeline (rescale not included).

Each timed step prepares one batch, submits it and collects the previous one; the clock stops after the last batch is
collected.  The feeds alternate within each of `--runs` runs.  Each run also times yv6_letterbox_frames alone with CUDA
events (bs32, 1080p -> 640, both layouts) and reports the bytes it must move -- the distinct source rows its taps read plus
the canvas -- over that time.  One JSON line per run.

    python tools/bench_raw.py [--steps 20] [--warmup 3] [--runs 2] [--jpeg]
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


def sampled_rows(h0, nh):
    """Distinct source rows that cv2's INTER_LINEAR vertical taps read for an h0 -> nh resize (yv6_resize.cuh lin_tap)."""
    scale = 1.0 / (nh / h0)
    f = ((np.arange(nh, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    return len(np.unique(np.clip(np.concatenate([s, s + 1]), 0, h0 - 1)))


def time_letterbox(frames_dev, S, iters=200):
    """yv6_letterbox_frames alone on device frames of one layout: ms per launch (CUDA events), GB/s of the bytes it must move."""
    from yolov6_b200.preprocess import GEO, REC, check_frames, letterbox_frames_launch, letterbox_geometry, pack_sources
    frs, layout = frames_dev
    B, dev = len(frs), frs[0].device
    geo, rec = torch.empty(B, GEO, dtype=torch.int32), torch.empty(B * REC, dtype=torch.uint8)
    pack_sources(check_frames(frs, B, layout, dev), B, S, S, True, layout, torch.empty(1, dtype=torch.uint8), geo, rec, 0)
    geo_dev, rec_dev = geo.to(dev), rec.to(dev)
    out = torch.empty(B, 3, S, S, dtype=torch.uint8, device=dev)
    for _ in range(20):
        letterbox_frames_launch(rec_dev, geo_dev, out)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        letterbox_frames_launch(rec_dev, geo_dev, out)
    t1.record()
    t1.synchronize()
    ms = t0.elapsed_time(t1) / iters
    nbytes = out.numel()
    for row in geo.tolist():
        h0, w0, nh = row[1], row[2], row[3]
        nbytes += sampled_rows(h0, nh) * w0 * 3
    return {"ms": round(ms, 4), "bytes_mb": round(nbytes / 1e6, 1), "gb_per_s": round(nbytes / ms / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--jpeg", action="store_true", help="also feed GPU-decoded JPEGs (torchvision.io.decode_jpeg on CUDA)")
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

    frames_dev = [[torch.from_numpy(f).to(dev) for f in fs] for fs in frames]
    chw_dev = [f.flip(2).permute(2, 0, 1).contiguous() for f in frames_dev[0]]          # what decode_jpeg returns: RGB CHW

    # the raw, dev and jpeg feeds share one raw-frame DetectStream (staging sized for a batch of host frames); each run()
    # drains it, so the feeds can alternate
    raw = DetectStream(model, B, S, S, raw_input=True, max_src_bytes=B * 1080 * 1920 * 3, **NMS_KW)
    host = DetectStream(model, B, S, S, host_input=True, **NMS_KW)
    batch = torch.empty(B, 3, S, S, dtype=torch.uint8)
    view = batch.numpy()

    def feed_cv2(i):
        def one(j):
            view[j] = cv2_letterbox_chw(frames[i & 1][j], S)
        list(pool.map(one, range(B)))
        host.submit(batch)

    feeds = {"raw": (raw, lambda i: raw.submit(frames[i & 1])),
             "dev": (raw, lambda i: raw.submit(frames_dev[i & 1]))}
    jpeg_mb = None
    if args.jpeg:
        import cv2
        from torchvision.io import decode_jpeg
        jpegs = [[torch.from_numpy(cv2.imencode(".jpg", f)[1].reshape(-1)) for f in fs] for fs in frames]
        jpeg_mb = round(sum(j.numel() for j in jpegs[0]) / B / 1e6, 2)
        feeds["jpeg"] = (raw, lambda i: raw.submit(decode_jpeg(jpegs[i & 1], device=dev), layout="rgb_chw"))
        from yolov6_b200.jpeg import JpegDecoder
        gdec = JpegDecoder(dev)
        jpeg_bytes = [[j.numpy().tobytes() for j in js] for js in jpegs]

        def feed_gpujpeg(i):
            frames, ready = gdec.decode(dict(enumerate(jpeg_bytes[i & 1])))
            raw.submit([frames[j] for j in range(B)], ready=ready)
        feeds["gpujpeg"] = (raw, feed_gpujpeg)

        def gpujpeg_ms(n=5):
            """This project's decode of one batch from host bytes: (device ms, call ms).  The device work alone (H2D of
            the staged bytes + the kernels) between CUDA events, the stream held behind a sleep kernel until the call has
            enqueued it; and the host wall time of the call."""
            times, calls = [], []
            for i in range(n + 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                torch.cuda._sleep(1_000_000_000)
                e0.record()
                w0 = time.perf_counter()
                gdec.decode(dict(enumerate(jpeg_bytes[i & 1])))
                calls.append((time.perf_counter() - w0) * 1e3)
                e1.record()
                assert not e0.query(), "the sleep ended before decode() had enqueued its work"
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            gdec.check()
            return round(float(np.median(times[1:])), 2), round(float(np.median(calls[1:])), 2)

        def decode_ms(n=5):
            """The decode of one batch alone: host clock around decode_jpeg + a device synchronise."""
            decode_jpeg(jpegs[0], device=dev)
            torch.cuda.synchronize()
            t = time.perf_counter()
            for i in range(n):
                decode_jpeg(jpegs[i & 1], device=dev)
            torch.cuda.synchronize()
            return round((time.perf_counter() - t) / n * 1e3, 1)
    feeds["cv2"] = (host, feed_cv2)

    for r in range(args.runs):
        fps = {name: round(run(ds, feed, args.steps, args.warmup), 1) for name, (ds, feed) in feeds.items()}
        kernel = {"bgr_hwc": time_letterbox((frames_dev[0], "bgr_hwc"), S), "rgb_chw": time_letterbox((chw_dev, "rgb_chw"), S)}
        line = {"metric": f"frames/s 1920x1080 BGR -> detections, YOLOv6-S {S} bs{B}", "raw_frames_per_s": fps["raw"],
                "cv2_host_frames_per_s": fps["cv2"], "dev_frames_per_s": fps["dev"], "letterbox_frames_kernel": kernel,
                "host_threads": threads, "steps": args.steps, "run": r, "gpu": gpu_info(0)}
        if args.jpeg:
            line.update(jpeg_frames_per_s=fps["jpeg"], jpeg_mb_per_frame=jpeg_mb, jpeg_decode_ms_per_batch=decode_ms(),
                        gpujpeg_frames_per_s=fps["gpujpeg"], gpujpeg_decode_ms_per_batch=dict(zip(("device", "call"), gpujpeg_ms())))
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
