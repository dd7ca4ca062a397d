"""The JPEG decoder on the device against cv2.imread's bytes (tests/golden/jpeg*): every golden case alone and in one
mixed batch, from host bytes and from a JpegStore, twice; the status report of a stream cut short inside a batch; no
host synchronisation; and the feeds fed with decoded frames against the same plans fed with those frames on the host."""
import hashlib
import random

import cv2
import numpy as np
import pytest
import torch

from conftest import golden_json, golden_npz
from oracle import augment as oa

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
META = golden_json("jpeg_cases.json")
BLOBS = golden_npz("jpeg.npz")
CASES = META["cases"]
NAMES = sorted(CASES)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def blob(name):
    return BLOBS[name].tobytes()


def decode(srcs, **kw):
    from yolov6_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    frames, ready = dec.decode(srcs, **kw)
    dec.check()
    return {k: v.cpu().numpy() for k, v in frames.items()}


@pytest.mark.parametrize("name", NAMES)
def test_each_case_alone(name):
    got = decode({name: blob(name)})[name]
    assert list(got.shape) == CASES[name]["shape"] and sha(got) == CASES[name]["sha256"], name


def test_mixed_batch_host_and_store_twice():
    from yolov6_b200.jpeg import JpegDecoder, JpegStore
    store = JpegStore((blob(n) for n in NAMES), device=DEV, chunk_bytes=1 << 18)     # a generator; several chunks
    assert len(store.chunks) > 1
    dec = JpegDecoder(DEV)
    runs = [dec.decode({n: blob(n) for n in NAMES}), dec.decode({n: i for i, n in enumerate(NAMES)}, store=store),
            dec.decode({n: blob(n) for n in NAMES})]
    dec.check()
    for frames, _ in runs:
        bad = [n for n in NAMES if sha(frames[n].cpu().numpy()) != CASES[n]["sha256"]]
        assert not bad, bad


def test_stream_cut_short_is_flagged_and_the_rest_is_exact():
    from yolov6_b200.jpeg import JpegDecoder, parse
    good = blob("q90_opt0_333x500")
    a, e = parse(good).scan
    cut = good[:a + (e - a) // 2] + b"\xff\xd9"
    srcs = {"cut": cut, **{n: blob(n) for n in ("samp420_33x65", "rst7_333x500", "gray_333x500")}}
    dec = JpegDecoder(DEV)
    frames, _ = dec.decode(srcs)
    with pytest.raises(ValueError, match=r"'cut': entropy data ran out") as ei:
        dec.check()
    assert "samp420" not in str(ei.value)
    for n in srcs:
        if n != "cut":
            assert sha(frames[n].cpu().numpy()) == CASES[n]["sha256"], n


def test_decode_does_not_synchronise_the_host():
    from yolov6_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    dec.decode({0: blob("size_481x640")})          # library load, handle
    dec.check()
    side = torch.cuda.Stream(DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)             # keeps the decode stream busy for tens of milliseconds
    frames, ready = dec.decode({n: blob(n) for n in NAMES}, stream=side)
    assert not ready.query(), "decode waited for its stream"
    dec.check()
    assert sha(frames["size_1080x1920"].cpu().numpy()) == CASES["size_1080x1920"]["sha256"]


# ---- the feeds, fed with decoded frames, against the same plans fed with those frames from the host ----
SRC = oa.dataset_sources()
JPG = {i: cv2.imencode(".jpg", s, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes() for i, s in SRC.items() if min(s.shape[:2]) > 0}
LABELS = {i: oa.synthetic_labels(i) for i in SRC}


def decoded(indices, side):
    from yolov6_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)
    frames, ready = dec.decode({i: JPG[i] for i in indices}, stream=side)
    return dec, frames, ready


def test_augment_feed_and_cache_from_decoded_frames():
    from yolov6_b200.augment import HYP_YOLOV6S, AugmentFeed, FrameCache
    n = len(SRC)
    shapes = [SRC[i].shape[:2] for i in range(n)]
    batch = list(range(min(4, n)))
    max_src = sum(s.nbytes for s in SRC.values())
    out = []
    for mode in ("host", "device", "cache"):
        feed = AugmentFeed(len(batch), 320, 320, HYP_YOLOV6S, n, max_src, 320, device=DEV)
        random.seed(3)
        np.random.seed(3)
        plan = feed.draw(batch)
        side = torch.cuda.Stream(DEV)
        dec, frames, ready = decoded(plan.sources, side)
        if mode == "host":
            dec.check()
            targets = feed.submit(plan, {i: f.cpu().numpy() for i, f in frames.items()}, LABELS)
        elif mode == "device":
            targets = feed.submit(plan, frames, LABELS, ready=ready)
        else:
            feed.cache = FrameCache(shapes, feed.sampler, 1 << 30, device=DEV)
            feed.cache.put(frames, ready=ready)
            targets = feed.submit(plan, {}, LABELS)
        feed.wait()
        dec.check()
        if mode == "host":
            for i, f in frames.items():
                assert np.array_equal(f.cpu().numpy(), cv2.imdecode(np.frombuffer(JPG[i], np.uint8), cv2.IMREAD_COLOR))
        out.append((feed.images.cpu().numpy(), targets.cpu().numpy() if torch.is_tensor(targets) else np.asarray(targets)))
    for imgs, tg in out[1:]:
        assert np.array_equal(imgs, out[0][0]) and np.array_equal(tg, out[0][1])


def test_val_feed_from_decoded_frames():
    from yolov6_b200.valdata import ValFeed
    shapes = [SRC[i].shape[:2] for i in range(len(SRC))]
    res = []
    for on_dev in (False, True):
        feed = ValFeed(4, 320, 32, shapes, device=DEV)
        idx = [int(i) for i in feed.batches()[1]]
        side = torch.cuda.Stream(DEV)
        dec, frames, ready = decoded(idx, side)
        if on_dev:
            torch.cuda.current_stream(DEV).wait_event(ready)
            fr = [frames[i] for i in idx]
        else:
            dec.check()
            fr = [frames[i].cpu().numpy() for i in idx]
        canvas, targets, shp, n = feed.feed(list(idx), fr, [LABELS[i] for i in idx])
        dec.check()
        res.append((canvas.cpu().numpy(), targets.numpy(), shp, n))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1]) and res[0][2:] == res[1][2:]


def test_detect_stream_from_decoded_frames():
    """A raw_input DetectStream fed decoded frames with `ready=` gives the rows of the same frames fed from the host."""
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectStream
    from yolov6_b200.synth import randomize_
    m = randomize_(build_model("yolov6n", 80, DEV), seed=3).eval()
    kw = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)
    idx = sorted(JPG)
    groups = [idx[j:j + 4] for j in range(0, 12, 4)]
    rows = []
    for on_dev in (True, False):
        ds = DetectStream(m, 4, 192, 192, raw_input=True, max_src_bytes=32 << 20, **kw)
        side = torch.cuda.Stream(DEV)
        outs, keep = [], []
        for g in groups:
            dec, frames, ready = decoded(g, side)
            keep.append(frames)
            if on_dev:
                ds.submit([frames[i] for i in g], ready=ready)
            else:
                dec.check()
                ds.submit([frames[i].cpu().numpy() for i in g])
            r = ds.collect()
            if r is not None:
                outs.append(r)
            if on_dev:
                dec.check()
        ds.drain()
        while len(outs) < len(groups):
            outs.append(ds.collect())
        rows.append([[t.numpy() for t in r] for r in outs])
    assert len(rows[0]) == len(rows[1]) == len(groups)
    for a, b in zip(*rows):
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    assert sum(len(x) for r in rows[0] for x in r) > 0
