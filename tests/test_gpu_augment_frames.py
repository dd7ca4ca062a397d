"""Training from frames in GPU memory: AugmentFeed fed with CUDA frames (contiguous, crop views, torchvision's RGB CHW, mixed
with host frames) and from a FrameCache, against the reference's goldens (tests/golden/augment_cases.json / augment.npz,
and the specific and rect `samples` of rect_train_cases.json / rect_train.npz); a TrainStep fed from device frames and
from the cache against the same step fed from host frames; stream ordering with `ready=` and the lifetime of dropped
frames; and the refusals, which leave the feed and the cache untouched."""
import hashlib
import random

import numpy as np
import pytest
import torch

from conftest import golden_json, golden_keys, golden_npz
from oracle import augment as oa
from oracle import fabricate as fab

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
AUG = golden_json("augment_cases.json")
AUG_NPZ = golden_npz("augment.npz")
RECT = golden_json("rect_train_cases.json")
RECT_NPZ = golden_npz("rect_train.npz")
SRC = oa.dataset_sources()
LABELS = {i: oa.synthetic_labels(i) for i in SRC}
MAX_SRC = sum(s.nbytes for s in SRC.values())
SHAPES = [SRC[i].shape[:2] for i in range(len(oa.DATASET))]
CASES = [(c, AUG_NPZ) for c in AUG["cases"]] + [(c, RECT_NPZ) for c in RECT["samples"]]
MODES = ["device", "crop", "rgb_chw", "mixed", "cache_host", "cache_device", "cache_partial"]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def feed_of(case, **kw):
    from yolov6_b200.augment import AugmentFeed
    target = case.get("target")
    full = (case["img_size"],) * 2 if target == "rect" else (case["H"], case["W"])
    return AugmentFeed(len(case["batch"]), *full, case["hyp"], len(oa.DATASET), MAX_SRC, case["img_size"], device=DEV,
                       target=target, **kw)


def draw(feed, case):
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    return feed.draw(case["batch"], (case["H"], case["W"]) if case.get("target") == "rect" else None)


def device_frame(i):
    return torch.from_numpy(SRC[i]).to(DEV)


def crop_frame(i):
    """SRC[i] as a view into a larger CUDA frame: rows padded beyond 3 * w0, a non-zero origin."""
    h, w, _ = SRC[i].shape
    big = torch.randint(0, 256, (h + 3, w + 5, 3), dtype=torch.uint8, device=DEV)
    big[1:1 + h, 2:2 + w] = torch.from_numpy(SRC[i]).to(DEV)
    return big[1:1 + h, 2:2 + w]


def chw_frame(i):
    return torch.from_numpy(np.ascontiguousarray(SRC[i][..., ::-1].transpose(2, 0, 1))).to(DEV)


def check(feed, case, npz, targets):
    got = feed.images.cpu().numpy()
    assert got.shape[2:] == (case["H"], case["W"])
    bad = [k for k in range(len(case["batch"])) if sha(got[k]) != case["chw_sha256"][k]]
    assert not bad, f"{case['name']}: samples {bad} differ from the reference"
    ref = []
    for k in range(len(case["batch"])):
        lab = npz[f"{case['name']}_{k}_labels"].copy()
        lab[:, 0] = k
        ref.append(lab)
    ref = np.concatenate(ref, 0)
    assert np.array_equal(targets.numpy(), ref)
    dev_t = feed.targets.cpu().numpy()
    assert np.array_equal(dev_t[:len(ref)], ref) and (dev_t[len(ref):] == -1).all()


def submit_mode(feed, plan, mode):
    """Submit `plan` with its sources given as `mode` says; returns the host targets."""
    from yolov6_b200.augment import FrameCache
    srcs = plan.sources
    if mode in ("device", "crop", "rgb_chw"):
        make = dict(device=device_frame, crop=crop_frame, rgb_chw=chw_frame)[mode]
        return feed.submit(plan, {i: make(i) for i in srcs}, LABELS, layout="rgb_chw" if mode == "rgb_chw" else "bgr_hwc")
    if mode == "mixed":
        return feed.submit(plan, {i: device_frame(i) if k % 2 else SRC[i] for k, i in enumerate(srcs)}, LABELS)
    cache = FrameCache(SHAPES, feed.sampler, 1 << 30, device=DEV)
    feed.cache = cache
    if mode == "cache_host":
        cache.put({i: SRC[i] for i in srcs})
        return feed.submit(plan, {}, LABELS)
    if mode == "cache_device":
        cache.put({i: chw_frame(i) for i in srcs}, layout="rgb_chw")
        return feed.submit(plan, {}, LABELS)
    half = srcs[::2]                               # partly filled: the rest come as frames, host and device
    cache.put({i: device_frame(i) for i in half})
    rest = [i for i in srcs if i not in half]
    return feed.submit(plan, {i: SRC[i] if k % 2 else crop_frame(i) for k, i in enumerate(rest)}, LABELS)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ci", range(len(CASES)), ids=[c["name"] for c, _ in CASES])
def test_feed_from_device_frames_and_cache_equals_reference(ci, mode):
    case, npz = CASES[ci]
    feed = feed_of(case)
    plan = draw(feed, case)
    targets = submit_mode(feed, plan, mode)
    feed.wait()
    check(feed, case, npz, targets)


def test_cache_feeds_every_rect_batch_of_one_feed():
    """One rect feed and one cache, filled from device frames as the batches arrive, serve the four rect cases in a row."""
    from yolov6_b200.augment import FrameCache
    cases = [c for c in RECT["samples"] if c["target"] == "rect"]
    feed = feed_of(cases[0])
    cache = FrameCache(SHAPES, feed.sampler, 1 << 30, device=DEV)
    feed.cache = cache
    for case in cases:
        feed.sampler.hyp = dict(case["hyp"])
        plan = draw(feed, case)
        cache.put({i: device_frame(i) for i in plan.sources if not cache.cached[i]})
        targets = feed.submit(plan, {}, LABELS)
        feed.wait()
        check(feed, case, RECT_NPZ, targets)


def test_trainstep_fed_from_device_frames_and_cache_equals_host_frames():
    """Two batches with mixup: the step's run() tensor is the same whether its feed reads host frames, CUDA frames or the
    cache (test_feed_drives_trainstep_like_load's setting)."""
    from yolov6_b200.augment import AugmentFeed, FrameCache
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.step import TrainStep
    H = W = 256
    B = 4
    hyp = dict(AUG["cases"][1]["hyp"], mixup=0.5)
    sd = fab.fabricate_state_dict(golden_keys("yolov6n"), seed=0)
    m = build_model("yolov6n", 80, DEV)
    m.load_state_dict(sd)
    crit = ComputeLoss(num_classes=80, ori_img_size=H, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    step = TrainStep(m.train(), crit, B, H, W, in_dtype=torch.uint8)
    host_feed = AugmentFeed(B, H, W, hyp, len(oa.DATASET), MAX_SRC, step=step)
    dev_feed = AugmentFeed(B, H, W, hyp, len(oa.DATASET), MAX_SRC, step=step)
    cache = FrameCache(SHAPES, dev_feed.sampler, 1 << 30)
    cache.put({i: device_frame(i) for i in SRC})
    cache_feed = AugmentFeed(B, H, W, hyp, len(oa.DATASET), MAX_SRC, step=step, cache=cache)
    dev_frames = {i: device_frame(i) for i in SRC}
    mixed = 0
    for it, batch in enumerate(([0, 1, 2, 3], [8, 11, 12, 13])):
        outs = []
        for feed, frames in ((host_feed, SRC), (dev_feed, dev_frames), (cache_feed, {})):
            random.seed(40 + it)
            np.random.seed(40 + it)
            plan = feed.draw(batch)
            feed.submit(plan, frames, LABELS)
            feed.wait()
            outs.append(step.run().clone())
        mixed += sum(s.mix_r is not None for s in plan.samples)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (it, [o.tolist() for o in outs])
        assert float(outs[0][0]) > 0
    assert mixed > 0


def test_frames_written_on_a_side_stream_with_ready():
    """Frames a kernel writes on a side stream, behind a long kernel there, are read after the `ready` event."""
    case = AUG["cases"][0]
    feed = feed_of(case)
    plan = draw(feed, case)
    side = torch.cuda.Stream(DEV)
    host = {i: torch.from_numpy(SRC[i]).to(DEV) for i in plan.sources}
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)                   # keeps the side stream busy for tens of milliseconds
        frames = {i: host[i].flip(1).flip(1) for i in plan.sources}       # written by kernels on the side stream
        ready = torch.cuda.Event()
        ready.record(side)
    targets = feed.submit(plan, frames, LABELS, ready=ready)
    feed.wait()
    check(feed, case, AUG_NPZ, targets)


def test_dropped_frames_are_held_until_the_batch_is_built():
    """Frames dropped right after submit, then allocations of the same sizes written on the caller's stream, leave the
    batch unchanged: the feed holds the frames until their slot is reused."""
    case = AUG["cases"][0]
    feed = feed_of(case)
    plan = draw(feed, case)
    frames = {i: device_frame(i) for i in plan.sources}
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)                       # the caller's stream is busy, so the feed's resize waits
    targets = feed.submit(plan, frames, LABELS)
    del frames
    junk = [torch.empty(SRC[i].shape, dtype=torch.uint8, device=DEV).fill_(255) for i in plan.sources]
    feed.wait()
    check(feed, case, AUG_NPZ, targets)
    del junk


def test_cache_fill_holds_dropped_frames():
    from yolov6_b200.augment import FrameCache
    case = AUG["cases"][2]
    feed = feed_of(case)
    plan = draw(feed, case)
    cache = FrameCache(SHAPES, feed.sampler, 1 << 30, device=DEV)
    feed.cache = cache
    frames = {i: device_frame(i) for i in plan.sources}
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)
    cache.put(frames)
    del frames
    junk = [torch.empty(SRC[i].shape, dtype=torch.uint8, device=DEV).fill_(255) for i in plan.sources]
    targets = feed.submit(plan, {}, LABELS)
    feed.wait()
    check(feed, case, AUG_NPZ, targets)
    del junk


def test_refusals_leave_feed_and_cache_untouched():
    from yolov6_b200.augment import AugmentFeed, FrameCache
    case = AUG["cases"][2]
    feed = feed_of(case)
    plan = draw(feed, case)
    i = plan.sources[0]
    h, w, _ = SRC[i].shape
    good = {j: device_frame(j) for j in plan.sources}
    bad_frames = [
        (torch.empty(h, w, 3, dtype=torch.uint8, device="meta"), "bgr_hwc"),                   # another device
        (good[i].float(), "bgr_hwc"),                                                         # another dtype
        (good[i].permute(2, 0, 1).contiguous(), "bgr_hwc"),                                   # channels first, read as HWC
        (good[i], "rgb_chw"),                                                                 # channels last, read as CHW
        (good[i].permute(2, 0, 1).contiguous().permute(1, 2, 0), "bgr_hwc"),                  # innermost stride h * w
        (torch.zeros(h, w, 4, dtype=torch.uint8, device=DEV)[..., :3], "bgr_hwc"),            # pixel stride 4
    ]
    for fr, layout in bad_frames:
        with pytest.raises(RuntimeError):
            feed.submit(plan, {**good, i: fr}, LABELS, layout=layout)
    assert feed.ready is None

    with pytest.raises(RuntimeError, match="bytes"):
        FrameCache(SHAPES, feed.sampler, 1000, device=DEV)                                     # over max_bytes
    cache = FrameCache(SHAPES, feed.sampler, 1 << 30, device=DEV)
    with pytest.raises(RuntimeError, match="FrameCache"):                                     # another geometry
        AugmentFeed(len(case["batch"]), case["H"], case["W"], case["hyp"], len(oa.DATASET), MAX_SRC, case["img_size"] // 2,
                    device=DEV, cache=cache)
    with pytest.raises(RuntimeError):
        FrameCache(SHAPES[:-1], feed.sampler, 1 << 30, device=DEV)                             # shapes of another dataset
    with pytest.raises(RuntimeError, match="shapes_hw"):                                      # a frame of another size
        cache.put({i: good[i][1:]})
    with pytest.raises(RuntimeError):
        cache.put({i: good[i], plan.sources[1]: good[i].float()})                              # one bad frame: nothing filled
    assert not cache.cached.any() and cache.filled is None
    cache.put({i: good[i]})
    filled = cache.filled
    with pytest.raises(RuntimeError, match="already cached"):
        cache.put({i: good[i]})
    feed.cache = cache
    with pytest.raises(RuntimeError, match="no frame"):                                       # neither cached nor given
        feed.submit(plan, {}, LABELS)
    assert feed.ready is None and cache.filled is filled and cache.cached.sum() == 1
    targets = feed.submit(plan, good, LABELS)                                                 # the valid form passes
    feed.wait()
    check(feed, case, AUG_NPZ, targets)
