"""GPU parity of device-resident frames: CUDA tensors letterboxed in place by yv6_letterbox_frames (contiguous BGR HWC, crop
views of larger frames, RGB CHW as torchvision's decoders return it, and batches that mix them with host frames) give the
cv2 canvases of tests/golden/letterbox_cases.json, and the raw-frame pipelines serve them with the rows of the reference
composition -- also when the frames are produced on another stream right before `submit` or dropped right after it."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import golden_json
from oracle import letterbox as ol
from test_gpu_letterbox import SIZES_A, SIZES_B, by_canvas, expected, frames

pytestmark = pytest.mark.gpu

G = golden_json("letterbox_cases.json")
DEV = torch.device("cuda:0")
KW = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)


def hwc(im):
    return torch.from_numpy(im).to(DEV)


def crop(im, seed):
    """`im` as a crop view of a larger noise frame whose first byte lies at an odd address."""
    h, w = im.shape[:2]
    g = torch.Generator().manual_seed(seed)
    flat = torch.randint(0, 256, (1 + (h + 7) * (w + 13) * 3,), dtype=torch.uint8, generator=g)
    flat[1:].view(h + 7, w + 13, 3)[3:3 + h, 5:5 + w] = torch.from_numpy(im)
    return flat.to(DEV)[1:].view(h + 7, w + 13, 3)[3:3 + h, 5:5 + w]


def chw(im):
    """BGR HWC -> the RGB CHW of torchvision.io.decode_jpeg."""
    return torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1].transpose(2, 0, 1))).to(DEV)


def chw_crop(im, seed):
    h, w = im.shape[:2]
    g = torch.Generator().manual_seed(seed)
    big = torch.randint(0, 256, (3, h + 4, w + 9), dtype=torch.uint8, generator=g)
    big[:, 2:2 + h, 6:6 + w] = torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1].transpose(2, 0, 1)))
    return big.to(DEV)[:, 2:2 + h, 6:6 + w]


FORMS = {
    "hwc": ("bgr_hwc", lambda im, k: hwc(im)),
    "crop": ("bgr_hwc", crop),
    "chw": ("rgb_chw", lambda im, k: chw(im)),
    "chw_crop": ("rgb_chw", chw_crop),
    "mixed": ("bgr_hwc", lambda im, k: hwc(im) if k % 2 else im),           # host numpy and device frames in one batch
    "mixed_chw": ("rgb_chw", lambda im, k: chw(im) if k % 2 == 0 else np.ascontiguousarray(im[:, :, ::-1].transpose(2, 0, 1))),
}


@pytest.mark.parametrize("form", list(FORMS))
def test_device_frames_canvases_byte_identical_to_cv2(form):
    from yolov6_b200.preprocess import letterbox_batch
    layout, make = FORMS[form]
    for (H, W), idx in by_canvas(ol.CASES).items():
        for su in (True, False):
            sel = [i for i in idx if ol.CASES[i][4] == su]
            if not sel:
                continue
            ims = [ol.synthetic_source(ol.CASES[i][0], ol.CASES[i][1], ol.CASES[i][5], i) for i in sel]
            srcs = [make(im, k) for k, im in enumerate(ims)]
            canvas, meta = letterbox_batch(srcs, H, W, scaleup=su, device=DEV, layout=layout)
            got = canvas.cpu().numpy()
            for k, i in enumerate(sel):
                c = G["cases"][i]
                if hashlib.sha256(np.ascontiguousarray(got[k]).tobytes()).hexdigest() != c["canvas_sha256"]:
                    ref = ol.letterbox(ims[k], H, W, su)
                    diff = np.abs(got[k].astype(np.int64) - ref.astype(np.int64))
                    pytest.fail(f"{form} case {i} {ol.CASES[i]}: {int((diff > 0).sum())} bytes differ, max {int(diff.max())}")
                assert meta.shapes[k][1][1] == (c["left"], c["top"])


def as_form(frs, form, seed=0):
    layout, make = FORMS[form]
    return [make(f, seed + k) for k, f in enumerate(frs)], layout


# (sizes, seed, form): successive batches of one pipeline change size mix, batch fill, layout and where the frames are
BATCHES = [(SIZES_A, 0, "hwc"), (SIZES_B, 10, "mixed"), (SIZES_A[::-1], 20, "chw"), (SIZES_B[:2], 30, "crop"), (SIZES_A, 40, "mixed_chw")]


@pytest.fixture(scope="module")
def model_and_refs():
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    m = randomize_(build_model("yolov6n", 80, DEV), seed=3).eval()
    refs = [expected(m, frames(sizes, seed), 4, 192, KW) for sizes, seed, _ in BATCHES]
    return m, refs


def check_rows(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert np.array_equal(g.numpy(), r)


def test_pipeline_device_frames(model_and_refs):
    """DetectPipeline: one captured graph serves device, host, mixed and both layouts; malformed frames raise before anything
    is enqueued and the pipeline keeps serving correct batches."""
    from yolov6_b200.pipeline import DetectPipeline
    m, refs = model_and_refs
    p = DetectPipeline(m, 4, 192, 192, raw_input=True, max_src_bytes=4 << 20, **KW)
    graph = p.graph
    total = 0
    for (sizes, seed, form), ref in zip(BATCHES, refs):
        frs, layout = as_form(frames(sizes, seed), form, seed)
        got = p(frs, layout=layout)
        check_rows(got, ref)
        total += sum(g.shape[0] for g in got)
        assert p.graph is graph
    assert total > 0
    good, layout = as_form(frames(SIZES_A, 0), "hwc")
    for bad, lay in (([good[0].float()], "bgr_hwc"), ([good[0]], "rgb_chw"), ([good[0].permute(2, 0, 1)], "bgr_hwc"),
                     ([torch.zeros(20, 20, 4, dtype=torch.uint8, device=DEV)[:, :, :3]], "bgr_hwc")):
        with pytest.raises(RuntimeError):
            p(bad, layout=lay)
    check_rows(p(good, layout=layout), refs[0])


def stream_rows(ds, batches, submit):
    outs = []
    for b in batches:
        submit(b)
        r = ds.collect()
        if r is not None:
            outs.append(r)
    ds.drain()
    while len(outs) < len(batches):
        outs.append(ds.collect())
    return outs


def test_stream_device_frames(model_and_refs):
    """DetectStream (including drain) with device / mixed frames and both layouts; the two step graphs are captured once."""
    from yolov6_b200.pipeline import DetectStream
    m, refs = model_and_refs
    ds = DetectStream(m, 4, 192, 192, raw_input=True, max_src_bytes=4 << 20, **KW)
    graphs = list(ds.graphs) + list(ds.drain_graphs)
    batches = [as_form(frames(sizes, seed), form, seed) for sizes, seed, form in BATCHES]
    outs = stream_rows(ds, batches, lambda b: ds.submit(b[0], layout=b[1]))
    for got, ref in zip(outs, refs):
        check_rows(got, ref)
    assert all(a is b for a, b in zip(graphs, list(ds.graphs) + list(ds.drain_graphs)))


def farm_rows(farm, batches, submit):
    """Batch j goes to lane j % lanes; each lane's batches are collected in order, the last ones after a drain on the lane's
    stream (as tests/test_gpu_nms.py feeds a farm)."""
    outs, nxt, L = {}, list(range(len(farm.lanes))), len(farm.lanes)
    for j, b in enumerate(batches):
        submit(b)
        r = farm.lanes[j % L].collect()
        if r is not None:
            outs[nxt[j % L]] = r
            nxt[j % L] += L
    for ln, lane in enumerate(farm.lanes):
        with torch.cuda.stream(farm.streams[ln]):
            lane.drain()
        torch.cuda.synchronize()
        r = lane.collect()
        if r is not None:
            outs[nxt[ln]] = r
    assert sorted(outs) == list(range(len(batches)))
    return [outs[j] for j in range(len(batches))]


def test_farm_device_frames(model_and_refs):
    from yolov6_b200.pipeline import DetectFarm
    m, refs = model_and_refs
    farm = DetectFarm(m, 4, 192, 192, lanes=2, raw_input=True, max_src_bytes=4 << 20, **KW)
    batches = [as_form(frames(sizes, seed), form, seed) for sizes, seed, form in BATCHES]
    for got, ref in zip(farm_rows(farm, batches, lambda b: farm.submit(b[0], layout=b[1])), refs):
        check_rows(got, ref)


def fill_late(frs_np, stream):
    """Device frames written on `stream` after a ~20 ms kernel: a reader not ordered after `stream` sees zeros."""
    out = [torch.zeros(f.shape, dtype=torch.uint8, device=DEV) for f in frs_np]
    src = [hwc(f) for f in frs_np]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(40_000_000)
        for o, s in zip(out, src):
            o.copy_(s, non_blocking=True)
    return out


def test_producer_on_side_stream_and_dropped_frames(model_and_refs):
    """Frames written by kernels still running on the caller's (side) stream at `submit` time, and frames the caller drops
    right after `submit` while allocating and overwriting new tensors of the same sizes, give the reference rows."""
    from yolov6_b200.pipeline import DetectFarm, DetectStream
    m, refs = model_and_refs
    side = torch.cuda.Stream(device=DEV)
    batches = [frames(sizes, seed) for sizes, seed, _ in BATCHES[:3]]
    with torch.cuda.stream(side):
        ds = DetectStream(m, 4, 192, 192, raw_input=True, max_src_bytes=4 << 20, **KW)
        outs = stream_rows(ds, batches, lambda b: ds.submit(fill_late(b, side)))
    farm = DetectFarm(m, 4, 192, 192, lanes=2, raw_input=True, max_src_bytes=4 << 20, **KW)

    def submit_and_drop(b):
        with torch.cuda.stream(side):
            farm.submit(fill_late(b, side))          # the frames go out of scope here
            junk = [torch.full(f.shape, 255, dtype=torch.uint8, device=DEV) for f in b]     # would reuse their blocks
            del junk
    farm_outs = farm_rows(farm, batches, submit_and_drop)
    for got, ref in zip(outs, refs):
        check_rows(got, ref)
    for got, ref in zip(farm_outs, refs):
        check_rows(got, ref)
