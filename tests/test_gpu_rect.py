"""GPU parity of minimum-rectangle serving (letterbox auto=True, the canvas Inferer.process_image gives): canvases and
rescaled rows against the reference's goldens (tests/golden/rect_cases.json, rect.npz), the three serving pipelines
against the eager chain letterbox_batch -> model -> non_max_suppression -> rescale_boxes, and every forward launch against
float64 at the rect canvases (the helpers of tests/test_gpu_forward_launches.py)."""
import hashlib

import numpy as np
import pytest
import torch

import test_gpu_forward_launches as fl
from conftest import golden_json, golden_npz
from oracle import letterbox as ol

pytestmark = pytest.mark.gpu

G = golden_json("rect_cases.json")["cases"]
NPZ = golden_npz("rect.npz")
KW = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)


def source(c):
    return ol.synthetic_source(c["h0"], c["w0"], c["kind"], c["seed"])


def as_frame(im, layout, dev=None):
    """The BGR HWC source as a host or CUDA frame in `layout` (rgb_chw: torchvision's decoders' RGB CHW)."""
    t = torch.from_numpy(im if layout == "bgr_hwc" else np.ascontiguousarray(im[..., ::-1].transpose(2, 0, 1)))
    return t.to(dev) if dev is not None else t


def by_canvas():
    groups = {}
    for k, c in enumerate(G):
        groups.setdefault((c["img_size"], c["stride"], c["H"], c["W"]), []).append(k)
    return groups


def test_rect_canvases_byte_identical_to_cv2():
    """Every golden case, one letterbox_batch(auto=True) per canvas with all of that canvas's sources in the batch, host
    and CUDA frames, bgr_hwc and rgb_chw."""
    from yolov6_b200.preprocess import letterbox_batch
    dev = torch.device("cuda:0")
    for (img, stride, H, W), idx in by_canvas().items():
        ims = [source(G[k]) for k in idx]
        for layout in ("bgr_hwc", "rgb_chw"):
            for on_dev in (False, True):
                frames = [as_frame(im, layout, dev if on_dev else None) for im in ims]
                canvas, meta = letterbox_batch(frames, img, img, layout=layout, device=dev, auto=True, stride=stride)
                assert tuple(canvas.shape) == (len(idx), 3, H, W) and (meta.H, meta.W) == (H, W)
                got = canvas.cpu().numpy()
                for j, k in enumerate(idx):
                    c = G[k]
                    digest = hashlib.sha256(np.ascontiguousarray(got[j]).tobytes()).hexdigest()
                    assert digest == c["canvas_sha256"], f"case {k} {(c['h0'], c['w0'])} at {img}/{stride} {layout} device={on_dev}"
                    assert meta.shapes[j][1][1] == (c["left"], c["top"])


def test_mixed_canvases_are_refused():
    from yolov6_b200.preprocess import letterbox_batch
    a, b = np.zeros((1080, 1920, 3), np.uint8), np.zeros((1920, 1080, 3), np.uint8)
    with pytest.raises(RuntimeError, match="1920 x 1080 frame letterboxes to a 640 x 384 canvas"):
        letterbox_batch([a, b], 640, 640, device=torch.device("cuda:0"), auto=True)


def test_rect_rescale_equals_inferer_rescale():
    """rescale_boxes with the meta of letterbox_batch(auto=True) on the goldens' NMS-like rows equals their
    Inferer.rescale(...).round(); rows beyond count come back zeroed."""
    from yolov6_b200.preprocess import letterbox_batch, rescale_boxes
    dev = torch.device("cuda:0")
    for (img, stride, H, W), idx in by_canvas().items():
        _, meta = letterbox_batch([source(G[k]) for k in idx], img, img, device=dev, auto=True, stride=stride)
        dets = [NPZ[f"c{k}_det"] for k in idx]
        out = torch.full((len(idx), max(d.shape[0] for d in dets) + 3, 6), 7.0)
        count = torch.zeros(len(idx), dtype=torch.int32)
        for j, d in enumerate(dets):
            n = d.shape[0] - j
            out[j, :n], count[j] = torch.from_numpy(d[:n]), n
        res = rescale_boxes(out.to(dev), count.to(dev), meta).cpu().numpy()
        for j, k in enumerate(idx):
            n = int(count[j])
            assert np.array_equal(res[j, :n], NPZ[f"c{k}_out"][:n]), (G[k]["h0"], G[k]["w0"], img, stride)
            assert not res[j, n:].any()


# ------------------------------------------------------------------------------------------------------ pipelines vs the eager chain
def model(name):
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    return randomize_(build_model(name, 80, torch.device("cuda:0")), seed=3).eval()


def eager(m, frames, img, stride, layout, B=2):
    """letterbox_batch(auto=True) -> model -> non_max_suppression -> rescale_boxes: Inferer.infer's `det` per frame, in a
    batch of B padded with all-border canvases as the pipelines' partial batches are."""
    from yolov6_b200.nms import non_max_suppression
    from yolov6_b200.preprocess import letterbox_batch, rect_canvas, rescale_boxes
    dev = torch.device("cuda:0")
    h0, w0 = frames[0].shape[:2] if layout == "bgr_hwc" else frames[0].shape[1:]
    out = torch.empty(B, 3, *rect_canvas(h0, w0, img, stride), dtype=torch.uint8, device=dev)
    canvas, meta = letterbox_batch(frames, img, img, out=out, layout=layout, auto=True, stride=stride)
    with torch.no_grad():
        det = non_max_suppression(m(canvas)[0], **KW)
    out = torch.zeros(B, KW["max_det"], 6, device=dev)
    count = torch.tensor([d.shape[0] for d in det], dtype=torch.int32, device=dev)
    for j, d in enumerate(det):
        out[j, :d.shape[0]] = d
    res = rescale_boxes(out, count, meta).cpu()
    return [res[j, :int(n)] for j, n in enumerate(count.tolist()[:len(frames)])]


def frames_of(shape, n, seed, layout="bgr_hwc", dev=None):
    return [as_frame(ol.synthetic_source(*shape, "grad" if i % 2 else "noise", seed + i), layout, dev) for i in range(n)]


def check_rows(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert torch.equal(g, w)
    return sum(g.shape[0] for g in got)


def test_pipeline_at_384x640_equals_eager():
    """YOLOv6-N at img_size 640 for 1080p: 1080p and 720p frames (the same canvas), host and CUDA, both layouts."""
    from yolov6_b200.pipeline import DetectPipeline
    m, dev = model("yolov6n"), torch.device("cuda:0")
    p = DetectPipeline(m, 2, 640, 640, raw_input=True, auto=True, source_shape=(1080, 1920), **KW)
    assert p.canvas == (384, 640)
    total = 0
    for layout, on_dev, seed in (("bgr_hwc", False, 0), ("rgb_chw", True, 10)):
        frs = frames_of((1080, 1920), 1, seed, layout, dev if on_dev else None) + frames_of((720, 1280), 1, seed + 5, layout)
        total += check_rows(p(frs, layout=layout), eager(m, frs, 640, 32, layout))
    with pytest.raises(RuntimeError, match="this batch's canvas is 384 x 640"):
        p(frames_of((1920, 1080), 1, 0))
    assert total > 0


def test_stream_at_640x384_equals_eager():
    """YOLOv6-N at img_size 640 for portrait 1080p, DetectStream: each batch rescaled one step later with its own rows."""
    from yolov6_b200.pipeline import DetectStream
    m, dev = model("yolov6n"), torch.device("cuda:0")
    ds = DetectStream(m, 2, 640, 640, raw_input=True, auto=True, source_shape=(1920, 1080), **KW)
    assert ds.canvas == (640, 384)
    batches = [frames_of((1920, 1080), 2, 20), frames_of((1920, 1080), 1, 30, dev=dev), frames_of((1920, 1080), 2, 40, dev=dev)]
    outs = []
    for frs in batches:
        ds.submit(frs)
        r = ds.collect()
        if r is not None:
            outs.append(r)
    ds.drain()
    while len(outs) < len(batches):
        outs.append(ds.collect())
    assert sum(check_rows(got, eager(m, frs, 640, 32, "bgr_hwc")) for frs, got in zip(batches, outs)) > 0


def test_farm_at_768x1280_equals_eager():
    """YOLOv6-N6 (stride 64) at img_size 1280 for 1080p, two-lane DetectFarm: each lane's rows equal the eager chain's."""
    from yolov6_b200.pipeline import DetectFarm
    m, dev = model("yolov6n6"), torch.device("cuda:0")
    farm = DetectFarm(m, 2, 1280, 1280, lanes=2, raw_input=True, auto=True, source_shape=(1080, 1920), **KW)
    assert farm.canvas == (768, 1280)
    batches = [frames_of((1080, 1920), 2, 50 + 10 * i, dev=dev if i % 2 else None) for i in range(4)]
    L, outs = len(farm.lanes), {}
    for i, frs in enumerate(batches):
        farm.submit(frs)
        r = farm.lanes[i % L].collect()
        if r is not None:
            outs[i - L] = r
    for ln, lane in enumerate(farm.lanes):
        with torch.cuda.stream(farm.streams[ln]):
            lane.drain()
    torch.cuda.synchronize()
    for i in range(len(batches)):
        if i not in outs:
            outs[i] = farm.lanes[i % L].collect()
    assert sum(check_rows(outs[i], eager(m, frs, 1280, 64, "bgr_hwc")) for i, frs in enumerate(batches)) > 0


# -------------------------------------------------------------------------------------------------- forward launches at rect canvases
RECT_CONFIGS = {
    "yolov6s_384x640_b8_u8": dict(cfg="yolov6s", N=8, H=384, W=640, u8=True),
    "yolov6s_640x384_b8_u8": dict(cfg="yolov6s", N=8, H=640, W=384, u8=True),
    "yolov6m_480x640_b2_u8": dict(cfg="yolov6m", N=2, H=480, W=640, u8=True),
    "yolov6n6_768x1280_b2_u8": dict(cfg="yolov6n6", N=2, H=768, W=1280, u8=True),
    "yolov6lite_s_192x320_b4_u8": dict(cfg="yolov6lite_s", N=4, H=192, W=320, u8=True),
}


@pytest.mark.parametrize("config", list(RECT_CONFIGS))
def test_every_inference_launch_matches_float64_at_rect_canvases(config, monkeypatch):
    """The launch-by-launch float64 check of tests/test_gpu_forward_launches.py at the canvases auto=True serves: 12-row
    P5 maps (384 x 640), their transpose, 4:3, P6 at 768 x 1280 and Lite at 192 x 320 (a 3 x 5 P6 map)."""
    monkeypatch.setitem(fl.CONFIGS, config, RECT_CONFIGS[config])
    fl.test_every_inference_launch_record_matches_float64(config)
