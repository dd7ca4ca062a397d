"""Minimum-rectangle letterboxing (letterbox auto=True, Inferer.process_image's default) on the CPU: the geometry against
the reference's goldens (tests/golden/rect_cases.json, written by tests/golden/make_golden_rect.py), and a replay of the
serving pipelines built with auto=True on the recorder of tests/test_serving_plan.py -- which shape each engine is pinned
and captured at, what the letterbox, NMS and rescale launches are given, and that a frame with another canvas is refused
before anything is staged."""
import numpy as np
import pytest
import torch

import test_serving_plan as tsp
from conftest import golden_json
from yolov6_b200 import pipeline
from yolov6_b200.preprocess import check_frames, common_canvas, inferer_size, inferer_stride, letterbox_geometry, rect_canvas

G = golden_json("rect_cases.json")["cases"]


@pytest.mark.parametrize("k", range(len(G)))
def test_rect_canvas_and_geometry_equal_the_reference(k):
    c = G[k]
    H, W = inferer_size(c["img_size"], c["stride"])
    assert [H, W] == c["checked"]
    assert rect_canvas(c["h0"], c["w0"], c["img_size"], c["stride"]) == (c["H"], c["W"])
    assert c["H"] % c["stride"] == 0 and c["W"] % c["stride"] == 0
    r, (nw, nh), top, left = letterbox_geometry(c["h0"], c["w0"], H, W, True, auto=True, stride=c["stride"])
    assert (r, top, left) == (c["r"], c["top"], c["left"])
    assert (nw, nh) == (int(round(c["w0"] * c["r"])), int(round(c["h0"] * c["r"])))
    assert top + nh <= c["H"] and left + nw <= c["W"]


def test_inferer_stride_and_auto_false_geometry():
    assert inferer_stride([8, 16, 32]) == 32 and inferer_stride([8, 16, 32, 64]) == 64 and inferer_stride([8, 16]) == 32
    assert inferer_size(600, 32) == (608, 608) and inferer_size((300, 641), 64) == (320, 704)
    for h0, w0, H, W in ((1080, 1920, 640, 640), (333, 517, 320, 640), (3, 5, 64, 96)):
        assert letterbox_geometry(h0, w0, H, W, True, auto=False, stride=32) == letterbox_geometry(h0, w0, H, W, True)


def test_common_canvas_names_both_shapes():
    frames = [np.zeros((1080, 1920, 3), np.uint8), np.zeros((720, 1280, 3), np.uint8), np.zeros((1920, 1080, 3), np.uint8)]
    srcs = check_frames(frames, 3, "bgr_hwc", torch.device("cpu"))
    assert common_canvas(srcs[:2], 640, 640, True, 32) == (384, 640)
    with pytest.raises(RuntimeError, match=r"1920 x 1080 frame letterboxes to a 640 x 384 canvas, a 1080 x 1920 frame .* 384 x 640"):
        common_canvas(srcs, 640, 640, True, 32)


# --------------------------------------------------------------------------------------------------------------- serving replay
def golden(h0, w0, img_size):
    return next(c for c in G if (c["h0"], c["w0"], c["img_size"]) == (h0, w0, img_size))


def ref_row(c):
    """The geometry row (without the byte offset) the reference's numbers give: h0, w0, nh, nw, top, left, 0."""
    return [c["h0"], c["w0"], int(round(c["h0"] * c["r"])), int(round(c["w0"] * c["r"])), c["top"], c["left"], 0]


def frame(h0, w0, layout="bgr_hwc", device=None):
    shape = (h0, w0, 3) if layout == "bgr_hwc" else (3, h0, w0)
    return torch.full(shape, 7, dtype=torch.uint8, device=device)


class Watch:
    """Snapshots of the letterbox, NMS and rescale launches as they run (at graph replay): canvas, level sizes and the
    geometry rows of the table each one reads."""

    def __init__(self, monkeypatch):
        self.lb, self.nms, self.rescale = [], [], []

        def letterbox(rec, h, rec_dev, geo, Bn, H, W, out, stream):
            self.lb.append(((H, W), tsp._array(geo, tsp.C.c_int32, Bn * 8).reshape(Bn, 8).tolist()))

        def nms(rec, h, cls, reg, Bn, nc, R, nl, lh, lw, *rest):
            self.nms.append([(lh[i], lw[i]) for i in range(nl)])
            tsp.nms_effect(rec, h, cls, reg, Bn, nc, R, nl, lh, lw, *rest)

        def rescale(rec, h, out, count, geo, Bn, max_det, H, W, res, stream):
            self.rescale.append(((H, W), tsp._array(geo, tsp.C.c_int32, Bn * 8).reshape(Bn, 8).tolist()))
            tsp.rescale_effect(rec, h, out, count, geo, Bn, max_det, H, W, res, stream)
        monkeypatch.setitem(tsp.EFFECTS, "yv6_letterbox_frames", letterbox)
        monkeypatch.setitem(tsp.EFFECTS, "yv6_nms_batched_head", nms)
        monkeypatch.setitem(tsp.EFFECTS, "yv6_rescale_boxes", rescale)


def served(cfg, monkeypatch, run):
    rec = tsp.ServingRecorder()
    engines = [tsp.dry(rec, cfg)]

    def lane():
        engines.append(tsp.dry(rec, cfg))
        return engines[-1]
    with tsp.stand_ins(rec, lane), torch.no_grad():
        run(rec, tsp.Model(engines[0]), Watch(monkeypatch), engines)


def assert_built_at(p, engines, canvas, strides):
    assert p.canvas == canvas
    for eng in engines:
        assert {k[1:3] for k in eng._pinned} == {canvas} and {k[1:3] for k in eng._plans} == {canvas}
    for ds in getattr(p, "lanes", [p]):
        assert ds.sizes == [(canvas[0] // s, canvas[1] // s) for s in strides]
        assert all(tuple(s.x_dev.shape[2:]) == canvas for s in ds.slots)


def refused(rec, p, slot, frames, match, **kw):
    """`frames` raise RuntimeError before anything is copied, cleared or launched, and leave the slot's staging tables as
    they were."""
    tables = [t.clone() for t in (slot.geo_host, slot.rec_host, slot.src_host)]
    nbytes, staged, n = slot.nbytes, list(slot.frames), len(rec.log)
    with pytest.raises(RuntimeError, match=match):
        p(frames, **kw)
    # what may come before the staging: waiting for the slot's previous step, recording the frames' producer
    assert all(e["fn"] in ("event_synchronize", "record_event") for e in rec.log[n:]), rec.log[n:]
    assert all(torch.equal(a, b) for a, b in zip(tables, (slot.geo_host, slot.rec_host, slot.src_host)))
    assert slot.nbytes == nbytes and slot.frames == staged


def test_pipeline_auto_serves_on_the_rect_canvas(monkeypatch):
    """DetectPipeline, YOLOv6-N at img_size 640 for 1080p: built at 384 x 640; 1080p and 720p frames, host and device, in
    both layouts, are letterboxed with the reference's rows and rescaled from that canvas; a portrait frame is refused."""
    c1080, c720 = golden(1080, 1920, 640), golden(720, 1280, 640)

    def run(rec, m, w, engines):
        p = pipeline.DetectPipeline(m, 2, 640, 640, raw_input=True, auto=True, source_shape=(1080, 1920))
        assert_built_at(p, [m.eng], (384, 640), m.graph.strides)
        w.lb.clear(), w.nms.clear(), w.rescale.clear()          # the warm-up and capture runs
        got = p([frame(1080, 1920), frame(720, 1280)])
        assert len(got) == 2
        got = p([frame(720, 1280, "rgb_chw", "cuda")], layout="rgb_chw")
        assert len(got) == 1
        assert [x[0] for x in w.lb] == [(384, 640)] * 2 and [x[0] for x in w.rescale] == [(384, 640)] * 2
        assert w.nms == [[(48, 80), (24, 40), (12, 20)]] * 2
        assert [r[1:] for r in w.lb[0][1]] == [ref_row(c1080), ref_row(c720)]
        assert [r[1:] for r in w.lb[1][1]] == [ref_row(c720), [384, 640, 0, 0, 0, 0, 0]]
        assert w.rescale[0][1] == w.lb[0][1] and w.rescale[1][1] == w.lb[1][1]
        refused(rec, p, p.slot, [frame(720, 1280), frame(1920, 1080)], r"1920 x 1080 frame letterboxes to a 640 x 384 canvas")
        refused(rec, p, p.slot, [frame(480, 640)], r"480 x 640 frame letterboxes to a 480 x 640 canvas .* this batch's canvas is 384 x 640")
        assert len(p([frame(1080, 1920)])) == 1
        assert w.lb[-1][0] == (384, 640) and w.lb[-1][1][0][1:] == ref_row(c1080)
    served("yolov6n", monkeypatch, run)


def test_stream_auto_default_stride_64(monkeypatch):
    """DetectStream, YOLOv6Lite-S (strides up to 64, so Inferer pads to 64) at img_size 320 for 720p: built at 192 x 320;
    each batch is letterboxed in its step and rescaled in the next with its own rows."""
    c1080, c720 = golden(1080, 1920, 320), golden(720, 1280, 320)

    def run(rec, m, w, engines):
        ds = pipeline.DetectStream(m, 2, 320, 320, raw_input=True, auto=True, source_shape=(720, 1280))
        assert_built_at(ds, [m.eng], (192, 320), m.graph.strides)
        w.lb.clear(), w.nms.clear(), w.rescale.clear()
        batches = [[frame(1080, 1920)], [frame(720, 1280), frame(1080, 1920, device="cuda")], [frame(720, 1280, "rgb_chw")]]
        rows = [[ref_row(c1080)], [ref_row(c720), ref_row(c1080)], [ref_row(c720)]]
        for i, b in enumerate(batches):
            ds.submit(b, layout="rgb_chw" if i == 2 else "bgr_hwc")
            ds.collect()
        refused(rec, ds.submit, ds.slots[ds.steps & 1], [frame(1920, 1080)], r"canvas is 192 x 320")
        ds.drain()
        # step 0 also post-processes the empty second slot: all border
        assert [x[0] for x in w.lb] == [(192, 320)] * 3 and [x[0] for x in w.rescale] == [(192, 320)] * 4
        assert w.rescale[0][1] == [[0, 192, 320, 0, 0, 0, 0, 0]] * 2
        assert len(w.nms) == 4 and all(n == [(24, 40), (12, 20), (6, 10), (3, 5)] for n in w.nms)
        for i, want in enumerate(rows):
            assert [r[1:] for r in w.lb[i][1][:len(want)]] == want
            assert [r[1:] for r in w.rescale[i + 1][1][:len(want)]] == want       # batch i rescaled in step i + 1 / the drain
    served("yolov6lite_s", monkeypatch, run)


def test_farm_auto_two_lanes(monkeypatch):
    """DetectFarm with two lanes at img_size 640 for portrait 1080p: both lanes' engines pinned and captured at 640 x 384;
    a landscape frame is refused by the lane it would go to."""
    cp = golden(1920, 1080, 640)

    def run(rec, m, w, engines):
        farm = pipeline.DetectFarm(m, 2, 640, 640, lanes=2, raw_input=True, auto=True, source_shape=(1920, 1080),
                                   max_src_bytes=2 * 1920 * 1080 * 3)
        assert farm.canvas == (640, 384)
        assert_built_at(farm, engines, (640, 384), m.graph.strides)
        w.lb.clear(), w.nms.clear(), w.rescale.clear()
        for j in range(4):
            farm.submit([frame(1920, 1080, device="cuda" if j % 2 else None)])
        lane = farm.lane_of_next()
        refused(rec, farm.submit, lane.slots[lane.steps & 1], [frame(1080, 1920)], r"canvas is 640 x 384")
        for ln, lane in enumerate(farm.lanes):
            with torch.cuda.stream(farm.streams[ln]):
                lane.drain()
        # per lane: step 0 post-processes the empty second slot, step 1 and the drain the lane's two batches
        assert [x[0] for x in w.lb] == [(640, 384)] * 4 and [x[0] for x in w.rescale] == [(640, 384)] * 6
        assert all(x[1][0][1:] == ref_row(cp) for x in w.lb)
        assert sorted(x[1][0][1:] == ref_row(cp) for x in w.rescale) == [False] * 2 + [True] * 4
        assert len(engines) == 2
    served("yolov6n", monkeypatch, run)


def test_auto_needs_raw_frames_and_a_source_shape(monkeypatch):
    def run(rec, m, w, engines):
        for kw in (dict(auto=True, source_shape=(1080, 1920)), dict(raw_input=True, auto=True)):
            with pytest.raises(RuntimeError, match="auto=True letterboxes decoded frames"):
                pipeline.DetectPipeline(m, 2, 640, 640, **kw)
        p = pipeline.DetectPipeline(m, 2, 600, 600, raw_input=True, auto=True, source_shape=(1080, 1920))
        assert p.canvas == (352, 608) == (golden(1080, 1920, 600)["H"], golden(1080, 1920, 600)["W"])
    served("yolov6n", monkeypatch, run)
