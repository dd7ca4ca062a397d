"""GPU parity of the decoded-frame front and back end (yv6_letterbox, yv6_rescale_boxes, the raw-frame pipelines) against the
reference's goldens (tests/golden/letterbox_cases.json: digests of the cv2 letterbox canvases; tests/golden/letterbox.npz:
Inferer.rescale(...).round() rows)."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import golden_json, golden_npz
from oracle import letterbox as ol

pytestmark = pytest.mark.gpu

G = golden_json("letterbox_cases.json")
NPZ = golden_npz("letterbox.npz")


def by_canvas(cases):
    groups = {}
    for i, c in enumerate(cases):
        groups.setdefault((c[-2], c[-1]) if len(c) == 4 else (c[2], c[3]), []).append(i)
    return groups


def test_letterbox_canvases_byte_identical_to_cv2():
    """Every golden case, one launch per canvas size with all of that size's sources (mixed sizes) in the batch."""
    from yolov6_b200.preprocess import letterbox_batch
    dev = torch.device("cuda:0")
    groups = by_canvas(ol.CASES)
    assert max(len(v) for v in groups.values()) >= 7
    for (H, W), idx in groups.items():
        for su in (True, False):
            sel = [i for i in idx if ol.CASES[i][4] == su]
            if not sel:
                continue
            ims = [ol.synthetic_source(ol.CASES[i][0], ol.CASES[i][1], ol.CASES[i][5], i) for i in sel]
            canvas, meta = letterbox_batch(ims, H, W, scaleup=su, device=dev)
            got = canvas.cpu().numpy()
            for k, i in enumerate(sel):
                c = G["cases"][i]
                if hashlib.sha256(np.ascontiguousarray(got[k]).tobytes()).hexdigest() != c["canvas_sha256"]:
                    # the oracle's canvas carries the golden digest (tests/test_oracle_letterbox.py): say where they differ
                    ref = ol.letterbox(ims[k], H, W, su)
                    diff = np.abs(got[k].astype(np.int64) - ref.astype(np.int64))
                    pytest.fail(f"case {i} {ol.CASES[i]}: {int((diff > 0).sum())} bytes differ, max {int(diff.max())}")
                assert meta.shapes[k][1][1] == (c["left"], c["top"])


def test_rescale_boxes_bit_identical_to_reference():
    from yolov6_b200.preprocess import GEO, LetterboxMeta, rescale_boxes
    dev = torch.device("cuda:0")
    for (H, W), idx in by_canvas(ol.RESCALE_CASES).items():
        dets = [NPZ[f"r{j}_det"] for j in idx]
        max_det = max(d.shape[0] for d in dets) + 3
        out = torch.full((len(idx), max_det, 6), 7.0)
        count = torch.zeros(len(idx), dtype=torch.int32)
        geo = torch.zeros(len(idx), GEO, dtype=torch.int32)
        for k, (j, d) in enumerate(zip(idx, dets)):
            n = d.shape[0] - k            # rows beyond count must come back zeroed
            out[k, :n] = torch.from_numpy(d[:n])
            count[k] = n
            geo[k, 1], geo[k, 2] = ol.RESCALE_CASES[j][0], ol.RESCALE_CASES[j][1]
        res = rescale_boxes(out.to(dev), count.to(dev), LetterboxMeta(geo, len(idx), H, W, None)).cpu().numpy()
        for k, j in enumerate(idx):
            n = int(count[k])
            assert np.array_equal(res[k, :n], NPZ[f"r{j}_out"][:n]), ol.RESCALE_CASES[j]
            assert not res[k, n:].any()


SIZES_A = [(138, 302), (480, 640), (33, 1000), (160, 160)]
SIZES_B = [(720, 1280), (1, 1), (301, 97)]


def frames(sizes, seed):
    return [ol.synthetic_source(h, w, "grad" if i % 2 else "noise", seed + i) for i, (h, w) in enumerate(sizes)]


def expected(m, frs, B, S, kw):
    """Reference composition: cv2-exact letterbox (oracle) -> existing DetectPipeline -> Inferer.rescale(...).round()."""
    from yolov6_b200.pipeline import DetectPipeline
    x = np.full((B, 3, S, S), 114, np.uint8)
    for i, f in enumerate(frs):
        x[i] = ol.letterbox(f, S, S)
    rows = DetectPipeline(m, B, S, S, host_input=True, **kw)(torch.from_numpy(x))
    return [ol.rescale(rows[i].numpy(), S, S, f.shape[0], f.shape[1]) for i, f in enumerate(frs)]


def test_raw_pipeline_matches_letterbox_pipeline_rescale():
    """Mixed-size batches through one captured raw-frame graph, two different size mixes in a row (the second one also
    a partial batch), equal the rows of the reference composition; the staging capacity and the frame format are checked
    before anything is enqueued."""
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectPipeline
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = randomize_(build_model("yolov6n", 80, dev), seed=3).eval()
    B, S = 4, 192
    kw = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)
    raw = DetectPipeline(m, B, S, S, raw_input=True, max_src_bytes=4 << 20, **kw)
    graph = raw.graph
    total = 0
    for sizes, seed in ((SIZES_A, 0), (SIZES_B, 10), (SIZES_A[::-1], 20)):
        frs = frames(sizes, seed)
        got = raw(frs)
        ref = expected(m, frs, B, S, kw)
        assert raw.graph is graph and len(got) == len(frs)
        for g, r in zip(got, ref):
            assert np.array_equal(g.numpy(), r)
            total += g.shape[0]
    assert total > 0
    with pytest.raises(RuntimeError):
        raw([np.zeros((1200, 1200, 3), np.uint8)] * 2)              # 8.6 MB > 4 MiB of staging
    with pytest.raises(RuntimeError):
        raw([np.zeros((20, 20, 3), np.float32)])
    with pytest.raises(RuntimeError):
        raw([np.zeros((20, 20, 4), np.uint8)])


def test_raw_stream_matches_letterbox_pipeline_rescale():
    """DetectStream with raw frames: batch i is letterboxed in step i and rescaled in step i + 1 (or drain) with its own
    geometry while the next batches' bytes are already being copied."""
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectStream
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = randomize_(build_model("yolov6n", 80, dev), seed=3).eval()
    B, S = 4, 192
    kw = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)
    ds = DetectStream(m, B, S, S, raw_input=True, max_src_bytes=4 << 20, **kw)
    batches = [frames(SIZES_A, 0), frames(SIZES_B, 10), frames(SIZES_A[::-1], 20), frames(SIZES_B[:2], 30)]
    outs = []
    for frs in batches:
        ds.submit(frs)
        r = ds.collect()
        if r is not None:
            outs.append(r)
    ds.drain()
    while len(outs) < len(batches):
        outs.append(ds.collect())
    for frs, got in zip(batches, outs):
        ref = expected(m, frs, B, S, kw)
        assert len(got) == len(frs)
        for g, r in zip(got, ref):
            assert np.array_equal(g.numpy(), r)
