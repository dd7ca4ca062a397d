"""GPU parity of the COCO box evaluation (yv6_coco_update / yv6_coco_load / yv6_coco_accumulate through
yolov6_b200.cocoeval.COCOMetric): bit-identical precision / recall / scores / stats against the CPU oracle on the
hand-worked cases and on fabricated sets, the device path against the json-row path, batch order and size, reset()."""
import json

import numpy as np
import pytest
import torch

from oracle import cocoeval as oc
from test_oracle_cocoeval import CASES, check_expectations

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def identical(res, ref):
    stats, precision, recall, scores = ref
    assert res.precision.shape == precision.shape
    for name, got, want in (("precision", res.precision, precision), ("recall", res.recall, recall), ("scores", res.scores, scores),
                            ("stats", res.stats, stats)):
        assert np.array_equal(got.view(np.int64), np.asarray(want, np.float64).view(np.int64)), (name, int((got != want).sum()))


def stream(metric, batches, order=None, B=None):
    """update() over the fabricated batches, optionally re-cut into batches of B images in the given image order."""
    if B is None and order is None:
        for out, count, shapes, ids in batches:
            metric.update(torch.from_numpy(out).to(DEV), torch.from_numpy(count).to(DEV), shapes, ids)
        return
    out = np.concatenate([b[0] for b in batches])
    count = np.concatenate([b[1] for b in batches])
    shapes = [s for b in batches for s in b[2]]
    ids = [i for b in batches for i in b[3]]
    order = np.arange(len(ids)) if order is None else order
    for i0 in range(0, len(order), B):
        sel = order[i0:i0 + B]
        metric.update(torch.from_numpy(out[sel]).to(DEV), torch.from_numpy(count[sel]).to(DEV), [shapes[i] for i in sel],
                      [ids[i] for i in sel])


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_case(name):
    from yolov6_b200.cocoeval import COCOMetric
    case = CASES[name]
    m = COCOMetric(case["gt"], [c["id"] for c in case["gt"]["categories"]], img_ids=case.get("img_ids"), device=DEV)
    m.load_results(case["results"])
    res = m.result()
    ref = oc.evaluate(case["gt"], case["results"], case.get("img_ids"))
    identical(res, ref)
    check_expectations(case, res.stats, res.precision, res.recall, res.scores)


@pytest.fixture(scope="module")
def mid():
    gt, batches, ids = oc.fabricate(11, 300, n_cats=80, crowd=0.02, B=32)
    return gt, batches, ids, oc.evaluate(gt, oc.rows_of(batches, ids))


def test_mid_size_set_against_oracle(mid):
    from yolov6_b200.cocoeval import COCOMetric
    gt, batches, ids, ref = mid
    assert any(a["iscrowd"] for a in gt["annotations"]) and ref[0][0] > 0
    m = COCOMetric(gt, ids, device=DEV)
    stream(m, batches)
    res = m.result()
    identical(res, ref)
    # reset(): a second epoch on the same buffers, the images in another order and other batch sizes
    m.reset()
    stream(m, batches, order=np.random.default_rng(0).permutation(300), B=7)
    identical(m.result(), ref)
    m.reset()
    stream(m, batches, order=np.arange(300)[::-1].copy(), B=300)
    identical(m.result(), ref)


def test_row_path_equals_device_path(mid, tmp_path):
    from yolov6_b200.cocoeval import COCOMetric
    gt, batches, ids, ref = mid
    rows = oc.rows_of(batches, ids)
    path = tmp_path / "predictions.json"
    with open(path, "w") as f:
        json.dump(rows, f)
    m = COCOMetric(gt, ids, device=DEV)
    m.load_results(str(path))
    identical(m.result(), ref)


def test_coco_scale_set_against_oracle():
    from yolov6_b200.cocoeval import COCOMetric
    gt, batches, ids = oc.fabricate(5, 1000, n_cats=80, crowd=0.01, B=32)
    img_ids = sorted(im["id"] for im in gt["images"])[:900]     # params.imgIds: a subset, the rest dropped silently
    ref = oc.evaluate(gt, oc.rows_of(batches, ids), img_ids)
    m = COCOMetric(gt, ids, img_ids=img_ids, device=DEV)
    stream(m, batches)
    identical(m.result(), ref)


def test_pipeline_rows_device_vs_json_path():
    """update() on DetectPipeline(multi_label=True) tensors of a seeded model against load_results of the Evaler's json
    rows (evalpost.convert_to_coco_format) of the same tensors; both against the oracle."""
    from yolov6_b200.cocoeval import COCOMetric
    from yolov6_b200.evalpost import convert_to_coco_format
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectPipeline
    from yolov6_b200.synth import randomize_
    from oracle.metrics import letterbox_shape
    net = randomize_(build_model("yolov6n", 80, DEV), seed=3).eval()
    B, S = 4, 192
    pipe = DetectPipeline(net, B, S, S, host_input=False, multi_label=True, conf_thres=0.03, iou_thres=0.65)
    rng = np.random.default_rng(7)
    ids = list(range(1, 81))                                 # coco80_to_coco91-like table, category 0 absent
    gt = {"images": [], "annotations": [], "categories": [{"id": c} for c in ids[:60]]}
    staged, rows = [], []
    for i in range(3):
        x = torch.from_numpy(rng.random((B, 3, S, S), dtype=np.float32)).to(DEV)
        dets = [d.cpu().numpy() for d in pipe(x)]
        shapes = [letterbox_shape(int(rng.integers(100, 900)), int(rng.integers(100, 900)), S, S) for _ in range(B)]
        img_ids = [100 * i + b + 1 for b in range(B)]
        for b, d in enumerate(dets):
            gt["images"].append({"id": img_ids[b]})
            (h0, w0), (gain, pad) = shapes[b]
            for r in d[:: max(1, len(d) // 8)]:                # gts on the model's own boxes, some shifted
                x1, y1 = (r[0] - pad[0]) / gain[1], (r[1] - pad[1]) / gain[0]
                w, h = (r[2] - r[0]) / gain[1], (r[3] - r[1]) / gain[0]
                j = rng.uniform(-3, 3, 2) * (rng.random() < 0.5)
                gt["annotations"].append({"id": len(gt["annotations"]), "image_id": img_ids[b], "category_id": ids[int(r[5])],
                                          "bbox": [float(x1 + j[0]), float(y1 + j[1]), float(w), float(h)], "area": float(w * h),
                                          "iscrowd": int(rng.random() < 0.05)})
        staged.append((pipe.out_dev.clone(), pipe.count_dev.clone(), shapes, img_ids))
        rows += convert_to_coco_format(pipe.out_dev, pipe.count_dev, [f"{k}.jpg" for k in img_ids], shapes, ids)
    assert len(rows) > 0 and len(gt["annotations"]) > 0
    dev_m = COCOMetric(gt, ids, max_det=pipe.out_dev.shape[1], device=DEV)
    for s in staged:
        dev_m.update(*s)
    row_m = COCOMetric(gt, ids, max_det=pipe.out_dev.shape[1], device=DEV)
    row_m.load_results(rows)
    a, b = dev_m.result(), row_m.result()
    ref = oc.evaluate(gt, rows)
    identical(a, ref)
    identical(b, ref)


def test_update_does_not_synchronize(mid):
    from yolov6_b200.cocoeval import COCOMetric
    gt, batches, ids, ref = mid
    m = COCOMetric(gt, ids, device=DEV)
    staged = [(torch.from_numpy(o).to(DEV), torch.from_numpy(c).to(DEV), s, i) for o, c, s, i in batches]
    m.update(*staged[0])                                    # first call: library load, handle, kernel attributes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for s in staged[1:]:
            m.update(*s)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    identical(m.result(), ref)


def test_errors():
    from yolov6_b200.cocoeval import COCOMetric
    case = CASES["tied_scores"]
    gt = case["gt"]
    m = COCOMetric(gt, [1, 2], max_det=10, device=DEV)
    out = torch.zeros(2, 10, 6, device=DEV)
    count = torch.zeros(2, dtype=torch.int32, device=DEV)
    shapes = [((100, 100), ((1.0, 1.0), (0.0, 0.0)))] * 2
    bad = [
        (out.double(), count, shapes, [1, 2]),                 # dtype
        (out[:, :, :5].contiguous(), count, shapes, [1, 2]),   # shape
        (out, count.long(), shapes, [1, 2]),
        (out, count[:1], shapes, [1, 2]),
        (out, count, shapes[:1], [1, 2]),
        (out, count, shapes, [1]),
        (torch.zeros(2, 11, 6, device=DEV), count, shapes, [1, 2]),   # more rows than max_det
        (out.cpu(), count, shapes, [1, 2]),                    # no CPU path
        (out, count, shapes, [1, 3]),                          # image id absent from the gt json
        (out, count, shapes, [1, 1]),                          # an image given twice
    ]
    for args in bad:
        with pytest.raises(RuntimeError):
            m.update(*args)
    m.update(out[:1].contiguous(), count[:1].contiguous(), shapes[:1], [1])
    with pytest.raises(RuntimeError):                          # image 1 again, in a later batch
        m.update(out[:1].contiguous(), count[:1].contiguous(), shapes[:1], [1])
    with pytest.raises(RuntimeError):                          # ... or through the rows
        m.load_results([{"image_id": 1, "category_id": 1, "bbox": [0, 0, 1, 1], "score": 0.5}])
    with pytest.raises(RuntimeError):                          # loadRes: an image the gt json does not have
        m.load_results([{"image_id": 7, "category_id": 1, "bbox": [0, 0, 1, 1], "score": 0.5}])
    with pytest.raises(RuntimeError):                          # capacity: 11 rows for one image
        m.load_results([{"image_id": 2, "category_id": 1, "bbox": [0, 0, 1, 1], "score": 0.5}] * 11)
    # a detection class outside the class table is reported by result()
    m.reset()
    o = out.clone()
    o[0, 0] = torch.tensor([1, 1, 20, 20, 0.5, 5.0])
    m.update(o, torch.tensor([1, 0], dtype=torch.int32, device=DEV), shapes, [1, 2])
    with pytest.raises(RuntimeError, match="detection class"):
        m.result()
    for kw in (dict(device="cpu"), dict(iou_type="segm"), dict(use_cats=0), dict(max_det=0)):
        with pytest.raises(RuntimeError):
            COCOMetric(gt, [1, 2], **{"device": DEV, **kw})
