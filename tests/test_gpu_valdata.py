"""GPU checks of yv6_letterbox_val through ValFeed: every canvas byte-identical (SHA-256) to the reference's
TrainValDataset(augment=False) image (tests/golden/valdata_cases.json) from host frames, device BGR HWC frames, crop
views, RGB CHW device frames and a host / device mix; PRMetric and COCOMetric fed from ValFeed equal to the same metrics
fed from the reference's targets and shapes; and feed() never synchronising the host."""
import hashlib

import numpy as np
import pytest
import torch

from oracle import valdata as ov
from test_valdata import NAMES, case_items, golden, shapes_tuple  # noqa: F401  (golden is a fixture)
from yolov6_b200.valdata import ValFeed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def as_frame(src, how, j):
    """One decoded BGR HWC source in the form `how` ("host", "bgr", "crop", "rgb_chw", or "mix": host / device alternating)."""
    if how == "host" or (how == "mix" and j % 2 == 0):
        return src
    t = torch.from_numpy(src).to(DEV)
    if how == "crop":                        # the source as a view into a larger frame, its rows padded
        h0, w0 = src.shape[:2]
        big = torch.full((h0 + 3, w0 + 5, 3), 7, dtype=torch.uint8, device=DEV)
        big[2:2 + h0, 3:3 + w0] = t
        return big[2:2 + h0, 3:3 + w0]
    if how == "rgb_chw":
        return t.flip(2).permute(2, 0, 1).contiguous()
    return t


def make_feed(c):
    return ValFeed(c["batch"], c["img_size"], c["stride"], c["sources"], pad=c["pad"], rect=c["rect"], shrink_size=c["shrink_size"],
                   device=DEV)


def run(c, feed, how, sources):
    """Every batch through feed: [(canvas, targets, shapes, n, indices)]."""
    out = []
    for idx in feed.batches():
        frames = [as_frame(sources[i], how, j) for j, i in enumerate(idx)]
        canvas, targets, shapes, n = feed.feed(list(idx), frames, [ov.synthetic_labels(int(i)) for i in idx],
                                               layout="rgb_chw" if how == "rgb_chw" else "bgr_hwc")
        out.append((canvas, targets, shapes, n, idx))
    return out


def check_case(c, items, results):
    k = 0
    for canvas, targets, shapes, n, idx in results:
        assert n == len(idx) and canvas.dtype == torch.uint8 and canvas.device == DEV
        host = canvas.cpu().numpy()
        assert (host[n:] == 114).all()
        want_t = []
        for j in range(n):
            i, sh, lab = items[k]
            assert int(idx[j]) == i
            assert hashlib.sha256(host[j].tobytes()).hexdigest() == c["sha256"][k], (k, i, c["sources"][i])
            assert shapes[j] == shapes_tuple(sh)
            lab = lab.copy()
            lab[:, 0] = j
            want_t.append(lab)
            k += 1
        assert targets.dtype == torch.float32 and np.array_equal(targets.numpy(), np.concatenate(want_t, 0))
    assert k == len(items)


@pytest.mark.parametrize("how", ["host", "bgr", "crop", "rgb_chw", "mix"])
@pytest.mark.parametrize("name", NAMES[:5])
def test_canvases_equal_the_reference(golden, name, how):  # noqa: F811
    c, items = case_items(golden, name)
    sources = [ov.synthetic_source(h0, w0, i) for i, (h0, w0) in enumerate(c["sources"])]
    check_case(c, items, run(c, make_feed(c), how, sources))


def detections(targets, n, H, W, seed):
    """Fabricated NMS output [n, 300, 6] / count [n] near the targets (jittered boxes, some class swaps) plus noise boxes."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 300, 6), np.float32)
    count = np.zeros(n, np.int32)
    t = targets.numpy()
    for j in range(n):
        tj = t[t[:, 0] == j]
        rows = []
        for cls, x, y, w, h in tj[:, 1:]:
            cx, cy, bw, bh = x * W, y * H, w * W, h * H
            jit = rng.normal(0, 0.08, 4) * [bw, bh, bw, bh]
            c = cls if rng.uniform() < 0.8 else rng.integers(0, 80)
            rows.append([cx - bw / 2 + jit[0], cy - bh / 2 + jit[1], cx + bw / 2 + jit[2], cy + bh / 2 + jit[3], rng.uniform(0.05, 1), c])
        for _ in range(int(rng.integers(0, 4))):
            x1, y1 = rng.uniform(0, W - 20), rng.uniform(0, H - 20)
            rows.append([x1, y1, x1 + rng.uniform(5, 80), y1 + rng.uniform(5, 80), rng.uniform(0.03, 0.5), rng.integers(0, 80)])
        rows.sort(key=lambda r: -r[4])
        count[j] = len(rows)
        if rows:
            out[j, :len(rows)] = np.array(rows, np.float32)
    return torch.from_numpy(out).to(DEV), torch.from_numpy(count).to(DEV)


def coco_anno(c):
    """A gt json for the fabricated set: each source's labels in source pixels."""
    anns, k = [], 1
    for i, (h0, w0) in enumerate(c["sources"]):
        for cls, x, y, w, h in ov.synthetic_labels(i).astype(np.float64):
            x1, y1 = max(0.0, (x - w / 2) * w0), max(0.0, (y - h / 2) * h0)
            x2, y2 = min(float(w0), (x + w / 2) * w0), min(float(h0), (y + h / 2) * h0)
            anns.append({"id": k, "image_id": i, "category_id": int(cls), "bbox": [x1, y1, x2 - x1, y2 - y1],
                         "area": (x2 - x1) * (y2 - y1), "iscrowd": 0})
            k += 1
    return {"images": [{"id": i} for i in range(len(c["sources"]))], "annotations": anns,
            "categories": [{"id": j} for j in range(80)]}


def test_metrics_through_valfeed_equal_the_reference_feed(golden):  # noqa: F811
    from yolov6_b200.cocoeval import COCOMetric
    from yolov6_b200.metrics import PRMetric
    c, items = case_items(golden, "metric200")
    sources = [ov.synthetic_source(h0, w0, i) for i, (h0, w0) in enumerate(c["sources"])]
    results = run(c, make_feed(c), "mix", sources)
    check_case(c, items, results)
    anno = coco_anno(c)
    pr_a, pr_b = PRMetric(80, 200, device=DEV, confusion=True), PRMetric(80, 200, device=DEV, confusion=True)
    co_a, co_b = COCOMetric(anno, list(range(80)), device=DEV), COCOMetric(anno, list(range(80)), device=DEV)
    k = 0
    for b, (canvas, targets, shapes, n, idx) in enumerate(results):
        H, W = c["batch_shapes"][b]
        # the reference feed: the loader's labels_out with the collate's image index, its shapes, its batch shape
        ref_t = []
        for j in range(n):
            lab = items[k + j][2].copy()
            lab[:, 0] = j
            ref_t.append(lab)
        ref_t = torch.from_numpy(np.concatenate(ref_t, 0))
        ref_shapes = [shapes_tuple(items[k + j][1]) for j in range(n)]
        ids = [int(i) for i in idx]
        out, count = detections(ref_t, n, H, W, seed=b)
        pr_a.update(out, count, targets, shapes, canvas.shape[2:])
        pr_b.update(out, count, ref_t, ref_shapes, (H, W))
        co_a.update(out, count, shapes, ids)
        co_b.update(out, count, ref_shapes, ids)
        k += n
    a, r = pr_a.result(), pr_b.result()
    assert a.seen == r.seen == 200 and a.ok
    for f in ("p", "r", "ap", "f1", "ap_class", "nt", "matrix"):
        assert np.array_equal(getattr(a, f), getattr(r, f)), f
    assert (a.map50, a.map, a.mp, a.mr, a.best) == (r.map50, r.map, r.mp, r.mr, r.best)
    ca, cr = co_a.result(), co_b.result()
    for f in ("stats", "precision", "recall", "scores"):
        assert np.array_equal(getattr(ca, f), getattr(cr, f)), f
    assert ca.stats[0] > 0


def test_feed_does_not_synchronize(golden):  # noqa: F811
    c, items = case_items(golden, "rect640")
    sources = [ov.synthetic_source(h0, w0, i) for i, (h0, w0) in enumerate(c["sources"])]
    feed = make_feed(c)
    batches = feed.batches()
    dev_frames = {int(i): torch.from_numpy(sources[i]).to(DEV) for i in range(len(sources))}
    first = batches[0]
    feed.feed(list(first), [sources[i] for i in first], [ov.synthetic_labels(int(i)) for i in first])   # library load, handle
    torch.cuda.synchronize()
    results = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for idx in batches:
            frames = [sources[i] if j % 2 else dev_frames[int(i)] for j, i in enumerate(idx)]
            results.append(feed.feed(list(idx), frames, [ov.synthetic_labels(int(i)) for i in idx]) + (idx,))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    check_case(c, items, results)
