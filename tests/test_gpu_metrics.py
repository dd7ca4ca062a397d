"""GPU parity of the PR metric (yv6_pr_match / yv6_pr_metric through yolov6_b200.metrics.PRMetric) against the goldens of
the unmodified reference Evaler and against the CPU oracle on a COCO-val-sized seeded set with conf and IoU ties."""
import os

import numpy as np
import pytest
import torch

from oracle import metrics as om
from test_oracle_metrics import CASES, GOLDEN, check_against_golden, golden_batches

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def run(metric, batches, max_det=300, device_targets=False):
    for preds, targets, shapes, hw in batches:
        out, count = om.pack(preds, max_det)
        t = torch.from_numpy(targets)
        metric.update(torch.from_numpy(out).to(DEV), torch.from_numpy(count).to(DEV), t.to(DEV) if device_targets else t, shapes, hw)
    return metric.result()


def as_dict(res):
    return dict(p=res.p, r=res.r, ap=res.ap, f1=res.f1, ap_class=res.ap_class, nt=res.nt, matrix=res.matrix, ok=res.ok,
                best=res.best, map50=res.map50, map=res.map, mp=res.mp, mr=res.mr)


def check_against_oracle(res, ref, stats=None):
    assert np.array_equal(res.nt, ref["nt"]) and np.array_equal(res.matrix, ref["matrix"]) and res.ok == ref["ok"]
    assert np.array_equal(res.ap_class, ref["ap_class"]) and res.best == ref["best"] and res.seen == ref["seen"]
    for k in ("p", "r", "ap", "f1"):
        err = float(np.abs(getattr(res, k) - ref[k]).max()) if ref[k].size else 0.0
        assert err <= 1e-12, (k, err)
    for k in ("map50", "map", "mp", "mr"):
        assert abs(getattr(res, k) - ref[k]) <= 1e-12, (k, getattr(res, k), ref[k])
    if stats is not None:
        correct, conf, pcls, tcls = stats
        assert np.array_equal(correct, ref["correct"]) and np.array_equal(conf, ref["conf"]) and np.array_equal(pcls, ref["pcls"])
        assert np.array_equal(tcls, ref["tcls"])


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "metrics.npz"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_cases(golden, name):
    from yolov6_b200.metrics import PRMetric
    batches = golden_batches(golden, name)
    n = sum(len(b[0]) for b in batches)
    metric = PRMetric(CASES[name]["nc"], max_images=n + 3, device=DEV, confusion=True)
    res = run(metric, batches, device_targets=(name == "rect20"))
    check_against_golden(as_dict(res), golden, name)
    correct, conf, pcls, tcls = metric.stats()
    assert np.array_equal(correct, golden[f"{name}/correct"]) and np.array_equal(conf, golden[f"{name}/conf"])
    assert np.array_equal(pcls, golden[f"{name}/pcls"]) and np.array_equal(tcls, golden[f"{name}/tcls"])


def test_coco_val_sized_against_oracle():
    from yolov6_b200.metrics import PRMetric
    batches, nc = om.coco_val_sized()
    metric = PRMetric(nc, max_images=5000, device=DEV, confusion=True)
    res = run(metric, batches)
    ref = om.evaluate(batches, nc)
    assert res.seen == 5000 and max(len(p) for b in batches for p in b[0]) == 300
    check_against_oracle(res, ref, metric.stats())
    # reset(): the next epoch on the same buffers gives the same result
    metric.reset()
    res2 = run(metric, batches)
    for k in ("p", "r", "ap", "f1", "matrix", "nt"):
        assert np.array_equal(getattr(res2, k), getattr(res, k)), k
    assert (res2.map50, res2.map, res2.mp, res2.mr, res2.best) == (res.map50, res.map, res.mp, res.mr, res.best)


def test_pipeline_rows_yolov6n():
    """update() straight on DetectPipeline's device tensors, checked against the oracle on the host copy of the same rows."""
    from yolov6_b200.metrics import PRMetric
    from yolov6_b200.model import build_model
    from yolov6_b200.pipeline import DetectPipeline
    from yolov6_b200.synth import randomize_
    m = randomize_(build_model("yolov6n", 80, DEV), seed=3).eval()
    B, S = 4, 192
    pipe = DetectPipeline(m, B, S, S, host_input=False, multi_label=True, conf_thres=0.03, iou_thres=0.65)
    metric = PRMetric(80, max_images=3 * B, device=DEV, confusion=True)
    rng = np.random.default_rng(7)
    batches = []
    for i in range(3):
        x = torch.from_numpy(rng.random((B, 3, S, S), dtype=np.float32)).to(DEV)
        rows = pipe(x)
        preds = [r.cpu().numpy() for r in rows]
        shapes = [om.letterbox_shape(int(rng.integers(100, 900)), int(rng.integers(100, 900)), S, S) for _ in range(B)]
        # labels on the model's own boxes (some exact, some shifted) so that matches happen at every threshold
        targets = []
        for b, p in enumerate(preds):
            for r in p[:: max(1, len(p) // 6)]:
                x1, y1, x2, y2 = r[:4] / S
                j = rng.uniform(-0.02, 0.02, 2) * (rng.random() < 0.5)
                targets.append([b, r[5] if rng.random() < 0.8 else rng.integers(0, 80), (x1 + x2) / 2 + j[0], (y1 + y2) / 2 + j[1],
                                x2 - x1, y2 - y1])
        targets = np.array(targets, np.float32).reshape(-1, 6)
        metric.update(pipe.out_dev, pipe.count_dev, torch.from_numpy(targets), shapes, (S, S))
        batches.append((preds, targets, shapes, (S, S)))
    assert sum(len(p) for b in batches for p in b[0]) > 0
    res = metric.result()
    ref = om.evaluate(batches, 80)
    assert ref["ok"] and ref["correct"].any()
    check_against_oracle(res, ref, metric.stats())


def test_update_does_not_synchronize(golden):
    from yolov6_b200.metrics import PRMetric
    batches = golden_batches(golden, "coco80")
    metric = PRMetric(80, max_images=64, device=DEV, confusion=True)
    staged = []
    for preds, targets, shapes, hw in batches:
        out, count = om.pack(preds, 300)
        staged.append((torch.from_numpy(out).to(DEV), torch.from_numpy(count).to(DEV), torch.from_numpy(targets), shapes, hw))
    metric.update(*staged[0])                               # first call: library load, handle, kernel attributes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for s in staged[1:]:
            metric.update(*s)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    check_against_golden(as_dict(metric.result()), golden, "coco80")


def test_errors():
    from yolov6_b200.metrics import PRMetric
    metric = PRMetric(5, max_images=4, device=DEV)
    out = torch.zeros(2, 10, 6, device=DEV)
    count = torch.zeros(2, dtype=torch.int32, device=DEV)
    t = torch.zeros(0, 6)
    shapes = [om.letterbox_shape(100, 100, 64, 64)] * 2
    bad = [
        (out.double(), count, t, shapes),                                   # dtype
        (out[:, :, :5].contiguous(), count, t, shapes),                     # shape
        (out, count.long(), t, shapes),
        (out, count[:1], t, shapes),
        (out, count, t.double(), shapes),
        (out, count, torch.zeros(0, 5), shapes),
        (out, count, t, shapes[:1]),
        (torch.zeros(2, 301, 6, device=DEV), count, t, shapes),             # more rows than max_det
        (out.cpu(), count, t, shapes),                                      # no CPU path
    ]
    for args in bad:
        with pytest.raises(RuntimeError):
            metric.update(*args, (64, 64))
    assert metric.seen == 0
    metric.update(out, count, t, shapes, (64, 64))
    metric.update(out, count, t, shapes, (64, 64))
    with pytest.raises(RuntimeError):                                       # more images than max_images
        metric.update(out, count, t, shapes, (64, 64))
    assert metric.seen == 4
    # a label class outside [0, nc) is reported by result()
    metric.reset()
    metric.update(out, count, torch.tensor([[0, 7, 0.5, 0.5, 0.2, 0.2]]), shapes, (64, 64))
    with pytest.raises(RuntimeError, match="label class"):
        metric.result()
    metric.reset()
    o = out.clone()
    o[0, 0] = torch.tensor([1, 1, 20, 20, 0.5, 5.0])
    metric.update(o, torch.tensor([1, 0], dtype=torch.int32, device=DEV), t, shapes, (64, 64))
    with pytest.raises(RuntimeError, match="detection class"):
        metric.result()
    with pytest.raises(RuntimeError):
        PRMetric(5, max_images=4, device="cpu")
