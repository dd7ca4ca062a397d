"""tests/golden/make_golden_metrics.py -- goldens of the Evaler's precision / recall metric from the UNMODIFIED reference
(build container only):

    python tests/golden/make_golden_metrics.py

Drives Evaler.predict_model (yolov6/core/evaler.py:100-228) with do_pr_metric=True, plot_confusion_matrix=True,
plot_curve=False over a fake model and dataloader; `non_max_suppression` is patched to return fabricated NMS rows
(oracle.metrics.dataset), matplotlib / seaborn / pycocotools are stub modules.  metrics.process_batch, ap_per_class and
ConfusionMatrix are wrapped to record the stats, the returned arrays and the matrix; pr_metric_result is read off the
Evaler.  Writes tests/golden/metrics.npz and metrics_cases.json.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(HERE, "refshim"), "/root/reference", ROOT]
for name in ("matplotlib", "matplotlib.pyplot", "seaborn"):        # metrics.py imports pyplot at module level
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
for name in ("pycocotools", "pycocotools.coco", "pycocotools.cocoeval"):
    mod = types.ModuleType(name)
    mod.COCO = mod.COCOeval = object
    sys.modules.setdefault(name, mod)

import torch  # noqa: E402

torch.cuda.is_available = lambda: False
import yolov6.core.evaler as evaler_mod  # noqa: E402
import yolov6.utils.metrics as metrics_mod  # noqa: E402
from yolov6.core.evaler import Evaler  # noqa: E402

from oracle import metrics as om  # noqa: E402

# name -> (dataset kwargs, nc)
CASES = {
    "coco80": (dict(seed=11, n_batches=3, B=8, H=640, W=640, nc=80, label_classes=np.arange(0, 70), pred_only_classes=range(70, 80)), 80),
    "rect20": (dict(seed=12, n_batches=3, B=8, H=384, W=640, nc=20, last_batch=5), 20),
    "nc1": (dict(seed=13, n_batches=2, B=6, H=320, W=320, nc=1, p_wrong_cls=0.0, p_dup=0.0), 1),
    "nothing": (dict(seed=14, n_batches=1, B=4, H=320, W=320, nc=5, iou_span=(0.0, 0.2), dets_per_label=0, fp_rate=3.0), 5),
}


def exact_case():
    """IoUs exactly at thresholds: [0,0,10,10] vs [0,0,10,5] = 0.5, vs [0,0,10,7.5] = 0.75, and 55/100 = iouv[1] in fp32.
    Canvas 100x100, no letterbox scaling (gain 1, pad 0)."""
    shapes = [((100, 100), ((1.0, 1.0), (0.0, 0.0)))] * 3
    # labels xywh normalised: [0,0,10,10] -> (0.05, 0.05, 0.1, 0.1)
    targets = np.array([[0, 0, 0.05, 0.05, 0.1, 0.1], [1, 1, 0.05, 0.05, 0.1, 0.1], [2, 0, 0.05, 0.05, 0.1, 0.1]], np.float32)
    preds = [np.array([[0, 0, 10, 5, 0.9, 0]], np.float32),
             np.array([[0, 0, 10, 7.5, 0.8, 1]], np.float32),
             np.array([[0, 0, 10, 5.5, 0.7, 0], [0, 0, 10, 5.5, 0.2, 0]], np.float32)]
    return [(preds, targets, shapes, (100, 100))]


def run_reference(batches, nc):
    rec = {"process_batch": [], "ap_per_class": None, "cm": None}
    pb, apc, CM = metrics_mod.process_batch, metrics_mod.ap_per_class, metrics_mod.ConfusionMatrix

    def process_batch(detections, labels, iouv):
        out = pb(detections, labels, iouv)
        rec["process_batch"].append(out.numpy().copy())
        return out

    def ap_per_class(*args, **kw):
        out = apc(*args, **kw)
        rec["ap_per_class"] = [np.asarray(o).copy() for o in out]
        return out

    class ConfusionMatrix(CM):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            rec["cm"] = self

    class NumpyRecorder:                 # the Evaler's `stats = [np.concatenate(x, 0) for x in zip(*stats)]` (evaler.py:197)
        def __getattr__(self, k):
            return getattr(np, k)

        def concatenate(self, x, *a, **kw):
            out = np.concatenate(x, *a, **kw)
            rec.setdefault("concat", []).append(out)
            return out

    metrics_mod.process_batch, metrics_mod.ap_per_class, metrics_mod.ConfusionMatrix = process_batch, ap_per_class, ConfusionMatrix
    evaler_mod.np = NumpyRecorder()
    outs = iter([[torch.from_numpy(p.copy()) for p in preds] for preds, _, _, _ in batches])
    evaler_mod.non_max_suppression = lambda *a, **kw: next(outs)

    class Model:
        def __init__(self):
            self.nc, self.names = nc, [str(i) for i in range(nc)]

        def __call__(self, imgs):
            return torch.zeros(imgs.shape[0], 1, 5 + nc), None

    loader = [(torch.zeros(len(preds), 3, hw[0], hw[1]), torch.from_numpy(targets), [f"{1000 + i}.jpg" for i in range(len(preds))], shapes)
              for preds, targets, shapes, hw in batches]
    ev = Evaler.__new__(Evaler)
    ev.device, ev.half, ev.conf_thres, ev.iou_thres = torch.device("cpu"), False, 0.03, 0.65
    ev.do_pr_metric, ev.plot_confusion_matrix, ev.plot_curve, ev.verbose = True, True, False, False
    ev.save_dir, ev.is_coco, ev.ids = "/tmp", True, list(range(1, 1000))
    ev.predict_model(Model(), loader, "val")
    try:
        rec["stats"] = rec["concat"][-4:]
        return rec, ev.pr_metric_result
    finally:
        metrics_mod.process_batch, metrics_mod.ap_per_class, metrics_mod.ConfusionMatrix = pb, apc, CM
        evaler_mod.np = np


def main():
    arrays, meta = {}, {}
    cases = {k: (om.dataset(no_ties=True, **kw), nc) for k, (kw, nc) in CASES.items()}
    cases["exact"] = (exact_case(), 2)
    for name, (batches, nc) in cases.items():
        om.assert_no_ties(batches, nc)
        rec, (map50, map_) = run_reference(batches, nc)
        for bi, (preds, targets, shapes, hw) in enumerate(batches):
            arrays[f"{name}/b{bi}/rows"] = np.concatenate(preds, 0)
            arrays[f"{name}/b{bi}/count"] = np.array([len(p) for p in preds], np.int32)
            arrays[f"{name}/b{bi}/targets"] = targets
        st = rec["stats"]
        arrays[f"{name}/correct"], arrays[f"{name}/conf"], arrays[f"{name}/pcls"], arrays[f"{name}/tcls"] = st
        if rec["ap_per_class"] is not None:
            for k, v in zip(("p", "r", "ap", "f1", "ap_class"), rec["ap_per_class"]):
                arrays[f"{name}/{k}"] = v
        arrays[f"{name}/matrix"] = rec["cm"].matrix
        ok = rec["ap_per_class"] is not None
        entry = {"nc": nc, "H": batches[0][3][0], "W": batches[0][3][1], "n_batches": len(batches), "ok": ok,
                 "shapes": [[list(map(list, [s[0], s[1][0], s[1][1]])) for s in b[2]] for b in batches],
                 "map50": float(map50), "map": float(map_), "nt": np.bincount(st[3].astype(np.int64), minlength=nc).tolist()}
        if ok:
            p, r, ap, f1, _ = rec["ap_per_class"]
            f1m = f1.mean(0)
            best = len(f1m) - f1m[::-1].argmax() - 1
            entry.update(best=int(best), mp=float(p[:, best].mean()), mr=float(r[:, best].mean()))
        meta[name] = entry
        print(name, "images", sum(len(b[0]) for b in batches), "rows", len(st[1]), "ok", ok, "map50 %.4f map %.4f" % (map50, map_))
    np.savez_compressed(os.path.join(HERE, "metrics.npz"), **arrays)
    with open(os.path.join(HERE, "metrics_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
