"""oracle/metrics.py -- CPU restatement of the Evaler's precision / recall metric (TEST INFRASTRUCTURE ONLY).

States the rules of yolov6_b200/csrc/yv6_metrics.cu, which are those of the reference's Evaler.predict_model with
do_pr_metric=True (yolov6/core/evaler.py:109-226), process_batch / ConfusionMatrix.process_batch / ap_per_class /
compute_ap (yolov6/utils/metrics.py), in rule form: box math in torch fp32 (oracle.evalpost.scale_coords), everything
after it in numpy float64 with a stable sort.  Pinned against the unmodified reference by
tests/golden/make_golden_metrics.py.
"""
import numpy as np
import torch

from oracle.evalpost import scale_coords

IOUV = torch.linspace(0.5, 0.95, 10).numpy()        # evaler.py:112, fp32
PX = np.linspace(0, 1, 1000)                        # metrics.py:36
X101 = np.linspace(0, 1, 101)                       # metrics.py:96


def box_iou(a, b):
    """general.box_iou (general.py:64-86) in fp32: a [n,4], b [m,4] -> [n,m]; 0/0 gives NaN, which never compares true."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    area1 = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area2 = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    iw = np.maximum(np.minimum(a[:, None, 2], b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0]), np.float32(0))
    ih = np.maximum(np.minimum(a[:, None, 3], b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1]), np.float32(0))
    inter = iw * ih
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / ((area1[:, None] + area2[None, :]) - inter)


def label_boxes(labels, hw, shape):
    """labels [n,5] (cls, x, y, w, h) normalised to the letterboxed canvas -> xyxy in source pixels (evaler.py:175-182)."""
    x = torch.as_tensor(labels[:, 1:5], dtype=torch.float32)
    t = x.clone()
    t[:, 0] = x[:, 0] - x[:, 2] / 2
    t[:, 1] = x[:, 1] - x[:, 3] / 2
    t[:, 2] = x[:, 0] + x[:, 2] / 2
    t[:, 3] = x[:, 1] + x[:, 3] / 2
    t[:, [0, 2]] *= hw[1]
    t[:, [1, 3]] *= hw[0]
    return scale_coords(t, shape[0], shape[1]).numpy()


def pred_boxes(pred, shape):
    return scale_coords(torch.as_tensor(pred[:, :4], dtype=torch.float32).clone(), shape[0], shape[1]).numpy()


def best_label(iou, ok):
    """Per column: the row with the highest IoU among rows where `ok` (ties: the lowest row); -1 where none."""
    masked = np.where(ok, iou, -np.inf)
    best = np.argmax(masked, axis=0) if masked.shape[0] else np.zeros(masked.shape[1], np.int64)
    has = ok.any(axis=0)
    return np.where(has, best, -1), np.where(has, masked[best, np.arange(masked.shape[1])] if masked.shape[0] else 0, 0)


def correct_flags(iou, lcls, dcls, iouv=IOUV):
    """process_batch's rule: L(d) = same-class label with the highest IoU; d is correct at t iff IoU(L(d), d) >= iouv[t]
    and no lower-indexed detection has the same L at t."""
    nd = iou.shape[1]
    same = lcls[:, None] == dcls[None, :]
    L, m = best_label(iou, same & (iou >= iouv[0]))
    cand = (L[:, None] >= 0) & (m[:, None] >= iouv[None, :])
    correct = np.zeros((nd, len(iouv)), bool)
    for t in range(len(iouv)):
        rows = np.nonzero(cand[:, t])[0]
        seen = set()
        for d in rows:
            if L[d] not in seen:
                seen.add(L[d])
                correct[d, t] = True
    return correct


def confusion_update(matrix, iou, lcls, dconf, dcls, nc):
    """ConfusionMatrix.process_batch (metrics.py:177-215): detections with conf > 0.25, class-agnostic IoU > 0.45; each
    detection keeps its best label, each label the detection with the highest IoU among those (ties: lowest index)."""
    keep = dconf > np.float32(0.25)
    k_iou, k_cls = iou[:, keep], dcls[keep]
    DL, Dm = best_label(k_iou, k_iou > np.float32(0.45))
    win = -np.ones(len(lcls), np.int64)
    for d in np.nonzero(DL >= 0)[0]:
        w = win[DL[d]]
        if w < 0 or Dm[d] > Dm[w]:
            win[DL[d]] = d
    any_match = (DL >= 0).any()
    for l, gc in enumerate(lcls.astype(np.int64)):
        if any_match and win[l] >= 0:
            matrix[int(k_cls[win[l]]), gc] += 1
        else:
            matrix[nc, gc] += 1
    if any_match:
        won = set(win[win >= 0].tolist())
        for d, dc in enumerate(k_cls.astype(np.int64)):
            if d not in won:
                matrix[dc, nc] += 1


def interp(x, xp, fp, left):
    """np.interp for non-decreasing xp: j = the last index with xp[j] <= x (on repeated points the last of them); x == xp[j]
    gives fp[j]; below xp[0] `left`, at or above the last point fp[-1]; otherwise slope * (x - xp[j]) + fp[j]."""
    x, xp, fp = np.asarray(x, np.float64), np.asarray(xp, np.float64), np.asarray(fp, np.float64)
    j = np.searchsorted(xp, x, side="right") - 1
    out = np.empty_like(x)
    below, last = j < 0, j >= len(xp) - 1
    out[below] = left
    out[last] = fp[-1]
    mid = ~below & ~last
    jm, xm = j[mid], x[mid]
    with np.errstate(divide="ignore", invalid="ignore"):
        slope = (fp[jm + 1] - fp[jm]) / (xp[jm + 1] - xp[jm])
        val = slope * (xm - xp[jm]) + fp[jm]
    out[mid] = np.where(xp[jm] == xm, fp[jm], val)
    return out


def compute_ap(recall, precision):
    """101-point interpolated AP over the precision envelope (metrics.py:77-102)."""
    mrec = np.concatenate(([0.0], recall, [recall[-1] + 0.01]))
    mpre = np.concatenate(([1.0], precision, [0.0]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]
    y = interp(X101, mrec, mpre, left=mpre[0])
    return np.sum(np.diff(X101) * (y[1:] + y[:-1]) / 2.0)


def ap_per_class(tp, conf, pred_cls, target_cls):
    """metrics.py:13-74 with a stable sort: ties in conf keep dataset order."""
    i = np.argsort(-conf, kind="stable")
    tp, conf, pred_cls = tp[i], conf[i], pred_cls[i]
    classes = np.unique(target_cls)
    ap, p, r = np.zeros((len(classes), tp.shape[1])), np.zeros((len(classes), 1000)), np.zeros((len(classes), 1000))
    for ci, c in enumerate(classes):
        sel = pred_cls == c
        n_l, n_p = int((target_cls == c).sum()), int(sel.sum())
        if n_p == 0 or n_l == 0:
            continue
        tpc = np.cumsum(tp[sel], 0).astype(np.float64)
        fpc = np.arange(1, n_p + 1, dtype=np.float64)[:, None] - tpc
        recall = tpc / (n_l + 1e-16)
        precision = tpc / (tpc + fpc)
        xp = -conf[sel].astype(np.float64)
        r[ci] = interp(-PX, xp, recall[:, 0], left=0)
        p[ci] = interp(-PX, xp, precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[ci, j] = compute_ap(recall[:, j], precision[:, j])
    f1 = 2 * p * r / (p + r + 1e-16)
    return p, r, ap, f1, classes.astype(np.int32)


def evaluate(batches, nc, confusion=True):
    """batches: list of (preds, targets, shapes, (H, W)); preds a list of per-image [k,6] fp32 NMS rows (letterboxed xyxy,
    conf, cls), targets [n,6] fp32.  Returns the Evaler's stats and summary as a dict."""
    stats, seen = [], 0
    matrix = np.zeros((nc + 1, nc + 1))
    for preds, targets, shapes, hw in batches:
        targets = np.asarray(targets, np.float32)
        for si, pred in enumerate(preds):
            pred = np.asarray(pred, np.float32).reshape(-1, 6)
            labels = targets[targets[:, 0] == si, 1:]
            tcls = labels[:, 0].astype(np.float64)
            seen += 1
            if len(pred) == 0:
                if len(labels):
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
                continue
            correct = np.zeros((len(pred), 10), bool)
            if len(labels):
                iou = box_iou(label_boxes(labels, hw, shapes[si]), pred_boxes(pred, shapes[si]))
                correct = correct_flags(iou, labels[:, 0], pred[:, 5])
                if confusion:
                    confusion_update(matrix, iou, labels[:, 0], pred[:, 4], pred[:, 5], nc)
            stats.append((correct, pred[:, 4], pred[:, 5], tcls))
    if stats:
        correct, conf, pcls, tcls = (np.concatenate(x, 0) for x in zip(*stats))
    else:
        correct, conf, pcls, tcls = np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), np.zeros(0)
    p, r, ap, f1, ap_class = ap_per_class(correct, conf, pcls, tcls)
    res = dict(correct=correct, conf=conf, pcls=pcls, tcls=tcls, p=p, r=r, ap=ap, f1=f1, ap_class=ap_class, seen=seen,
               nt=np.bincount(tcls.astype(np.int64), minlength=nc), matrix=matrix, ok=bool(correct.any()),
               map50=0.0, map=0.0, mp=0.0, mr=0.0, best=-1)
    if res["ok"]:
        f1m = f1.mean(0)
        best = len(f1m) - f1m[::-1].argmax() - 1                  # the last arg-max (evaler.py:202)
        res.update(best=int(best), mp=float(p[:, best].mean()), mr=float(r[:, best].mean()), map50=float(ap[:, 0].mean()),
                   map=float(ap.mean(1).mean()))
    return res


# ------------------------------------------------------------------------------------------------
# seeded synthetic validation sets
# ------------------------------------------------------------------------------------------------
def letterbox_shape(h0, w0, H, W):
    """The Evaler dataloader's shapes entry for a (h0, w0) source letterboxed to (H, W) (datasets.py:197-198)."""
    r = min(H / h0, W / w0)
    nh, nw = int(round(h0 * r)), int(round(w0 * r))
    return (h0, w0), ((nh / h0, nw / w0), ((W - nw) / 2, (H - nh) / 2))


def synthetic_batch(rng, B, H, W, nc, *, max_labels=8, dets_per_label=3, fp_rate=2.0, p_no_labels=0.15, p_no_dets=0.15,
                    p_wrong_cls=0.15, p_dup=0.2, conf_lo=0.03, label_classes=None, pred_only_classes=(), iou_span=(0.3, 1.0)):
    """One batch of letterboxed NMS rows (sorted by conf, like nms_batched's output), targets and shapes.  Detections are
    jittered copies of labels (IoU roughly in `iou_span`), label boxes may cross the canvas edge, some detections take a
    wrong class, some are duplicated under another class (multi-label NMS), and random false positives are added."""
    label_classes = np.arange(nc) if label_classes is None else np.asarray(label_classes)
    preds, targets, shapes = [], [], []
    for b in range(B):
        h0, w0 = int(rng.integers(200, 1400)), int(rng.integers(200, 1400))
        shapes.append(letterbox_shape(h0, w0, H, W))
        nl = 0 if rng.random() < p_no_labels else int(rng.integers(1, max_labels + 1))
        labs = []
        for _ in range(nl):
            w, h = rng.uniform(0.03, 0.5), rng.uniform(0.03, 0.5)
            x, y = rng.uniform(-0.05, 1.05), rng.uniform(-0.05, 1.05)       # centres near the edge cross it
            labs.append([b, float(rng.choice(label_classes)), x, y, w, h])
        targets += labs
        rows = []
        if rng.random() >= p_no_dets:
            for lab in labs:
                for _ in range(int(rng.integers(0, dets_per_label + 1))):
                    s = rng.uniform(0.0, 1.0 - iou_span[0]) ** 1.5
                    x1 = (lab[2] - lab[4] / 2 + rng.uniform(-s, s) * lab[4]) * W
                    y1 = (lab[3] - lab[5] / 2 + rng.uniform(-s, s) * lab[5]) * H
                    x2 = (lab[2] + lab[4] / 2 + rng.uniform(-s, s) * lab[4]) * W
                    y2 = (lab[3] + lab[5] / 2 + rng.uniform(-s, s) * lab[5]) * H
                    c = lab[1] if rng.random() >= p_wrong_cls else float(rng.integers(0, nc))
                    rows.append([min(x1, x2), min(y1, y2), max(x1, x2) + 1, max(y1, y2) + 1, rng.uniform(conf_lo, 1.0), c])
                    if rng.random() < p_dup:                                 # same box, another class
                        rows.append(rows[-1][:4] + [rng.uniform(conf_lo, 0.25), float(rng.integers(0, nc))])
            for _ in range(int(rng.poisson(fp_rate))):
                x1, y1 = rng.uniform(0, W - 20), rng.uniform(0, H - 20)
                pool = list(pred_only_classes) + list(range(nc)) if len(pred_only_classes) else range(nc)
                rows.append([x1, y1, x1 + rng.uniform(8, W / 3), y1 + rng.uniform(8, H / 3), rng.uniform(conf_lo, 1.0),
                             float(rng.choice(pool))])
        rows = np.array(rows, np.float32).reshape(-1, 6)
        rows[:, :4] = np.clip(rows[:, :4], 0, [W, H, W, H])
        preds.append(rows[np.argsort(-rows[:, 4], kind="stable")])
    return preds, np.array(targets, np.float32).reshape(-1, 6), shapes


def assert_no_ties(batches, nc):
    """The reference's argsorts are unstable: a golden is only well defined without conf ties within a class and without
    IoU ties among the candidates of one detection or of one label."""
    seen = {}
    for preds, targets, shapes, hw in batches:
        for si, pred in enumerate(preds):
            for c, f in zip(pred[:, 5], pred[:, 4]):
                assert (c, f) not in seen, f"conf tie in class {c}"
                seen[(c, f)] = 1
            labels = targets[targets[:, 0] == si, 1:]
            if not len(labels) or not len(pred):
                continue
            iou = box_iou(label_boxes(labels, hw, shapes[si]), pred_boxes(pred, shapes[si]))
            for d in range(iou.shape[1]):
                col = iou[:, d]
                for ok in (labels[:, 0] == pred[d, 5], np.ones(len(col), bool)):
                    v = col[ok & (col >= np.float32(0.45))]
                    assert len(np.unique(v)) == len(v), "IoU tie for one detection"
            keep = pred[:, 4] > np.float32(0.25)
            for l in range(iou.shape[0]):
                v = iou[l, keep]
                v = v[v > np.float32(0.45)]
                assert len(np.unique(v)) == len(v), "IoU tie for one label"


def dataset(seed, n_batches, B, H, W, nc, last_batch=None, **kw):
    """Seeded batches; redraws a batch until it has no ties (see assert_no_ties) when kw has no_ties=True."""
    no_ties = kw.pop("no_ties", False)
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_batches):
        bs = last_batch if (last_batch and i == n_batches - 1) else B
        while True:
            preds, targets, shapes = synthetic_batch(rng, bs, H, W, nc, **kw)
            batch = (preds, targets, shapes, (H, W))
            if not no_ties:
                break
            try:
                assert_no_ties(out + [batch], nc)
                break
            except AssertionError:
                continue
        out.append(batch)
    return out


def coco_val_sized(seed=5, n_images=5000, B=32, nc=80):
    """5000 images in batches of 32 (the last partial), up to 300 rows per image; conf quantised to 1/256 gives ties within
    a class, duplicated label boxes give IoU ties between labels."""
    nb = (n_images + B - 1) // B
    batches = dataset(seed, nb, B, 640, 640, nc, last_batch=n_images - (nb - 1) * B, max_labels=24, dets_per_label=4, fp_rate=30.0)
    rng = np.random.default_rng(seed + 1)
    out = []
    for preds, targets, shapes, hw in batches:
        qp = []
        for p in preds:
            if rng.random() < 0.02:                                   # a crowded image: false positives up to max_det
                k = 300 - len(p)
                x1, y1 = rng.uniform(0, 600, k), rng.uniform(0, 600, k)
                extra = np.stack([x1, y1, x1 + rng.uniform(4, 40, k), y1 + rng.uniform(4, 40, k), rng.uniform(0.03, 1, k),
                                  rng.integers(0, nc, k)], 1).astype(np.float32)
                p = np.concatenate([p, extra])
            p = p.copy()
            p[:, 4] = np.round(p[:, 4] * 256) / 256
            qp.append(p[np.argsort(-p[:, 4], kind="stable")][:300])
        dup = targets[rng.random(len(targets)) < 0.1]
        out.append((qp, np.concatenate([targets, dup]) if len(dup) else targets, shapes, hw))
    return out, nc


def pack(preds, max_det):
    """Per-image rows -> the batched NMS layout: out [B,max_det,6] fp32 (zero beyond count), count [B] int32."""
    out = np.zeros((len(preds), max_det, 6), np.float32)
    count = np.zeros(len(preds), np.int32)
    for i, p in enumerate(preds):
        out[i, :len(p)] = p
        count[i] = len(p)
    return out, count
