"""oracle/cocoeval.py -- CPU restatement of pycocotools' COCO box evaluation (TEST INFRASTRUCTURE ONLY).

States the rules of yolov6_b200/csrc/yv6_cocoeval.cu, which are those of pycocotools >= 2.0 (`COCO.loadRes`,
`COCOeval._prepare / computeIoU / evaluateImg / accumulate / summarize` and maskApi.c `bbIou`) as the reference's
`Evaler.eval_model` drives them (yolov6/core/evaler.py:231-321): iouType 'bbox', useCats 1, default Params.  The
methods keep pycocotools' names and structure so that they can be read side by side with it; everything is float64.
pycocotools itself is not a dependency: where it imports, tests/test_oracle_cocoeval.py compares the two.
"""
import copy
import json
from collections import defaultdict

import numpy as np

# Params.setDetParams
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]


def load_json(anno):
    """A COCO instances json path or an already parsed dict."""
    if isinstance(anno, dict):
        return anno
    with open(anno) as f:
        return json.load(f)


def load_res(gt, anns):
    """COCO.loadRes for bbox results: every image id must be a gt image; area = w*h of the given box, id = index + 1,
    iscrowd = 0.  anns: a list of {image_id, category_id, bbox, score} or the path of such a json."""
    if isinstance(anns, str):
        with open(anns) as f:
            anns = json.load(f)
    anns = copy.deepcopy(list(anns))
    gt_imgs = {im["id"] for im in gt["images"]}
    ids = {a["image_id"] for a in anns}
    assert ids == (ids & gt_imgs), "Results do not correspond to current coco set"
    for i, a in enumerate(anns):
        bb = a["bbox"]
        a["area"] = bb[2] * bb[3]
        a["id"] = i + 1
        a["iscrowd"] = 0
    return anns


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou: dt [m,4], gt [n,4] (x, y, w, h) -> [m,n] float64, one rounding per operation (no FMA)."""
    o = np.zeros((len(dt), len(gt)))
    for g, G in enumerate(gt):
        ga = G[2] * G[3]
        crowd = bool(iscrowd[g])
        for d, D in enumerate(dt):
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if crowd else (da + ga) - i
            o[d, g] = i / u
    return o


class COCOEvalOracle:
    """COCOeval(cocoGt, cocoGt.loadRes(results), 'bbox') with params.imgIds = img_ids (None: every gt image)."""

    def __init__(self, gt, results, img_ids=None):
        self.gt = load_json(gt)
        self.dts_all = load_res(self.gt, results)
        self.imgIds = list(np.unique(img_ids if img_ids is not None else sorted(im["id"] for im in self.gt["images"])))
        self.catIds = sorted(c["id"] for c in self.gt["categories"])

    def _prepare(self):
        imgset, catset = set(self.imgIds), set(self.catIds)
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        by_img = defaultdict(list)                               # getAnnIds: per image, annotation-file order
        for a in self.gt["annotations"]:
            by_img[a["image_id"]].append(a)
        for img in self.imgIds:
            for g in by_img.get(img, []):
                if g["category_id"] in catset:
                    g = dict(g)
                    g["ignore"] = int(bool("iscrowd" in g and g["iscrowd"]))
                    self._gts[img, g["category_id"]].append(g)
        for d in self.dts_all:
            if d["image_id"] in imgset and d["category_id"] in catset:
                self._dts[d["image_id"], d["category_id"]].append(d)

    def evaluate(self):
        self._prepare()
        self.ious = {(i, c): self.computeIoU(i, c) for i in self.imgIds for c in self.catIds}
        self.evalImgs = [self.evaluateImg(i, c, a, MAX_DETS[-1]) for c in self.catIds for a in AREA_RNG for i in self.imgIds]

    def computeIoU(self, imgId, catId):
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in inds][:MAX_DETS[-1]]
        if len(gt) == 0 or len(dt) == 0:
            return []
        return bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gt], [int(o["iscrowd"]) for o in gt])

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        ig = [1 if (g["ignore"] or (g["area"] < aRng[0] or g["area"] > aRng[1])) else 0 for g in gt]
        gtind = np.argsort(ig, kind="mergesort")
        gt = [gt[i] for i in gtind]
        gtIg = np.array([ig[i] for i in gtind])
        dtind = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o["iscrowd"]) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        gtm = np.zeros((T, G))
        dtm = np.zeros((T, D))
        dtIg = np.zeros((T, D))
        if len(ious) != 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:      # matched and not a crowd
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:     # matched a regular gt, now on ignored ones
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]["id"]                           # the gt's id: id 0 reads as "no match" below
                    gtm[tind, m] = d["id"]
        a = np.array([d["area"] < aRng[0] or d["area"] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"dtMatches": dtm, "dtScores": [d["score"] for d in dt], "gtIgnore": gtIg, "dtIgnore": dtIg}

    def accumulate(self):
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.catIds), len(AREA_RNG), len(MAX_DETS)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        I0 = len(self.imgIds)
        for k in range(K):
            Nk = k * A * I0
            for a in range(A):
                Na = a * I0
                for m, maxDet in enumerate(MAX_DETS):
                    E = [self.evalImgs[Nk + Na + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e["dtScores"][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind="mergesort")
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e["dtMatches"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e["dtIgnore"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp, fp = np.array(tp), np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q, ss = np.zeros((R,)), np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr, q = pr.tolist(), q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, REC_THRS, side="left")
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {"precision": precision, "recall": recall, "scores": scores}

    def summarize(self):
        self.stats = summarize(self.eval["precision"], self.eval["recall"])
        return self.stats

    def run(self):
        self.evaluate()
        self.accumulate()
        return self.summarize()


def summarize(precision, recall):
    """COCOeval.summarize's 12 numbers from eval['precision'] [T,R,K,A,M] and eval['recall'] [T,K,A,M]."""

    def _s(ap=1, iouThr=None, areaRng="all", maxDets=100):
        aind = [i for i, r in enumerate(AREA_LBL) if r == areaRng]
        mind = [i for i, d in enumerate(MAX_DETS) if d == maxDets]
        s = precision if ap == 1 else recall
        if iouThr is not None:
            s = s[np.where(iouThr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    stats = np.zeros((12,))
    stats[0] = _s(1)
    stats[1] = _s(1, iouThr=.5, maxDets=100)
    stats[2] = _s(1, iouThr=.75, maxDets=100)
    stats[3] = _s(1, areaRng="small", maxDets=100)
    stats[4] = _s(1, areaRng="medium", maxDets=100)
    stats[5] = _s(1, areaRng="large", maxDets=100)
    stats[6] = _s(0, maxDets=1)
    stats[7] = _s(0, maxDets=10)
    stats[8] = _s(0, maxDets=100)
    stats[9] = _s(0, areaRng="small", maxDets=100)
    stats[10] = _s(0, areaRng="medium", maxDets=100)
    stats[11] = _s(0, areaRng="large", maxDets=100)
    return stats


def evaluate(gt, results, img_ids=None):
    """(stats [12], precision, recall, scores) of pycocotools' bbox evaluation."""
    e = COCOEvalOracle(gt, results, img_ids)
    stats = e.run()
    return stats, e.eval["precision"], e.eval["recall"], e.eval["scores"]


# ------------------------------------------------------------------------------------------------
# seeded fabricated sets
# ------------------------------------------------------------------------------------------------
def fabricate(seed, n_images, n_cats=80, gts_per_image=7.4, crowd=0.01, dets=300, H=640, W=640, B=32, p_tie=0.05, p_full=0.7):
    """A COCO-like gt json (non-contiguous category ids, image ids shuffled, annotation ids from 1 with one id-0 gt) and
    batches of letterboxed NMS output: per batch (out [B,dets,6] fp32 xyxy/conf/cls, count [B] int32, shapes, image_ids).
    Detections are jittered gts (some with the wrong class) plus false positives, up to `dets` rows in a share p_full of
    the images and a few otherwise; conf is quantised so that scores tie.
    Returns (gt, batches, class_to_category)."""
    rng = np.random.default_rng(seed)
    cat_ids = sorted(rng.choice(np.arange(1, 3 * n_cats), n_cats, replace=False).tolist())
    # the Evaler's ids table: class -> category, with one class whose category is not in the json
    ids = list(cat_ids)
    gt = {"images": [], "annotations": [], "categories": [{"id": c, "name": f"c{c}"} for c in cat_ids[:-1]] if n_cats > 1
          else [{"id": c, "name": f"c{c}"} for c in cat_ids]}
    img_ids = rng.choice(np.arange(1, 20 * n_images + 1), n_images, replace=False).tolist()
    ann_id = 1
    per_image = []
    for img in img_ids:
        h0, w0 = int(rng.integers(200, 800)), int(rng.integers(200, 800))
        gt["images"].append({"id": img, "height": h0, "width": w0})
        ng = int(rng.poisson(gts_per_image)) if rng.random() > 0.05 else 0
        boxes = []
        for _ in range(ng):
            # log-uniform side lengths: areas over all three ranges
            bw, bh = np.exp(rng.uniform(np.log(4), np.log(0.9 * w0))), np.exp(rng.uniform(np.log(4), np.log(0.9 * h0)))
            x, y = rng.uniform(0, w0 - bw), rng.uniform(0, h0 - bh)
            c = int(rng.integers(0, n_cats))
            iscrowd = int(rng.random() < crowd)
            area = bw * bh * (rng.uniform(0.5, 1.0) if rng.random() < 0.5 else 1.0)       # mask-like area <= box area
            gt["annotations"].append({"id": ann_id, "image_id": img, "category_id": ids[c], "bbox": [x, y, bw, bh],
                                      "area": area, "iscrowd": iscrowd})
            ann_id += 1
            boxes.append((c, x, y, bw, bh))
        per_image.append((img, h0, w0, boxes))
    if gt["annotations"]:
        gt["annotations"][len(gt["annotations"]) // 2]["id"] = 0          # the generated-labels id 0
    batches = []
    for b0 in range(0, n_images, B):
        chunk = per_image[b0:b0 + B]
        out = np.zeros((len(chunk), dets, 6), np.float32)
        count = np.zeros(len(chunk), np.int32)
        shapes, bids = [], []
        for bi, (img, h0, w0, boxes) in enumerate(chunk):
            r = min(H / h0, W / w0)
            nh, nw = int(round(h0 * r)), int(round(w0 * r))
            gain, pad = (nh / h0, nw / w0), ((W - nw) / 2, (H - nh) / 2)
            shapes.append(((h0, w0), (gain, pad)))
            bids.append(img)
            rows = []
            for c, x, y, bw, bh in boxes:
                for _ in range(int(rng.integers(1, 4))):
                    j = rng.normal(0, 0.08, 4) * [bw, bh, bw, bh]
                    cc = c if rng.random() < 0.9 else int(rng.integers(0, n_cats))
                    rows.append([x + j[0], y + j[1], x + bw + j[2], y + bh + j[3], rng.uniform(0.2, 1.0), cc])
            n_fp = max(0, dets - len(rows)) if rng.random() < p_full else int(rng.integers(0, 20))
            bw, bh = np.exp(rng.uniform(np.log(2), np.log(w0), n_fp)), np.exp(rng.uniform(np.log(2), np.log(h0), n_fp))
            x, y = rng.uniform(-10, w0, n_fp), rng.uniform(-10, h0, n_fp)
            fps = np.stack([x, y, x + bw, y + bh, rng.uniform(0.001, 0.6, n_fp), rng.integers(0, n_cats, n_fp)], 1)
            rows = np.concatenate([np.array(rows, np.float64).reshape(-1, 6), fps])
            tie = rng.random(len(rows)) < p_tie
            rows[tie, 4] = np.round(rows[tie, 4] * 16) / 16
            rows = rows[np.argsort(-rows[:, 4], kind="stable")][:dets]
            # to the letterboxed canvas, as the model sees it
            rows[:, [0, 2]] = rows[:, [0, 2]] * gain[1] + pad[0]
            rows[:, [1, 3]] = rows[:, [1, 3]] * gain[0] + pad[1]
            out[bi, :len(rows)] = rows
            count[bi] = len(rows)
        batches.append((out, count, shapes, bids))
    return gt, batches, ids


def rows_of(batches, ids):
    """The Evaler's pred_results for fabricated batches: oracle.evalpost.convert_to_coco_format per batch."""
    import torch

    from oracle.evalpost import convert_to_coco_format
    res = []
    for out, count, shapes, bids in batches:
        preds = [torch.from_numpy(out[i, :count[i]].copy()) for i in range(len(count))]
        res += convert_to_coco_format(preds, [f"{i}.jpg" for i in bids], shapes, ids, is_coco=isinstance(bids[0], int))
    return res
