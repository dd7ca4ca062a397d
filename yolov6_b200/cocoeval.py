"""The COCO box mAP on the GPU: pycocotools' COCOeval (iouType 'bbox', default Params) as the reference's Evaler.eval_model
runs it (yolov6/core/evaler.py:231-321), fed straight from the batched NMS tensors.

The reference dumps every detection to predictions.json, reads it back with `COCO.loadRes` and runs `COCOeval.evaluate /
accumulate / summarize`: Python loops over every (image, category, area range).  Here the gt json is parsed once and
uploaded, `COCOMetric.update` is one kernel launch per batch (`yv6_coco_update`: the json rows' geometry and rounding,
the per-(image, category) ranking and greedy matching), and `COCOMetric.result` sorts and accumulates on the device
(`yv6_coco_accumulate`) and copies precision / recall / scores to the host, where the 12 summary numbers are taken with
numpy exactly as `summarize()` takes them.

    m = COCOMetric(anno_json, class_to_category=ids, img_ids=img_ids, device=dev)
    for imgs, targets, paths, shapes in dataloader:
        ...                                             # pipe = DetectPipeline(..., host_input=False, multi_label=True)
        m.update(pipe.out_dev, pipe.count_dev, shapes, [int(Path(p).stem) for p in paths])
    res = m.result()                                    # res.stats[:2] = (mAP@0.5:0.95, mAP@0.5)

`load_results` takes the Evaler's pred_results (or a predictions.json) instead, as `loadRes` does.
"""
import ctypes as C
import json
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .evalpost import image_meta

# Params.setDetParams
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)
LOAD_CHUNK = 4096                                       # images per yv6_coco_load launch


@dataclass
class COCOResult:
    """`stats` are COCOeval.stats (12 numbers, summarize()'s order); `precision` [10,101,K,4,3], `recall` [10,K,4,3] and
    `scores` [10,101,K,4,3] are COCOeval.eval's arrays; `cat_ids` / `img_ids` are params.catIds / params.imgIds."""
    stats: np.ndarray
    precision: np.ndarray
    recall: np.ndarray
    scores: np.ndarray
    cat_ids: list
    img_ids: list


def summarize(precision, recall):
    """COCOeval.summarize's 12 numbers: each the mean over the entries > -1 of its slice, -1 when there are none."""

    def _s(ap=1, iouThr=None, areaRng="all", maxDets=100):
        aind = [i for i, r in enumerate(AREA_LBL) if r == areaRng]
        mind = [i for i, d in enumerate(MAX_DETS) if d == maxDets]
        s = precision if ap == 1 else recall
        if iouThr is not None:
            s = s[np.where(iouThr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    return np.array([_s(1), _s(1, iouThr=.5), _s(1, iouThr=.75), _s(1, areaRng="small"), _s(1, areaRng="medium"),
                     _s(1, areaRng="large"), _s(0, maxDets=1), _s(0, maxDets=10), _s(0), _s(0, areaRng="small"),
                     _s(0, areaRng="medium"), _s(0, areaRng="large")], dtype=np.float64)


class COCOMetric:
    """Device state of one COCO box evaluation.  anno: the instances json (path or dict); class_to_category: the Evaler's
    `ids` (model class -> category id); img_ids: params.imgIds (None: every gt image); max_det: NMS rows per image."""

    def __init__(self, anno, class_to_category, img_ids=None, max_det=300, device=None, iou_type="bbox", use_cats=1):
        if iou_type != "bbox" or use_cats != 1:
            raise RuntimeError(f"COCOMetric: only iouType='bbox' with useCats=1 is supported (got {iou_type!r}, {use_cats})")
        if max_det <= 0:
            raise RuntimeError(f"COCOMetric: max_det={max_det} must be positive")
        dev = torch.device(device if device is not None else "cuda")
        if dev.type != "cuda":
            raise RuntimeError("yolov6_b200.cocoeval runs on CUDA devices only (no CPU fallback)")
        self.dev = dev = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        if not isinstance(anno, dict):
            with open(anno) as f:
                anno = json.load(f)
        self.cat_ids = sorted(c["id"] for c in anno["categories"])
        if not self.cat_ids:
            raise RuntimeError("COCOMetric: the gt json has no categories")
        self._cat_of = {c: i for i, c in enumerate(self.cat_ids)}
        self._gt_images = {im["id"] for im in anno["images"]}
        ids = sorted(self._gt_images) if img_ids is None else list(img_ids)
        self.img_ids = np.unique(ids).tolist() if len(ids) else []
        if not self.img_ids:
            raise RuntimeError("COCOMetric: no images to evaluate")
        self._slot_of = {v: i for i, v in enumerate(self.img_ids)}
        self.max_det = int(max_det)
        self.cls_cat = torch.tensor([self._cat_of.get(c, -1) for c in class_to_category] or [-1], dtype=torch.int32).to(dev)
        self.n_cls = len(class_to_category)
        I, K = len(self.img_ids), len(self.cat_ids)

        # gts of the evaluated images and categories, CSR by (slot, category) in annotation-file order (_prepare)
        key, box, area, flags = [], [], [], []
        for g in anno["annotations"]:
            s, c = self._slot_of.get(g["image_id"], -1), self._cat_of.get(g["category_id"], -1)
            if s < 0 or c < 0:
                continue
            crowd = bool(g.get("iscrowd", 0))                 # _prepare: ignore = iscrowd
            key.append(s * K + c)
            box.append([float(v) for v in g["bbox"]])
            area.append(float(g["area"]))
            flags.append(int(crowd) | (2 if g["id"] != 0 else 0))
        key = np.array(key, np.int64)
        order = np.argsort(key, kind="stable")
        box = np.array(box, np.float64).reshape(-1, 4)[order]
        area = np.array(area, np.float64)[order]
        flags = np.array(flags, np.uint8)[order]
        per_pair = np.bincount(key, minlength=I * K)
        off = np.zeros(I * K + 1, np.int64)
        np.cumsum(per_pair, out=off[1:])
        if off[-1] >= 2 ** 31:
            raise RuntimeError("COCOMetric: too many gts")
        self.max_gts = int(per_pair.max()) if len(per_pair) else 0
        # npig per (category, area range): gts neither crowd nor outside the range
        cats = key[order] % K if len(key) else key
        npig = np.zeros((K, A), np.int32)
        for a, (lo, hi) in enumerate(AREA_RNG):
            ok = ((flags & 1) == 0) & ~((area < lo) | (area > hi))
            npig[:, a] = np.bincount(cats[ok], minlength=K)
        self.npig = npig

        def up(x):
            return torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        self.gt_off = up(off.astype(np.int32))
        self.gt_box = up(box if len(box) else np.zeros((1, 4)))
        self.gt_area = up(area if len(area) else np.zeros(1))
        self.gt_flags = up(flags if len(flags) else np.zeros(1, np.uint8))
        self.npig_dev = up(npig)
        self.area_rng = up(np.array(AREA_RNG, np.float64))
        self.iou_thrs = up(IOU_THRS)
        self.rec_thrs = up(REC_THRS)
        n = I * self.max_det
        self.score = torch.zeros(n, dtype=torch.float64, device=dev)
        self.cat = torch.zeros(n, dtype=torch.int32, device=dev)
        self.rank = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.tp = torch.zeros(n, dtype=torch.int64, device=dev)
        self.fp = torch.zeros(n, dtype=torch.int64, device=dev)
        self.ndet = torch.zeros(I, dtype=torch.int32, device=dev)
        self.flags = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ws = torch.empty(int(_lib.lib().yv6_coco_workspace_bytes(I, self.max_det, K)), dtype=torch.uint8, device=dev)
        self.out = torch.empty(2 * T * R * K * A * M + T * K * A * M, dtype=torch.float64, device=dev)
        p = lambda t: t.data_ptr()  # noqa: E731
        self.state = _lib.CocoState(I, K, self.max_det, self.max_gts, p(self.gt_off), p(self.gt_box), p(self.gt_area), p(self.gt_flags),
                                    p(self.npig_dev), p(self.area_rng), p(self.iou_thrs), p(self.rec_thrs), p(self.score), p(self.cat),
                                    p(self.rank), p(self.tp), p(self.fp), p(self.ndet), p(self.flags))
        self._seen = set()

    def reset(self):
        """Start a new epoch on the same buffers."""
        self.ndet.zero_()
        self.flags.zero_()
        self._seen = set()

    def _slots(self, image_ids, where):
        slots = []
        for i in image_ids:
            if i not in self._gt_images:
                raise RuntimeError(f"COCOMetric.{where}: image id {i!r} is not in the gt json")
            s = self._slot_of.get(i, -1)
            if s >= 0 and (s in self._seen or s in slots):
                raise RuntimeError(f"COCOMetric.{where}: image id {i!r} was given twice")
            slots.append(s)
        return slots

    def update(self, out, count, shapes, image_ids):
        """One batch: out [B,max_det,6] fp32 / count [B] int32, the batched NMS tensors on the device (nms_batched,
        DetectPipeline.out_dev / count_dev); shapes the dataloader's per-image ((h0, w0), ((h_ratio, w_ratio), (pad_w,
        pad_h))); image_ids the gt json's id of each image.  Asynchronous on the current stream."""
        if not (isinstance(out, torch.Tensor) and out.device == self.dev and out.dtype == torch.float32 and out.dim() == 3
                and out.shape[2] == 6 and out.is_contiguous()):
            raise RuntimeError(f"COCOMetric.update: out must be a contiguous fp32 [B,max_det,6] tensor on {self.dev}")
        B, D = int(out.shape[0]), int(out.shape[1])
        if not (isinstance(count, torch.Tensor) and count.device == self.dev and count.dtype == torch.int32 and count.shape == (B,)
                and count.is_contiguous()):
            raise RuntimeError(f"COCOMetric.update: count must be a contiguous int32 [{B}] tensor on {self.dev}")
        if B == 0 or D == 0 or D > self.max_det:
            raise RuntimeError(f"COCOMetric.update: out has {D} rows per image (1..{self.max_det}) and {B} images")
        if len(shapes) != B or len(image_ids) != B:
            raise RuntimeError(f"COCOMetric.update: {len(shapes)} shapes and {len(image_ids)} image ids for {B} images")
        slots = self._slots(image_ids, "update")
        meta = image_meta(shapes, "cpu").pin_memory().to(self.dev, non_blocking=True)
        sl = torch.tensor(slots, dtype=torch.int32).pin_memory().to(self.dev, non_blocking=True)
        _lib.check(_lib.lib().yv6_coco_update(_lib.handle(self.dev.index or 0), C.byref(self.state), C.c_void_p(out.data_ptr()),
                                              C.c_void_p(count.data_ptr()), C.c_void_p(meta.data_ptr()), C.c_void_p(self.cls_cat.data_ptr()),
                                              self.n_cls, C.c_void_p(sl.data_ptr()), B, D, _lib.stream_ptr()))
        self._seen.update(s for s in slots if s >= 0)

    def load_results(self, results):
        """loadRes: the Evaler's pred_results (dicts with image_id, category_id, bbox, score) or a predictions.json path.
        Every image id must be a gt image; rows of other images than params.imgIds, or of categories the gt json does not
        have, are dropped.  Each image's rows keep their order."""
        if not isinstance(results, (list, tuple)):
            with open(results) as f:
                results = json.load(f)
        slots, rows = [], []
        for r in results:
            if r["image_id"] not in self._gt_images:
                raise RuntimeError(f"COCOMetric.load_results: image id {r['image_id']!r} is not in the gt json")
            s, c = self._slot_of.get(r["image_id"], -1), self._cat_of.get(r["category_id"], -1)
            if s < 0 or c < 0:
                continue
            slots.append(s)
            bb = r["bbox"]
            rows.append([float(bb[0]), float(bb[1]), float(bb[2]), float(bb[3]), float(r["score"]), float(c)])
        if not rows:
            return
        slots = np.array(slots, np.int64)
        order = np.argsort(slots, kind="stable")
        uniq, counts = np.unique(slots, return_counts=True)
        if counts.max() > self.max_det:
            raise RuntimeError(f"COCOMetric.load_results: an image has {int(counts.max())} rows (max_det={self.max_det})")
        dup = [self.img_ids[s] for s in uniq.tolist() if s in self._seen]
        if dup:
            raise RuntimeError(f"COCOMetric.load_results: image id {dup[0]!r} was given twice")
        rows = np.array(rows, np.float64)[order]
        off = np.zeros(len(uniq) + 1, np.int64)
        np.cumsum(counts, out=off[1:])
        L, h = _lib.lib(), _lib.handle(self.dev.index or 0)
        for i0 in range(0, len(uniq), LOAD_CHUNK):
            i1 = min(len(uniq), i0 + LOAD_CHUNK)
            rdev = torch.from_numpy(rows[off[i0]:off[i1]]).to(self.dev)
            odev = torch.from_numpy((off[i0:i1 + 1] - off[i0]).astype(np.int32)).to(self.dev)
            sdev = torch.from_numpy(uniq[i0:i1].astype(np.int32)).to(self.dev)
            _lib.check(L.yv6_coco_load(h, C.byref(self.state), C.c_void_p(rdev.data_ptr()), C.c_void_p(odev.data_ptr()),
                                       C.c_void_p(sdev.data_ptr()), i1 - i0, _lib.stream_ptr()))
        self._seen.update(uniq.tolist())

    def result(self):
        """COCOeval.accumulate over every image since the last reset() on the device, then summarize() on the host."""
        K = len(self.cat_ids)
        n_pr = T * R * K * A * M
        o = self.out
        _lib.check(_lib.lib().yv6_coco_accumulate(_lib.handle(self.dev.index or 0), C.byref(self.state), C.c_void_p(self.ws.data_ptr()),
                                                  self.ws.numel(), C.c_void_p(o.data_ptr()), C.c_void_p(o[n_pr:].data_ptr()),
                                                  C.c_void_p(o[n_pr + T * K * A * M:].data_ptr()), _lib.stream_ptr()))
        host = o.cpu().numpy()
        if int(self.flags.cpu()[0]):
            raise RuntimeError(f"COCOMetric: a detection class is outside [0, {self.n_cls}) or not a whole number")
        precision = host[:n_pr].reshape(T, R, K, A, M).copy()
        recall = host[n_pr:n_pr + T * K * A * M].reshape(T, K, A, M).copy()
        scores = host[n_pr + T * K * A * M:].reshape(T, R, K, A, M).copy()
        return COCOResult(stats=summarize(precision, recall), precision=precision, recall=recall, scores=scores,
                          cat_ids=list(self.cat_ids), img_ids=list(self.img_ids))
