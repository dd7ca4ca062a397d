"""The Evaler's precision / recall metric on the GPU (`do_pr_metric`, yolov6/core/evaler.py:109-226).

The reference walks every image in Python (`process_batch`, `ConfusionMatrix.process_batch`, utils/metrics.py:145-215) and
runs `ap_per_class` / `compute_ap` (metrics.py:13-102) in numpy over every detection of the validation set.  Here
`PRMetric.update` is one kernel launch per batch on the batched NMS tensors (`yv6_pr_match`), and `PRMetric.result` sorts
and scores everything on the device (`yv6_pr_metric`) and copies one small block to the host.

    metric = PRMetric(nc=80, max_images=5000, device=dev, confusion=True)
    for imgs, targets, paths, shapes in dataloader:
        ...                                             # pipe = DetectPipeline(..., host_input=False, multi_label=True)
        metric.update(pipe.out_dev, pipe.count_dev, targets, shapes, imgs.shape[2:])
    res = metric.result()                               # res.map50, res.map, res.p, res.r, res.ap, res.matrix, ...
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .evalpost import image_meta

NIOU = 10
NCURVE = 1000


@dataclass
class PRResult:
    """`p, r, ap, f1, ap_class` as ap_per_class returns them (rows = classes that have labels, ascending), `nt` the label
    count per class, `seen` the images, `map50` / `map` the Evaler's pr_metric_result, `mp` / `mr` the mean precision /
    recall at `best` (the last arg-max of f1.mean(0)), `matrix` the (nc+1, nc+1) confusion matrix (zeros unless enabled).
    `ok` is False in the Evaler's "Calculate metric failed" case (no row correct at any threshold): then
    map50 = map = mp = mr = 0 and best = -1."""
    p: np.ndarray
    r: np.ndarray
    ap: np.ndarray
    f1: np.ndarray
    ap_class: np.ndarray
    nt: np.ndarray
    seen: int
    map50: float
    map: float
    mp: float
    mr: float
    best: int
    matrix: np.ndarray
    ok: bool


class PRMetric:
    """Device accumulators of the PR metric for up to `max_images` images with up to `max_det` NMS rows each."""

    def __init__(self, nc, max_images, max_det=300, device=None, confusion=False):
        if nc <= 0 or max_images <= 0 or max_det <= 0:
            raise RuntimeError(f"PRMetric: nc={nc}, max_images={max_images}, max_det={max_det} must be positive")
        dev = torch.device(device if device is not None else "cuda")
        if dev.type != "cuda":
            raise RuntimeError("yolov6_b200.metrics runs on CUDA devices only (no CPU fallback)")
        self.dev = dev = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.nc, self.max_images, self.max_det, self.confusion = int(nc), int(max_images), int(max_det), bool(confusion)
        n = self.max_images * self.max_det
        self.conf = torch.zeros(n, dtype=torch.float32, device=dev)
        self.cls = torch.zeros(n, dtype=torch.float32, device=dev)
        self.correct = torch.zeros(n, dtype=torch.int16, device=dev)
        self.ndet = torch.zeros(self.max_images, dtype=torch.int32, device=dev)
        # nt, npred, matrix, flags: one buffer, cleared by one fill in reset()
        nm = (self.nc + 1) ** 2
        self.counts = torch.zeros(2 * self.nc + nm + 2, dtype=torch.int32, device=dev)
        self.nt, self.npred = self.counts[:self.nc], self.counts[self.nc:2 * self.nc]
        self.matrix, self.flags = self.counts[2 * self.nc:2 * self.nc + nm], self.counts[2 * self.nc + nm:]
        self.iouv = torch.linspace(0.5, 0.95, NIOU).to(dev)                       # evaler.py:112
        self.px = torch.from_numpy(np.linspace(0, 1, NCURVE)).to(dev)             # metrics.py:36
        self.x101 = torch.from_numpy(np.linspace(0, 1, 101)).to(dev)              # metrics.py:96
        self.ws = torch.empty(max(1, int(_lib.lib().yv6_pr_workspace_bytes(self.max_images, self.max_det))), dtype=torch.uint8, device=dev)
        self.out = torch.empty(self._out_size(), dtype=torch.float64, device=dev)
        self.state = _lib.PrState(self.max_images, self.max_det, self.nc, int(self.confusion), self.conf.data_ptr(), self.cls.data_ptr(),
                                  self.correct.data_ptr(), self.ndet.data_ptr(), self.nt.data_ptr(), self.npred.data_ptr(),
                                  self.matrix.data_ptr(), self.flags.data_ptr())
        self.seen = 0
        self._targets = []

    def _out_size(self):
        nc = self.nc
        return nc * (3 * NCURVE + NIOU) + nc + (nc + 1) ** 2 + 8            # YV6_PR_OUT_SIZE

    def reset(self):
        """Start a new epoch on the same buffers."""
        self.counts.zero_()
        self.seen = 0
        self._targets = []

    def update(self, out, count, targets, shapes, img_hw):
        """One batch: out [B,max_det,6] fp32 / count [B] int32, the batched NMS tensors on the device (nms_batched,
        DetectPipeline.out_dev / count_dev); targets [n,6] (image in batch, cls, x, y, w, h) as the Evaler's dataloader gives
        them (host or device); shapes the dataloader's per-image ((h0, w0), ((h_ratio, w_ratio), (pad_w, pad_h))); img_hw the
        letterboxed (H, W).  Asynchronous on the current stream: nothing waits for the device."""
        if not (isinstance(out, torch.Tensor) and out.device == self.dev and out.dtype == torch.float32 and out.dim() == 3
                and out.shape[2] == 6 and out.is_contiguous()):
            raise RuntimeError(f"PRMetric.update: out must be a contiguous fp32 [B,max_det,6] tensor on {self.dev}")
        B, D = int(out.shape[0]), int(out.shape[1])
        if not (isinstance(count, torch.Tensor) and count.device == self.dev and count.dtype == torch.int32 and count.shape == (B,)
                and count.is_contiguous()):
            raise RuntimeError(f"PRMetric.update: count must be a contiguous int32 [{B}] tensor on {self.dev}")
        if B == 0 or D == 0 or D > self.max_det:
            raise RuntimeError(f"PRMetric.update: out has {D} rows per image (1..{self.max_det}) and {B} images")
        if not (isinstance(targets, torch.Tensor) and targets.dtype == torch.float32 and targets.dim() == 2 and targets.shape[1] == 6
                and targets.device in (torch.device("cpu"), self.dev)):
            raise RuntimeError("PRMetric.update: targets must be an fp32 [n,6] tensor on the host or the metric's device")
        if len(shapes) != B:
            raise RuntimeError(f"PRMetric.update: {len(shapes)} shapes for {B} images")
        H, W = int(img_hw[0]), int(img_hw[1])
        if H <= 0 or W <= 0:
            raise RuntimeError(f"PRMetric.update: bad canvas {H}x{W}")
        if self.seen + B > self.max_images:
            raise RuntimeError(f"PRMetric.update: {self.seen + B} images exceed max_images={self.max_images}")
        meta = image_meta(shapes, "cpu").pin_memory().to(self.dev, non_blocking=True)
        if targets.device.type == "cpu":
            kept = targets.contiguous().clone()
            tdev = kept.pin_memory().to(self.dev, non_blocking=True)
        else:
            kept = tdev = targets.contiguous().clone()
        n = int(targets.shape[0])
        L = _lib.lib()
        _lib.check(L.yv6_pr_match(_lib.handle(self.dev.index or 0), C.byref(self.state), C.c_void_p(out.data_ptr()),
                                  C.c_void_p(count.data_ptr()), B, D, C.c_void_p(tdev.data_ptr() if n else None), n,
                                  C.c_void_p(meta.data_ptr()), H, W, C.c_void_p(self.iouv.data_ptr()), self.seen, _lib.stream_ptr()))
        self._targets.append((kept, B))
        self.seen += B

    def result(self):
        """ap_per_class and the Evaler's summary over every image since the last reset(); one device-to-host copy."""
        L = _lib.lib()
        _lib.check(L.yv6_pr_metric(_lib.handle(self.dev.index or 0), C.byref(self.state), self.seen, C.c_void_p(self.px.data_ptr()),
                                   C.c_void_p(self.x101.data_ptr()), C.c_void_p(self.ws.data_ptr()), self.ws.numel(),
                                   C.c_void_p(self.out.data_ptr()), _lib.stream_ptr()))
        host = self.out.cpu().numpy()
        nc = self.nc
        o = 0

        def take(k):
            nonlocal o
            o += k
            return host[o - k:o]
        p = take(nc * NCURVE).reshape(nc, NCURVE)
        r = take(nc * NCURVE).reshape(nc, NCURVE)
        f1 = take(nc * NCURVE).reshape(nc, NCURVE)
        ap = take(nc * NIOU).reshape(nc, NIOU)
        nt = take(nc).astype(np.int64)
        matrix = take((nc + 1) ** 2).reshape(nc + 1, nc + 1).copy()
        s = take(8)
        err = int(s[6])
        if err:
            why = []
            if err & 1:
                why.append("a label class is outside [0, nc) or not a whole number")
            if err & 2:
                why.append("a detection class is outside [0, nc) or not a whole number")
            if err & 4:
                why.append("an image has more labels than the matching kernel holds")
            raise RuntimeError("PRMetric: " + "; ".join(why))
        rows = np.nonzero(nt > 0)[0]
        return PRResult(p=p[rows].copy(), r=r[rows].copy(), ap=ap[rows].copy(), f1=f1[rows].copy(), ap_class=rows.astype(np.int32),
                        nt=nt, seen=self.seen, map50=float(s[0]), map=float(s[1]), mp=float(s[2]), mr=float(s[3]), best=int(s[4]),
                        matrix=matrix, ok=bool(s[5]))

    def stats(self):
        """The Evaler's concatenated `stats` (evaler.py:197): (correct [N,10] bool, conf [N], pcls [N], tcls [M]) in dataset
        order (image, then NMS row / label row)."""
        ndet = self.ndet[:self.seen].cpu().numpy()
        D = self.max_det
        conf = self.conf[:self.seen * D].cpu().numpy().reshape(self.seen, D)
        cls = self.cls[:self.seen * D].cpu().numpy().reshape(self.seen, D)
        bits = self.correct[:self.seen * D].cpu().numpy().view(np.uint16).reshape(self.seen, D)
        keep = np.arange(D)[None, :] < ndet[:, None]
        b = bits[keep]
        correct = ((b[:, None] >> np.arange(NIOU, dtype=np.uint16)[None, :]) & 1).astype(bool)
        tcls = []
        for targets, B in self._targets:
            t = targets.cpu()
            for si in range(B):
                tcls.extend(t[t[:, 0] == si, 1].tolist())
        return correct, conf[keep], cls[keep], np.array(tcls, dtype=np.float64)
