"""Training augmentation on the device: decoded frames in, the `TrainStep` batch out.

The reference builds every training sample on the host in `TrainValDataset.__getitem__` (yolov6/data/datasets.py:166-255):
`load_image`'s INTER_LINEAR resize, a 2H x 2W mosaic canvas (or a letterbox), `random_affine`'s cv2.warpAffine, mixup,
`augment_hsv`'s BGR -> HSV -> LUT -> BGR round trip and the flips.  Here that work is split three ways:

  - `Sampler` draws every random number the reference draws, in the reference's order, from the same generators (Python's
    global `random` and numpy's global `np.random`), and returns one plain-data `Sample` per image.  A training script that
    seeds those generators as the reference does gets the reference's augmentation sequence.
  - `sample_labels` moves the labels with the reference's own float64 / float32 numpy expressions: about seven boxes per
    image are not worth a kernel, and the same arithmetic gives the same rows.
  - Two kernels per batch (`yv6_aug_resize_frames` / `yv6_aug_resize`, `yv6_augment`, csrc/yv6_augment.cu) produce the
    pixels, bit-exact against the cv2 calls above.  The canvas is never materialised: a per-sample table describes it as
    a 114 background with up to four placed rectangles of resized sources, and the augment kernel samples it where
    warpAffine would.

`AugmentFeed` ties them to a `TrainStep`: it stages the sources of batch i+1 in pinned memory, copies and resizes them on
side streams while batch i's graphs run, and writes the augmented images straight into the step's static uint8 input,
ordered by events rather than host synchronisation.  Frames may also be CUDA tensors (a GPU decoder's output, read in
place), and `FrameCache` is the reference's --cache-ram in device memory.  JPEGs are decoded on the device, with
cv2.imread's pixels, by `jpeg.JpegDecoder` (its frames and `ready` event go straight into `submit` or `FrameCache.put`);
other formats, and the JPEG kinds it refuses, are decoded by the caller.

Off the square: `Sampler(..., target="specific")` is `--specific-shape` (every sample on one H x W, load_image at
min(W / w0, H / h0)); `target="rect"` with `rect_batches` is `--rect` (each batch on its own aspect-ratio canvas, which
`Sampler.draw` / `AugmentFeed.draw` take per batch).  Not provided: `shrink_size` datasets and the dataloader's workers.
"""
import ctypes as C
import math
import random
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from .preprocess import LAYOUTS, REC, check_frame

# yolov6/configs/*.py data_aug of the two flagship configurations
HYP_YOLOV6S = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, flipud=0.0,
                   fliplr=0.5, mosaic=1.0, mixup=0.0)
HYP_YOLOV6L6 = dict(HYP_YOLOV6S, scale=0.9, mixup=0.2)

@dataclass
class Canvas:
    """One canvas of a sample: the source indices placed on it (4 for a mosaic, 1 for a letterbox), the mosaic centre
    (yc, xc; None for a letterbox), and get_transform_matrix's M (float64 3x3) and scale s."""
    indices: list
    yc: int
    xc: int
    M: np.ndarray
    s: float


@dataclass
class Sample:
    """Everything `__getitem__` draws for one image: the mosaic decision, one canvas (two with mixup), the mixup ratio,
    the HSV gains (None when every gain is 0) and the two flips."""
    index: int
    mosaic: bool
    canvases: list = field(default_factory=list)
    mix_r: float = None
    gains: np.ndarray = None
    flipud: bool = False
    fliplr: bool = False

    def sources(self):
        return [i for cv in self.canvases for i in cv.indices]


def transform_matrix(img_shape, new_shape, degrees, scale, shear, translate):
    """get_transform_matrix (data_augment.py:116-143): six random.uniform draws, always made.  cv2.getRotationMatrix2D
    about (0, 0) is [[cos(a') s, sin(a') s], [-sin(a') s, cos(a') s]] with a' = a * (pi / 180) in double."""
    new_height, new_width = new_shape
    Cm = np.eye(3)
    Cm[0, 2] = -img_shape[1] / 2
    Cm[1, 2] = -img_shape[0] / 2
    R = np.eye(3)
    a = random.uniform(-degrees, degrees)
    s = random.uniform(1 - scale, 1 + scale)
    ang = a * (math.pi / 180)
    alpha, beta = math.cos(ang) * s, math.sin(ang) * s
    R[:2] = [[alpha, beta, 0.0], [-beta, alpha, 0.0]]
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - translate, 0.5 + translate) * new_width
    T[1, 2] = random.uniform(0.5 - translate, 0.5 + translate) * new_height
    M = T @ S @ R @ Cm
    return M, s


TARGETS = (None, "specific", "rect")


class Sampler:
    """The random draws of TrainValDataset.__getitem__ with augment=True, for a dataset of `n_images` images, training
    images of H x W and `load_image` size `img_size` (default max(H, W)).

    `target` says where __getitem__'s target_shape comes from, which decides load_image's size and the letterbox branch's
    label arithmetic (`sample_labels`):
      - None: the original rule of this class (an img_size load; float64 box arithmetic when H != W);
      - "specific": --specific-shape, (height, width) as a Python tuple: load at min(W / w0, H / h0) (datasets.py:279-281),
        box arithmetic in float32 at every shape;
      - "rect": a numpy row of --rect's batch_shapes: an img_size load, box arithmetic in float64 at every shape, square
        canvases included.  Each batch names its canvas in `draw(indices, canvas)`."""

    def __init__(self, n_images, H, W, hyp, img_size=None, target=None):
        if target not in TARGETS:
            raise ValueError(f"augment: target must be one of {TARGETS}, got {target!r}")
        self.n, self.H, self.W, self.hyp = int(n_images), int(H), int(W), dict(hyp)
        self.img_size = int(img_size or max(H, W))
        self.target = target

    def _mosaic(self, index, H, W):
        """get_mosaic (datasets.py:452-467) + the draws of mosaic_augmentation (data_augment.py:156, 201)."""
        indices = [index] + random.choices(range(0, self.n), k=3)
        random.shuffle(indices)
        yc, xc = (int(random.uniform(x // 2, 3 * x // 2)) for x in (H, W))
        h = self.hyp
        M, s = transform_matrix((2 * H, 2 * W), (H, W), h["degrees"], h["scale"], h["shear"], h["translate"])
        return Canvas(indices, yc, xc, M, s)

    def draw_one(self, index, canvas=None):
        h = self.hyp
        H, W = canvas or (self.H, self.W)
        rec = Sample(int(index), random.random() < h["mosaic"])
        if rec.mosaic:
            rec.canvases.append(self._mosaic(index, H, W))
            if random.random() < h["mixup"]:
                rec.canvases.append(self._mosaic(random.randint(0, self.n - 1), H, W))
                rec.mix_r = float(np.random.beta(32.0, 32.0))
        else:
            M, s = transform_matrix((H, W), (H, W), h["degrees"], h["scale"], h["shear"], h["translate"])
            rec.canvases.append(Canvas([int(index)], None, None, M, s))
        if h["hsv_h"] or h["hsv_s"] or h["hsv_v"]:
            rec.gains = np.random.uniform(-1, 1, 3) * [h["hsv_h"], h["hsv_s"], h["hsv_v"]] + 1
        rec.flipud = random.random() < h["flipud"]
        rec.fliplr = random.random() < h["fliplr"]
        return rec

    def draw(self, indices, canvas=None):
        """One Sample per dataset index, in order, on `canvas` (H, W) (a --rect batch's; default the sampler's H x W).
        `Plan.sources` lists the distinct source images the batch needs."""
        H, W = (int(canvas[0]), int(canvas[1])) if canvas is not None else (self.H, self.W)
        return Plan([self.draw_one(i, (H, W)) for i in indices], H, W)

    def geometry(self):
        """What decides load_image's size: (n_images, target, img_size, and H x W for target="specific")."""
        return self.n, self.target, self.img_size, (self.H, self.W) if self.target == "specific" else None

    def load_shape(self, h0, w0, H, W):
        """load_image's size for a source of h0 x w0 drawn on an H x W canvas."""
        if self.target == "specific":
            return resized_shape(h0, w0, None, (H, W))
        return resized_shape(h0, w0, self.img_size)


def rect_batches(shapes_hw, img_size, batch, stride, world=1, rank=0):
    """--rect's training batches of one rank: [(dataset indices, (H, W) canvas)], as the reference's train loader yields them
    (create_dataloader(rect=True, pad=0.0, shuffle=False), data_load.py:40-92; core/engine.py:385-391) for sources of
    (h0, w0) `shapes_hw` in dataset order.  Batch canvases come from `sort_files_shapes` over batch * world images
    (datasets.py:89-100, 497-520; valdata.val_batches with pad 0); under DDP, DistributedSampler(shuffle=False,
    drop_last=True) gives rank r the sorted positions r::world of the first floor(n / world) * world.  `stride` is
    max(max(model strides), 32).  The last batch may be short, as the DataLoader's."""
    from .valdata import val_batches
    order, batch_index, canvases = val_batches(shapes_hw, img_size, batch * world, stride, pad=0.0)
    n = len(order)
    pos = range(n) if world == 1 else range(rank, n // world * world, world)
    per_rank = min(batch, n)                 # create_dataloader's batch_size = min(batch_size, len(dataset))
    out = []
    for k in range(0, len(pos), per_rank):
        p = pos[k:k + per_rank]
        out.append(([int(order[i]) for i in p], tuple(int(v) for v in canvases[batch_index[p[0]]])))
    return out


class Plan:
    """The records of one batch, its canvas H x W and the distinct source indices they read, in first-use order."""

    def __init__(self, samples, H=None, W=None):
        self.samples, self.H, self.W = samples, H, W
        self.sources = list(dict.fromkeys(i for s in samples for i in s.sources()))


def resized_shape(h0, w0, img_size, specific=None):
    """load_image's size (datasets.py:279-295): (int(h0 * r), int(w0 * r)) with r = img_size / max(h0, w0), or with
    `specific` = (H, W) r = min(W / w0, H / h0); (h0, w0) when r == 1."""
    ratio = min(specific[1] / w0, specific[0] / h0) if specific is not None else img_size / max(h0, w0)
    if ratio == 1:
        return h0, w0
    return int(h0 * ratio), int(w0 * ratio)


def letterbox_fit(h, w, H, W):
    """letterbox(..., auto=False, scaleup=True) of an h x w image on H x W: (r, (nw, nh), (left, top))."""
    r = min(H / h, W / w)
    nw, nh = int(round(w * r)), int(round(h * r))
    dw, dh = (W - nw) / 2, (H - nh) / 2
    return r, (nw, nh), (int(round(dw - 0.1)), int(round(dh - 0.1)))


def box_candidates(box1, box2, wh_thr=2, ar_thr=20, area_thr=0.1, eps=1e-16):
    """data_augment.py:69-74."""
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)


def _affine_labels(labels, M, s, height, width):
    """The label half of random_affine (data_augment.py:90-111)."""
    n = len(labels)
    if n:
        xy = np.ones((n * 4, 3))
        xy[:, :2] = labels[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
        xy = xy @ M.T
        xy = xy[:, :2].reshape(n, 8)
        x = xy[:, [0, 2, 4, 6]]
        y = xy[:, [1, 3, 5, 7]]
        new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
        new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
        new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
        i = box_candidates(box1=labels[:, 1:5].T * s, box2=new.T, area_thr=0.1)
        labels = labels[i]
        labels[:, 1:5] = new[i]
    return labels


def _canvas_labels(rec, cv, hw, labels, H, W, target=None):
    """Pixel-space labels of one canvas after its affine: mosaic_augmentation (data_augment.py:158-206) or the letterbox
    branch of __getitem__ (datasets.py:196-229).  `target`: Sampler's."""
    if rec.mosaic:
        tiles = _tiles(hw, cv.yc, cv.xc, H, W)
        labels4 = []
        for (h, w), (y1a, _, x1a, _, y1b, x1b), lab in zip(hw, tiles, labels):
            padw, padh = x1a - x1b, y1a - y1b
            lab = lab.copy()
            if lab.size:
                boxes = np.copy(lab[:, 1:])
                boxes[:, 0] = w * (lab[:, 1] - lab[:, 3] / 2) + padw
                boxes[:, 1] = h * (lab[:, 2] - lab[:, 4] / 2) + padh
                boxes[:, 2] = w * (lab[:, 1] + lab[:, 3] / 2) + padw
                boxes[:, 3] = h * (lab[:, 2] + lab[:, 4] / 2) + padh
                lab[:, 1:] = boxes
            labels4.append(lab)
        labels4 = np.concatenate(labels4, 0)
        labels4[:, 1::2] = np.clip(labels4[:, 1::2], 0, 2 * W)
        labels4[:, 2::2] = np.clip(labels4[:, 2::2], 0, 2 * H)
        return _affine_labels(labels4, cv.M, cv.s, H, W)
    (h, w), lab = hw[0], labels[0].copy()
    ratio, _, pad = letterbox_fit(h, w, H, W)
    if target == "rect" or (target is None and H != W):
        # a numpy row of batch_shapes makes the ratio a numpy float64 and so the box arithmetic below float64 instead of
        # float32; --specific-shape's (height, width) tuple keeps it a Python float.  target=None assumes a non-square
        # shape came from batch_shapes.
        ratio = np.float64(ratio)
    if lab.size:
        w *= ratio
        h *= ratio
        boxes = np.copy(lab[:, 1:])
        boxes[:, 0] = w * (lab[:, 1] - lab[:, 3] / 2) + pad[0]
        boxes[:, 1] = h * (lab[:, 2] - lab[:, 4] / 2) + pad[1]
        boxes[:, 2] = w * (lab[:, 1] + lab[:, 3] / 2) + pad[0]
        boxes[:, 3] = h * (lab[:, 2] + lab[:, 4] / 2) + pad[1]
        lab[:, 1:] = boxes
    return _affine_labels(lab, cv.M, cv.s, H, W)


def sample_labels(rec, shapes, labels, H, W, img_size, target=None):
    """labels_out of __getitem__ (float32 [n, 6], column 0 zero) for a Sample, from the decoded sources' (h0, w0) and
    their YOLO-format labels (float32 [k, 5]: cls, cx, cy, w, h normalised), both keyed by source index.  `target`:
    Sampler's."""
    out = []
    for cv in rec.canvases:
        hw = [resized_shape(*shapes[i], img_size, (H, W) if target == "specific" else None) for i in cv.indices]
        out.append(_canvas_labels(rec, cv, hw, [labels[i] for i in cv.indices], H, W, target))
    lab = np.concatenate(out, 0) if len(out) > 1 else out[0]
    if len(lab):
        h, w = H, W
        lab[:, [1, 3]] = lab[:, [1, 3]].clip(0, w - 1e-3)
        lab[:, [2, 4]] = lab[:, [2, 4]].clip(0, h - 1e-3)
        boxes = np.copy(lab[:, 1:])
        boxes[:, 0] = ((lab[:, 1] + lab[:, 3]) / 2) / w
        boxes[:, 1] = ((lab[:, 2] + lab[:, 4]) / 2) / h
        boxes[:, 2] = (lab[:, 3] - lab[:, 1]) / w
        boxes[:, 3] = (lab[:, 4] - lab[:, 2]) / h
        lab[:, 1:] = boxes
    if rec.flipud and len(lab):
        lab[:, 2] = 1 - lab[:, 2]
    if rec.fliplr and len(lab):
        lab[:, 1] = 1 - lab[:, 1]
    labels_out = torch.zeros((len(lab), 6))
    if len(lab):
        labels_out[:, 1:] = torch.from_numpy(lab)
    return labels_out


def _tiles(hw, yc, xc, H, W):
    """mosaic placement (data_augment.py:162-175) of four h x w tiles: (y1a, y2a, x1a, x2a, y1b, x1b) each."""
    out = []
    for i, (h, w) in enumerate(hw):
        if i == 0:
            x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
            x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
        elif i == 1:
            x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, W * 2), yc
            x1b, y1b = 0, h - (y2a - y1a)
        elif i == 2:
            x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(H * 2, yc + h)
            x1b, y1b = w - (x2a - x1a), 0
        else:
            x1a, y1a, x2a, y2a = xc, yc, min(xc + w, W * 2), min(H * 2, yc + h)
            x1b, y1b = 0, 0
        out.append((y1a, y2a, x1a, x2a, y1b, x1b))
    return out


def check_labels(lab, where):
    """YOLO-format label rows of one image -> float32 [k, 5]; RuntimeError when malformed (check_label_files' rules)."""
    a = np.asarray(lab.numpy() if isinstance(lab, torch.Tensor) else lab, dtype=np.float32)
    if a.size == 0:
        return np.zeros((0, 5), np.float32)
    if a.ndim != 2 or a.shape[1] != 5:
        raise RuntimeError(f"augment: labels of {where} must be [k, 5] (cls, cx, cy, w, h), got shape {a.shape}")
    if not np.isfinite(a).all() or (a < 0).any() or (a[:, 1:] > 1).any():
        raise RuntimeError(f"augment: labels of {where} must be finite, non-negative and normalised to [0, 1]")
    return a


# ---------------------------------------------------------------------------------------------------- the device side
class AugTile(C.Structure):
    """Mirror of `yv6_aug_tile` (include/yv6.h)."""
    _fields_ = [("org", C.c_int64), ("pitch", C.c_int32), ("y0", C.c_int32), ("y1", C.c_int32), ("x0", C.c_int32),
                ("x1", C.c_int32), ("pad", C.c_int32)]


class AugSample(C.Structure):
    """Mirror of `yv6_aug_sample` (include/yv6.h)."""
    _fields_ = [("minv", (C.c_double * 6) * 2), ("mix_r", C.c_double), ("tile", (AugTile * 4) * 2),
                ("ch", C.c_int32 * 2), ("cw", C.c_int32 * 2), ("ntile", C.c_int32 * 2),
                ("mixup", C.c_int32), ("hsv", C.c_int32), ("flipud", C.c_int32), ("fliplr", C.c_int32),
                ("lut", (C.c_uint8 * 256) * 3)]


JOB = 8               # int64 per resize job (YV6_AUG_JOB)


def invert_affine(M):
    """cv::warpAffine's inversion of M[:2] (double), the matrix its kernel maps destination pixels with."""
    m = [float(v) for v in np.asarray(M, np.float64)[:2].reshape(-1)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = m[4] * D, m[0] * D
    m[0] = A11
    m[1] *= -D
    m[3] *= -D
    m[4] = A22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return m


def hsv_luts(gains):
    """augment_hsv's lookup tables (data_augment.py:20-23) for the drawn gains."""
    x = np.arange(0, 256, dtype=np.float64)
    return (((x * gains[0]) % 180).astype(np.uint8), np.clip(x * gains[1], 0, 255).astype(np.uint8),
            np.clip(x * gains[2], 0, 255).astype(np.uint8))


@dataclass
class Source:
    """Where the pixels of one source of a batch come from.  `staged`: a host frame copied into the batch arena (tensor
    `t`); otherwise `base` is its device address (a CUDA frame, or a FrameCache entry).  (h0, w0) is the decoded size the
    labels and load_image use, (ph, pw) the size of the pixels the record addresses (the load size for a cache entry)."""
    t: torch.Tensor
    staged: bool
    h0: int
    w0: int
    ph: int
    pw: int
    base: int
    row_pitch: int
    plane_pitch: int
    layout: int


def as_source(checked, layout):
    """A Source from `preprocess.check_frame`'s result for a frame in `layout`."""
    t, on_dev, h0, w0, row_pitch, plane_pitch = checked
    return Source(t, not on_dev, h0, w0, h0, w0, t.data_ptr() if on_dev else 0, row_pitch, plane_pitch, LAYOUTS[layout])


def batch_tables(sampler, B, plan, srcs):
    """Arena layout, resize jobs and sample tables of one batch (host only), from a Source per plan.sources entry.
    The arena holds the staged host frames back to back, then the first pass's outputs, then the letterbox pass's.  A
    staged BGR HWC frame already at its load size is read in place; every other source gets a first-pass job whose
    record (in_arena, address or arena offset, row_pitch, plane_pitch, layout) says where it lies -- a copy job when it
    is at its load size, so every source reaches the arena as packed BGR HWC.
    Returns (staged bytes, arena bytes, {i: (h0, w0)}, {i: arena offset of a staged frame}, jobs1, recs1, jobs2, samples)."""
    H, W = plan.H, plan.W
    off, loc = 0, {}
    for i in plan.sources:
        if srcs[i].staged:
            loc[i] = off
            off += srcs[i].t.numel()
    used = off
    shapes = {i: (srcs[i].h0, srcs[i].w0) for i in plan.sources}
    jobs1, recs1, jobs2, res, lb = [], [], [], {}, {}
    for i in plan.sources:
        s = srcs[i]
        h, w = sampler.load_shape(s.h0, s.w0, H, W)
        if h < 1 or w < 1:
            raise RuntimeError(f"augment: source {i} of {s.h0}x{s.w0} resizes to {h}x{w}")
        if s.staged and s.layout == _lib.LB_BGR_HWC and (h, w) == (s.h0, s.w0):
            res[i] = (loc[i], h, w)
        else:
            jobs1.append([loc.get(i, 0), s.ph, s.pw, off, h, w, 0, 0])
            recs1.append((s.staged, loc[i] if s.staged else s.base, s.row_pitch, s.plane_pitch, s.layout))
            res[i] = (off, h, w)
            off += h * w * 3
    smp = (AugSample * B)()
    for k, rec in enumerate(plan.samples):
        s = smp[k]
        for j, cv in enumerate(rec.canvases):
            s.minv[j][:] = invert_affine(cv.M)
            if rec.mosaic:
                hw = [res[i][1:] for i in cv.indices]
                s.ch[j], s.cw[j], s.ntile[j] = 2 * H, 2 * W, 4
                for t, (i, (y1a, y2a, x1a, x2a, y1b, x1b)) in enumerate(zip(cv.indices, _tiles(hw, cv.yc, cv.xc, H, W))):
                    o, _, w = res[i]
                    s.tile[j][t] = AugTile(o + ((y1b - y1a) * w + (x1b - x1a)) * 3, w, y1a, y2a, x1a, x2a, 0)
            else:
                i = cv.indices[0]
                o, h, w = res[i]
                _, (nw, nh), (left, top) = letterbox_fit(h, w, H, W)
                if (nh, nw) != (h, w):
                    if i not in lb:
                        jobs2.append([o, h, w, off, nh, nw, 0, 0])
                        lb[i] = off
                        off += nh * nw * 3
                    o = lb[i]
                s.ch[j], s.cw[j], s.ntile[j] = H, W, 1
                s.tile[j][0] = AugTile(o - (top * nw + left) * 3, nw, top, top + nh, left, left + nw, 0)
        s.mixup = int(rec.mix_r is not None)
        s.mix_r = rec.mix_r or 0.0
        s.hsv = int(rec.gains is not None)
        if rec.gains is not None:
            for c, lut in enumerate(hsv_luts(rec.gains)):
                s.lut[c][:] = lut.tolist()
        s.flipud, s.fliplr = int(rec.flipud), int(rec.fliplr)
    return used, off, shapes, loc, jobs1, recs1, jobs2, smp


def frame_records(recs, arena_ptr):
    """The yv6_lb_src table of first-pass records (`batch_tables`) for an arena at device address `arena_ptr`."""
    out = (_lib.LbSrc * max(len(recs), 1))()
    for k, (in_arena, addr, row_pitch, plane_pitch, layout) in enumerate(recs):
        out[k] = _lib.LbSrc(arena_ptr + addr if in_arena else addr, row_pitch, plane_pitch, layout, 0)
    return out


def resize_frames_launch(dev, recs_ptr, jobs_ptr, J, max_pix, base_ptr, stream):
    """yv6_aug_resize_frames on device tables at `recs_ptr` / `jobs_ptr`, in launches of at most 65535 jobs."""
    L, h = _lib.lib(), _lib.handle(dev.index or 0)
    for k in range(0, J, 65535):
        n = min(65535, J - k)
        _lib.check(L.yv6_aug_resize_frames(h, C.c_void_p(recs_ptr + k * REC), C.c_void_p(jobs_ptr + k * JOB * 8), n, max_pix,
                                           C.c_void_p(base_ptr), _lib.stream_ptr(stream)))


class AugmentFeed:
    """Double-buffered device augmentation for batches of `batch` H x W training images.

        feed = AugmentFeed(batch, H, W, hyp, n_images, max_src_bytes, step=train_step)
        plan = feed.draw(indices)                    # Sampler draws; plan.sources = images to decode
        feed.submit(plan, frames, labels)            # frames / labels keyed by source index
        feed.wait()                                  # the current stream waits; step.images / step.targets hold the batch
        out = train_step.run(epoch)

    Off the square: `target` is Sampler's.  With target="rect", H x W is the largest canvas (img_size x img_size), which
    sizes the staging, and each batch brings its own: `feed.draw(indices, canvas)` (`rect_batches` gives both); a step
    built with `shapes` is switched to that canvas by `submit`.  With target="specific", H and W must be multiples of
    `stride` (the model's largest stride when a step is given, else 32).

    `submit` validates every frame and label array ([k, 5] normalised) and raises RuntimeError before anything is
    enqueued.  It then stages the host frames in pinned memory, copies them on a copy stream, resizes every source on an
    augmentation stream -- host frames from the arena, CUDA frames in place, `cache` entries from the FrameCache -- and
    writes the batch into `images` / `targets` once everything enqueued on the caller's stream before the call (the
    previous step) is done.  The host waits only before reusing a staging slot, for the batch submitted two calls
    earlier.  Without `step`, the feed owns `images` and `targets`.  With `cache` (a FrameCache built on this feed's
    `sampler` geometry), sources the cache holds need no frame."""

    def __init__(self, batch, H, W, hyp, n_images, max_src_bytes, img_size=None, step=None, max_targets=None, device=None,
                 target=None, stride=None, cache=None):
        if W % 32:
            raise RuntimeError(f"augment: W ({W}) must be a multiple of 32")
        if target == "specific":
            stride = int(stride or (max(step.eng.g.strides) if step is not None else 32))
            if H % stride or W % stride:
                raise ValueError(f"augment: a specific shape of {H} x {W} is not a multiple of the model's largest stride {stride}")
        self.B, self.H, self.W = int(batch), int(H), int(W)
        self.sampler = Sampler(n_images, H, W, hyp, img_size, target)
        self.img_size = self.sampler.img_size
        self.max_src = int(max_src_bytes)
        self.step = step
        if step is not None:
            full = step.shapes[0] if step.shapes is not None else (step.H, step.W)
            if (step.B, *full) != (self.B, self.H, self.W) or step.images.dtype != torch.uint8:
                raise RuntimeError("augment: the TrainStep must take uint8 [batch, 3, H, W] images")
            self.dev, self.images, self.targets = step.dev, step.images, step.targets
        else:
            self.dev = _cuda_device(device)
            self._store = torch.empty(self.B * 3 * H * W, dtype=torch.uint8, device=self.dev)
            self.images = self._store.view(self.B, 3, H, W)
            self.targets = torch.full((int(max_targets or self.B * 64), 6), -1.0, device=self.dev)
        self.max_targets = self.targets.shape[0]
        if cache is not None and (cache.geometry != self.sampler.geometry() or cache.dev != self.dev):
            raise RuntimeError(f"augment: the FrameCache holds images loaded for {cache.geometry} on {cache.dev}, this feed loads "
                               f"them for {self.sampler.geometry()} on {self.dev}")
        self.cache = cache
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.aug_stream = torch.cuda.Stream(device=self.dev)
        self.slots = [dict(staged=torch.empty(self.max_src, dtype=torch.uint8).pin_memory(), arena=None,
                           samples=torch.empty(self.B * C.sizeof(AugSample), dtype=torch.uint8).pin_memory(),
                           samples_dev=torch.empty(self.B * C.sizeof(AugSample), dtype=torch.uint8, device=self.dev),
                           jobs=torch.empty(2, 2 * 8 * self.B * JOB, dtype=torch.int64).pin_memory(),
                           jobs_dev=torch.empty(2, 2 * 8 * self.B * JOB, dtype=torch.int64, device=self.dev),
                           recs=torch.empty(8 * self.B * REC, dtype=torch.uint8).pin_memory(),
                           recs_dev=torch.empty(8 * self.B * REC, dtype=torch.uint8, device=self.dev),
                           tgt=torch.empty(self.max_targets, 6).pin_memory(), frames=[], done=None) for _ in range(2)]
        self.turn = 0
        self.ready = None

    def draw(self, indices, canvas=None):
        if len(indices) != self.B:
            raise RuntimeError(f"augment: {len(indices)} indices for a batch of {self.B}")
        if canvas is not None:
            h, w = int(canvas[0]), int(canvas[1])
            if h > self.H or w > self.W or w % 32:
                raise RuntimeError(f"augment: canvas {h} x {w} must fit inside {self.H} x {self.W} with a width that is a "
                                   f"multiple of 32")
        return self.sampler.draw(indices, canvas)

    def submit(self, plan, frames, labels, layout="bgr_hwc", ready=None):
        """Enqueue one batch.  frames: {source index: frame} covering the plan.sources the cache does not hold; labels:
        {source index: float32 [k, 5] YOLO rows}.  Returns the host targets [n, 6] (collate_fn's rows).

        A frame is a host image (numpy array or CPU tensor, staged through pinned memory) or a uint8 CUDA tensor on the
        feed's device (read in place); both kinds may be mixed.  `layout` applies to every frame of the call: "bgr_hwc"
        is cv2 imread's [h0, w0, 3] (rows may be padded, e.g. a crop view), "rgb_chw" torchvision's decoders' [3, h0, w0].
        Device frames are read after the work enqueued on the current stream before this call, or after the event
        `ready` when one is given.  Pass `ready` when the frames come from a side stream (a GPU decoder's): the current
        stream usually holds the running step, and waiting for it would serialise this batch's augmentation behind that
        step.  The feed keeps a reference to each device frame until its slot is reused, which waits for this batch, so a
        frame may be dropped right after the call; work enqueued on the current stream after `wait()` for this batch may
        overwrite the frames."""
        srcs = {}
        for i in plan.sources:
            if self.cache is not None and self.cache.cached[i]:
                srcs[i] = self.cache.source(i)
                continue
            if i not in frames:
                raise RuntimeError(f"augment: no frame for source {i}" + (" and the cache does not hold it" if self.cache else ""))
            try:
                srcs[i] = as_source(check_frame(frames[i], layout, self.dev), layout)
            except RuntimeError as e:
                raise RuntimeError(f"augment: source {i}: {e}") from None
        try:
            lab = {i: check_labels(labels[i], f"source {i}") for i in plan.sources}
        except KeyError as e:
            raise RuntimeError(f"augment: no labels for source {e.args[0]}") from None
        used = sum(s.t.numel() for s in srcs.values() if s.staged)
        if used > self.max_src:
            raise RuntimeError(f"augment: the host frames hold {used} bytes, the staging buffer {self.max_src} (raise max_src_bytes)")
        used, total, shapes, loc, jobs1, recs1, jobs2, smp = batch_tables(self.sampler, self.B, plan, srcs)
        H, W = plan.H, plan.W
        tg = [sample_labels(rec, shapes, lab, H, W, self.img_size, self.sampler.target) for rec in plan.samples]
        for k, t in enumerate(tg):
            t[:, 0] = k
        targets = torch.cat(tg, 0)
        if targets.shape[0] > self.max_targets:
            raise RuntimeError(f"augment: {targets.shape[0]} target rows exceed max_targets={self.max_targets}")
        if self.step is not None and self.step.shapes is None and (H, W) != (self.step.H, self.step.W):
            raise RuntimeError(f"augment: a {H} x {W} batch for a TrainStep of {self.step.H} x {self.step.W} (build it with shapes=)")

        slot = self.slots[self.turn]
        self.turn ^= 1
        if slot["done"] is not None:
            slot["done"].synchronize()              # the batch submitted two calls ago has left this slot
        slot["frames"] = [s.t for s in srcs.values() if not s.staged and s.t is not None]
        if slot["arena"] is None or slot["arena"].numel() < total:
            slot["arena"] = torch.empty(max(total, 1), dtype=torch.uint8, device=self.dev)
        arena = slot["arena"]
        for i in plan.sources:
            if srcs[i].staged:
                slot["staged"][loc[i]:loc[i] + srcs[i].t.numel()].copy_(srcs[i].t.view(-1))
        C.memmove(slot["samples"].data_ptr(), C.addressof(smp), C.sizeof(smp))
        recs = frame_records(recs1, arena.data_ptr())
        C.memmove(slot["recs"].data_ptr(), recs, C.sizeof(recs))
        for r, jobs in enumerate((jobs1, jobs2)):
            if jobs:
                slot["jobs"][r, :len(jobs) * JOB].copy_(torch.tensor(jobs, dtype=torch.int64).view(-1))
        n = targets.shape[0]
        slot["tgt"][:n].copy_(targets)

        if self.step is None:                             # the feed's own buffer, viewed at this batch's canvas
            self.images = self._store[:self.B * 3 * H * W].view(self.B, 3, H, W)
        elif self.step.shapes is not None:
            self.step.use_shape(H, W)
            self.images = self.step.images
        released = torch.cuda.Event()
        released.record(torch.cuda.current_stream(self.dev))       # the consumer's previous step has read images / targets
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_stream(self.aug_stream)          # the previous batch is done with this slot's arena
            arena[:used].copy_(slot["staged"][:used], non_blocking=True)
            slot["samples_dev"].copy_(slot["samples"], non_blocking=True)
            slot["jobs_dev"].copy_(slot["jobs"], non_blocking=True)
            slot["recs_dev"][:len(recs1) * REC].copy_(slot["recs"][:len(recs1) * REC], non_blocking=True)
        h = _lib.handle(self.dev.index or 0)
        L = _lib.lib()
        with torch.cuda.stream(self.aug_stream):
            self.aug_stream.wait_stream(self.copy_stream)
            if slot["frames"]:
                self.aug_stream.wait_event(ready if ready is not None else released)
            if any(s.t is None for s in srcs.values()):
                self.aug_stream.wait_event(self.cache.filled)     # the fills that wrote the cached sources
            sp = _lib.stream_ptr(self.aug_stream)
            if jobs1:
                resize_frames_launch(self.dev, slot["recs_dev"].data_ptr(), slot["jobs_dev"][0].data_ptr(), len(jobs1),
                                     max(j[4] * j[5] for j in jobs1), arena.data_ptr(), self.aug_stream)
            if jobs2:
                _lib.check(L.yv6_aug_resize(h, C.c_void_p(arena.data_ptr()), C.c_void_p(slot["jobs_dev"][1].data_ptr()), len(jobs2),
                                            max(j[4] * j[5] for j in jobs2), sp))
            self.aug_stream.wait_event(released)
            _lib.check(L.yv6_augment(h, C.c_void_p(arena.data_ptr()), C.c_void_p(slot["samples_dev"].data_ptr()), self.B, H, W,
                                     C.c_void_p(self.images.data_ptr()), sp))
            self.targets[:n].copy_(slot["tgt"][:n], non_blocking=True)
            if n < self.max_targets:
                self.targets[n:].fill_(-1.0)
            done = torch.cuda.Event()
            done.record(self.aug_stream)
        slot["done"] = self.ready = done
        return targets

    def wait(self):
        """Make the current stream wait for the last submitted batch (no host synchronisation)."""
        if self.ready is None:
            raise RuntimeError("augment: no batch was submitted")
        torch.cuda.current_stream(self.dev).wait_event(self.ready)


def _cuda_device(dev):
    """`dev` (a torch.device, a string or None for the current device) with its CUDA index filled in."""
    dev = torch.device(dev) if dev is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError(f"augment: runs on a CUDA device only (no CPU fallback), got {dev}")
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def cache_layout(shapes_hw, sampler):
    """FrameCache's arena for sources of (h0, w0) `shapes_hw`: each image at load_image's size for `sampler`'s target,
    img_size and H x W, packed BGR HWC back to back.  Returns (load sizes int64 [n, 2], byte offsets int64 [n], total
    bytes) -- the exact count, not cal_cache_occupy's estimate from 32 images."""
    shapes = np.asarray(shapes_hw, dtype=np.int64).reshape(-1, 2)
    loaded = np.array([sampler.load_shape(int(h0), int(w0), sampler.H, sampler.W) for h0, w0 in shapes],
                      dtype=np.int64).reshape(-1, 2)
    bad = np.flatnonzero((shapes < 1).any(1) | (loaded < 1).any(1))
    if len(bad):
        i = int(bad[0])
        raise RuntimeError(f"FrameCache: image {i} of {shapes[i][0]} x {shapes[i][1]} loads at {loaded[i][0]} x {loaded[i][1]}")
    size = loaded[:, 0] * loaded[:, 1] * 3
    offsets = np.zeros(len(shapes), dtype=np.int64)
    offsets[1:] = np.cumsum(size)[:-1]
    return loaded, offsets, int(size.sum())


class FrameCache:
    """--cache-ram on the device: every training image as load_image returns it with augment=True (datasets.py:106-160,
    257-269), so later epochs neither decode nor resize again.

        cache = FrameCache(shapes_hw, feed.sampler, max_bytes)     # RuntimeError when the images need more than max_bytes
        feed = AugmentFeed(..., cache=cache)
        for each batch of the first epoch:
            plan = feed.draw(indices)
            new = {i: decode(i) for i in plan.sources if not cache.cached[i]}
            cache.put(new)                                         # resized into the cache on its own stream
            feed.submit(plan, {}, labels)                          # every source now comes from the cache

    `shapes_hw` are the (h0, w0) of the decoded images in dataset order; `sampler` (the feed's) fixes the target, img_size
    and H x W, and so each image's load size (`cache_layout`).  The images live packed BGR HWC in one device arena of
    exactly `nbytes`.  A feed built with another geometry refuses the cache.  Every rank of a DDP job holds the whole
    dataset, as the reference's does: a mosaic draws any index.  The cache never draws from `random` / `np.random`."""

    def __init__(self, shapes_hw, sampler, max_bytes, device=None):
        self.shapes_hw = np.asarray(shapes_hw, dtype=np.int64).reshape(-1, 2)
        if len(self.shapes_hw) != sampler.n:
            raise RuntimeError(f"FrameCache: {len(self.shapes_hw)} shapes for a sampler of {sampler.n} images")
        self.geometry = sampler.geometry()
        self.loaded, self.offsets, self.nbytes = cache_layout(self.shapes_hw, sampler)
        if self.nbytes > max_bytes:
            raise RuntimeError(f"FrameCache: the {len(self.shapes_hw)} images need {self.nbytes} bytes at their load sizes, "
                               f"max_bytes is {int(max_bytes)}; train from frames instead")
        self.dev = _cuda_device(device)
        self.arena = torch.empty(max(self.nbytes, 1), dtype=torch.uint8, device=self.dev)
        self.cached = np.zeros(len(self.shapes_hw), dtype=bool)
        self.stream = torch.cuda.Stream(device=self.dev)
        self.filled = None                 # event recorded after the last fill
        self._held = []                    # (fill event, device frames it reads)

    def source(self, i):
        """Source of cached image i: a BGR HWC record at its load size, labelled with its decoded (h0, w0)."""
        (h0, w0), (h, w) = self.shapes_hw[i], self.loaded[i]
        return Source(None, False, int(h0), int(w0), int(h), int(w), self.arena.data_ptr() + int(self.offsets[i]), int(w) * 3, 0,
                      _lib.LB_BGR_HWC)

    def put(self, frames, layout="bgr_hwc", ready=None):
        """Resize {index: frame} into the cache (host frames or uint8 CUDA tensors on the cache's device, `layout` as for
        AugmentFeed.submit) on the cache's own stream.  Device frames are read after the work enqueued on the current
        stream before the call, or after the event `ready`; they may be dropped right after the call.  RuntimeError
        before anything is written or enqueued when an index is out of range or already cached, or a frame is unusable
        or differs in size from its shapes_hw entry."""
        srcs = {}
        for i, im in frames.items():
            i = int(i)
            if not 0 <= i < len(self.shapes_hw):
                raise RuntimeError(f"FrameCache: index {i} outside the {len(self.shapes_hw)} images")
            if self.cached[i] or i in srcs:
                raise RuntimeError(f"FrameCache: image {i} is already cached")
            try:
                s = as_source(check_frame(im, layout, self.dev), layout)
            except RuntimeError as e:
                raise RuntimeError(f"FrameCache: image {i}: {e}") from None
            if (s.h0, s.w0) != tuple(int(v) for v in self.shapes_hw[i]):
                raise RuntimeError(f"FrameCache: image {i} is {s.h0} x {s.w0}, its entry in shapes_hw says "
                                   f"{self.shapes_hw[i][0]} x {self.shapes_hw[i][1]}")
            srcs[i] = s
        if not srcs:
            return
        J = len(srcs)
        head = J * (REC + JOB * 8)
        used = sum(s.t.numel() for s in srcs.values() if s.staged)
        host = torch.empty(head + used, dtype=torch.uint8, pin_memory=True)
        jobs, recs, off = [], [], head
        for i, s in srcs.items():
            if s.staged:
                host[off:off + s.t.numel()].copy_(s.t.view(-1))
            jobs.append([0, s.ph, s.pw, int(self.offsets[i]), int(self.loaded[i][0]), int(self.loaded[i][1]), 0, 0])
            recs.append((s.staged, off if s.staged else s.base, s.row_pitch, s.plane_pitch, s.layout))
            off += s.t.numel() if s.staged else 0
        devs = [s.t for s in srcs.values() if not s.staged]
        cur = torch.cuda.current_stream(self.dev)
        with torch.cuda.stream(self.stream):
            buf = torch.empty(head + used, dtype=torch.uint8, device=self.dev)     # freed in this stream's order
            table = frame_records(recs, buf.data_ptr())
            C.memmove(host.data_ptr(), table, C.sizeof(table))
            host[J * REC:head].view(torch.int64).copy_(torch.tensor(jobs, dtype=torch.int64).view(-1))
            buf.copy_(host, non_blocking=True)     # the pinned block is reused only after this copy (torch's host allocator)
            if devs:
                if ready is not None:
                    self.stream.wait_event(ready)
                else:
                    self.stream.wait_stream(cur)
            resize_frames_launch(self.dev, buf.data_ptr(), buf.data_ptr() + J * REC, J, max(j[4] * j[5] for j in jobs),
                                 self.arena.data_ptr(), self.stream)
            filled = torch.cuda.Event()
            filled.record(self.stream)
        self.cached[list(srcs)] = True
        self.filled = filled
        # the caller may drop its device frames: hold them until the fill that reads them is done
        self._held = [(e, t) for e, t in self._held if not e.query()] + ([(filled, devs)] if devs else [])
