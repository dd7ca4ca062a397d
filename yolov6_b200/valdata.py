"""Validation batches from decoded frames: the images, targets and shapes the reference's Evaler gets from its DataLoader.

`Evaler.init_data` (core/evaler.py:84-98) validates through `TrainValDataset(augment=False, rect=infer_on_rect,
pad=0.5 if rect else 0.0)` with `hyp={"shrink_size": shrink_size}` and the model's `stride = int(model.stride.max())`
(evaler.py:68: 32 for the P5 detectors, 64 for the P6 ones); `tools/eval.py` runs it with infer_on_rect=True, and the
Trainer's per-epoch loader (core/engine.py:396-398) is built the same way with rect=True, pad=0.5.  For each image:

1. `load_image` (datasets.py:257-296) resizes the source by r = img_size / max(h0, w0) (or (img_size - shrink_size) /
   max(h0, w0)) to (int(w0 * r), int(h0 * r)) -- truncated, not rounded -- with cv2.INTER_AREA when r < 1 and
   INTER_LINEAR when r > 1; nothing happens at r == 1.
2. `letterbox(img, batch_shape, auto=False, scaleup=False)` pads it onto its batch's canvas, which the rect batch shapes
   (`sort_files_shapes`, datasets.py:498-520) make at least as large as every loaded image, so this step never resizes.
3. `shapes` and the labels (datasets.py:197-246) follow from the truncated loaded size.

With --specific-shape (`Evaler(specific_shape=True, height, width)`, the Trainer's loader with `--specific-shape`) every
canvas is (height, width), load_image's r is min(width / w0, height / h0) whatever shrink_size says, and the batch order is
still rect's when rect is on: `ValFeed(..., specific_shape=(height, width))`.

`val_batches`, `val_geometry` and `val_labels` restate those expressions on the host; `ValFeed` runs steps 1-2 for a whole
batch in one `yv6_letterbox_val` launch, bit-exact against cv2 (OpenCV's INTER_AREA has two paths: the integer-factor
box mean and the generic weighted one; the host picks the one cv::resize would).  Decoding stays with the caller.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .preprocess import GEO, LAYOUTS, REC, check_frames

DBL_EPSILON = 2.220446049250313e-16
DEFAULT_SRC_BYTES = 1920 * 1080 * 3        # staging bytes per image when max_src_bytes is not given: one 1080p frame


def val_batches(shapes_hw, img_size, batch, stride, pad=0.5, rect=True):
    """TrainValDataset's batch layout for sources of (h0, w0) `shapes_hw` (the dataset's own order):
    (order, batch_index, canvases) -- order[k] is the source of the k-th image the loader yields, batch_index[k] its batch
    (floor(k / batch)), canvases [n_batches, 2] int each batch's (H, W).  rect=True is `sort_files_shapes` line for line
    (sources sorted by the float64 aspect ratio w0 / h0 with numpy's default argsort; each side
    ceil(shape * img_size / stride + pad) * stride); rect=False keeps the order and gives every batch the square img_size
    canvas (the Evaler's infer_on_rect=False, where pad is 0)."""
    s = np.array(shapes_hw, dtype=np.float64).reshape(-1, 2)
    if len(s) == 0:
        raise RuntimeError("val_batches: no images")
    batch_indices = np.floor(np.arange(len(s)) / batch).astype(np.int_)
    batch_num = batch_indices[-1] + 1
    if not rect:
        return np.arange(len(s)), batch_indices, np.full((batch_num, 2), img_size, dtype=np.int_)
    ar = s[:, 1] / s[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    shapes = [[1, 1]] * batch_num
    for i in range(batch_num):
        ari = ar[batch_indices == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [1, maxi]
        elif mini > 1:
            shapes[i] = [1 / mini, 1]
    canvases = np.ceil(np.array(shapes) * img_size / stride + pad).astype(np.int_) * stride
    return irect, batch_indices, canvases


class ValGeometry:
    """One image's numbers: mode (`_lib.VAL_*`), source (h0, w0), loaded (h, w), its placement (top, left) on the canvas
    (H, W), and the Evaler's `shapes` entry ((h0, w0), ((h * ratio / h0, w * ratio / w0), (left, top)))."""

    def __init__(self, mode, h0, w0, h, w, top, left, canvas, ratio, shapes):
        self.mode, self.h0, self.w0, self.h, self.w, self.top, self.left = mode, h0, w0, h, w, top, left
        self.canvas, self.ratio, self.shapes = tuple(canvas), ratio, shapes

    def row(self, src_off=0):
        """The image's yv6_letterbox_val geometry row."""
        return [src_off, self.h0, self.w0, self.h, self.w, self.top, self.left, self.mode]


def area_fast(h0, w0, h, w):
    """cv::resize's is_area_fast: both scales 1 / (n / n0), in doubles, within DBL_EPSILON of their rounded integers."""
    sx, sy = 1.0 / (w / w0), 1.0 / (h / h0)
    return abs(sx - round(sx)) < DBL_EPSILON and abs(sy - round(sy)) < DBL_EPSILON


def val_geometry(h0, w0, canvas, img_size, shrink_size=None, specific_shape=False):
    """load_image + letterbox(auto=False, scaleup=False) of an h0 x w0 source onto its batch canvas (H, W), with the
    reference's own expressions (datasets.py:189-198, 279-296).  With `specific_shape` (--specific-shape: the canvas is the
    (height, width) of every batch) load_image's ratio is min(W / w0, H / h0) and shrink_size is not read.  RuntimeError
    when the loaded size truncates to 0 (cv2.resize raises there) or when the canvas is smaller than the loaded image (the
    letterbox would resize a second time)."""
    h0, w0 = int(h0), int(w0)
    H, W = int(canvas[0]), int(canvas[1])
    if specific_shape:
        ratio = min(W / w0, H / h0)
    else:
        ratio = (img_size - shrink_size) / max(h0, w0) if shrink_size else img_size / max(h0, w0)
    h, w = h0, w0
    if ratio != 1:
        w, h = int(w0 * ratio), int(h0 * ratio)
        if w < 1 or h < 1:
            raise RuntimeError(f"val_geometry: a {h0} x {w0} image loads to {h} x {w} at ratio {ratio} (img_size {img_size}, "
                               f"shrink_size {shrink_size}); cv2.resize refuses an empty size")
    if (h, w) == (h0, w0):
        mode = _lib.VAL_COPY                 # cv::resize copies when the size does not change
    elif ratio > 1:
        mode = _lib.VAL_LINEAR
    else:
        mode = _lib.VAL_AREA_FAST if area_fast(h0, w0, h, w) else _lib.VAL_AREA
    if H < h or W < w:
        raise RuntimeError(f"val_geometry: a {h0} x {w0} image loads to {h} x {w}, larger than its {H} x {W} batch canvas "
                           f"(letterbox would resize it again)")
    r = min(min(H / h, W / w), 1.0)          # data_augment.py:38-40, scaleup=False: 1.0 on this path
    dw, dh = (W - w) / 2, (H - h) / 2
    top, left = int(round(dh - 0.1)), int(round(dw - 0.1))
    shapes = (h0, w0), ((h * r / h0, w * r / w0), (left, top))
    return ValGeometry(mode, h0, w0, h, w, top, left, (H, W), r, shapes)


def val_labels(labels, geo):
    """datasets.py:200-246 for one image: YOLO labels [k, 5] (class, x, y, w, h normalised to the source, float32 as the
    dataset stores them) -> the [k, 6] float32 `labels_out` rows (column 0 left 0 for the collate's image index, then
    class and canvas-normalised x, y, w, h), with the reference's numpy arithmetic and its clip to w - 1e-3."""
    labels = np.array(labels, dtype=np.float32).reshape(-1, 5)
    if labels.size:
        w, h = geo.w * geo.ratio, geo.h * geo.ratio
        pad = (geo.left, geo.top)
        boxes = np.copy(labels[:, 1:])
        boxes[:, 0] = w * (labels[:, 1] - labels[:, 3] / 2) + pad[0]
        boxes[:, 1] = h * (labels[:, 2] - labels[:, 4] / 2) + pad[1]
        boxes[:, 2] = w * (labels[:, 1] + labels[:, 3] / 2) + pad[0]
        boxes[:, 3] = h * (labels[:, 2] + labels[:, 4] / 2) + pad[1]
        labels[:, 1:] = boxes
        h, w = geo.canvas
        labels[:, [1, 3]] = labels[:, [1, 3]].clip(0, w - 1e-3)
        labels[:, [2, 4]] = labels[:, [2, 4]].clip(0, h - 1e-3)
        boxes = np.copy(labels[:, 1:])
        boxes[:, 0] = ((labels[:, 1] + labels[:, 3]) / 2) / w
        boxes[:, 1] = ((labels[:, 2] + labels[:, 4]) / 2) / h
        boxes[:, 2] = (labels[:, 3] - labels[:, 1]) / w
        boxes[:, 3] = (labels[:, 4] - labels[:, 2]) / h
        labels[:, 1:] = boxes
    out = np.zeros((len(labels), 6), dtype=np.float32)
    out[:, 1:] = labels
    return out


def letterbox_val_launch(rec_dev, geo_dev, out, stream=None):
    """yv6_letterbox_val on device tables: rec_dev the B yv6_lb_src records, geo_dev int32 [B, GEO], out uint8 [B, 3, H, W]."""
    B, _, H, W = out.shape
    _lib.check(_lib.lib().yv6_letterbox_val(_lib.handle(out.device.index or 0), C.c_void_p(rec_dev.data_ptr()),
                                            C.c_void_p(geo_dev.data_ptr()), B, H, W, C.c_void_p(out.data_ptr()),
                                            _lib.stream_ptr(stream)))
    return out


class ValFeed:
    """The Evaler's validation batches from decoded frames, on the device.

    Built from every source's (h0, w0) in the dataset's order (`shapes_hw`) with the loader's settings; `batches()` lists
    the source indices of each batch in the order the reference's loader yields them.  `feed(indices, frames, labels)`
    takes 1..batch images of one batch -- cv2 BGR HWC host frames (numpy or CPU tensors) and uint8 CUDA tensors on
    `device`, mixed freely, all in `layout` ("bgr_hwc", or "rgb_chw" as torchvision's decoders return) -- with their YOLO
    labels [k, 5] and returns what the Evaler's loop gets from its DataLoader:
      canvas  uint8 [batch, 3, H, W] on the device (slots after n_real all border 114),
      targets float32 [n, 6] host tensor (image index within the call, class, canvas-normalised x, y, w, h),
      shapes  per image ((h0, w0), ((h / h0, w / w0), (left, top))),
      n_real  the number of images.
    These go unchanged into `PRMetric.update(out[:n], count[:n], targets, shapes, canvas.shape[2:])` and
    `COCOMetric.update`.  Every check (frame type and layout, a frame whose size differs from its entry in shapes_hw,
    indices from two batches, a loaded size of 0, a canvas smaller than the loaded image, more host bytes than
    `max_src_bytes`) raises RuntimeError before anything is written or enqueued.

    Each call stages its tables and host frames (at most `max_src_bytes`, default one 1080p frame per image) through one
    pinned buffer from torch's caching host allocator, which hands a block out again only once its copy has completed;
    the one copy and the one launch go on the current stream, and device frames are read there in place, in stream order.
    `feed` never waits for the device.
    """

    def __init__(self, batch, img_size, stride, shapes_hw, pad=0.5, rect=True, shrink_size=None, max_src_bytes=None, device=None,
                 specific_shape=None):
        self.batch, self.img_size, self.stride, self.shrink_size = int(batch), int(img_size), int(stride), shrink_size
        self.shapes_hw = np.array(shapes_hw, dtype=np.int64).reshape(-1, 2)
        self.order, self.batch_index, self.canvases = val_batches(self.shapes_hw, img_size, batch, stride, pad, rect)
        self.specific_shape = specific_shape is not None
        if self.specific_shape:      # --specific-shape: the order stays as rect sorts it, every canvas is (height, width)
            self.canvases = np.empty_like(self.canvases)
            self.canvases[:] = [int(specific_shape[0]), int(specific_shape[1])]
        self.position = np.empty(len(self.order), dtype=np.int64)
        self.position[self.order] = np.arange(len(self.order))
        self.dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.dev.type != "cuda":
            raise RuntimeError("ValFeed runs on a CUDA device only (no CPU fallback)")
        self.max_src_bytes = int(max_src_bytes) if max_src_bytes else self.batch * DEFAULT_SRC_BYTES

    def batches(self):
        """The source indices of each batch, in the loader's order."""
        return [self.order[self.batch_index == i] for i in range(len(self.canvases))]

    def geometry(self, index):
        """val_geometry of source `index` on its batch's canvas."""
        h0, w0 = self.shapes_hw[index]
        canvas = self.canvases[self.batch_index[self.position[index]]]
        return val_geometry(h0, w0, canvas, self.img_size, self.shrink_size, self.specific_shape)

    def plan(self, indices, srcs):
        """Checks and numbers of one call (nothing written): the batch's canvas and each image's ValGeometry."""
        if len(indices) != len(srcs):
            raise RuntimeError(f"ValFeed: {len(indices)} indices for {len(srcs)} frames")
        idx = [int(i) for i in indices]
        for i in idx:
            if not 0 <= i < len(self.shapes_hw):
                raise RuntimeError(f"ValFeed: index {i} outside the {len(self.shapes_hw)} images")
        b = {int(self.batch_index[self.position[i]]) for i in idx}
        if len(b) != 1:
            raise RuntimeError(f"ValFeed: indices {idx} span batches {sorted(b)}; one call takes images of one batch")
        geos = []
        for i, (_, _, h0, w0, *_) in zip(idx, srcs):
            if (h0, w0) != tuple(int(v) for v in self.shapes_hw[i]):
                raise RuntimeError(f"ValFeed: image {i} is {h0} x {w0}, its entry in shapes_hw says "
                                   f"{self.shapes_hw[i][0]} x {self.shapes_hw[i][1]}")
            geos.append(self.geometry(i))
        return tuple(int(v) for v in self.canvases[b.pop()]), geos

    def feed(self, indices, frames, labels, layout="bgr_hwc"):
        """One batch (see the class): returns (canvas, targets, shapes, n_real)."""
        srcs = check_frames(frames, self.batch, layout, self.dev)
        if len(labels) != len(srcs):
            raise RuntimeError(f"ValFeed: {len(labels)} label arrays for {len(srcs)} frames")
        (H, W), geos = self.plan(indices, srcs)
        used = sum(t.numel() for t, on_dev, *_ in srcs if not on_dev)
        if used > self.max_src_bytes:
            raise RuntimeError(f"ValFeed: the host frames hold {used} bytes, more than max_src_bytes={self.max_src_bytes}")
        targets = []
        for j, (lab, g) in enumerate(zip(labels, geos)):
            t = val_labels(lab, g)
            t[:, 0] = j
            targets.append(t)
        targets = torch.from_numpy(np.concatenate(targets, 0))
        # one pinned staging buffer: the B records, the B geometry rows, then the host frames back to back
        head = self.batch * (REC + GEO * 4)
        host = torch.empty(head + used, dtype=torch.uint8, pin_memory=True)
        dev = torch.empty(head + used, dtype=torch.uint8, device=self.dev)
        recs = (_lib.LbSrc * self.batch)()
        rows, off = [], head
        for j, ((t, on_dev, h0, w0, row_pitch, plane_pitch), g) in enumerate(zip(srcs, geos)):
            if on_dev:
                base = t.data_ptr()
            else:
                host[off:off + t.numel()].copy_(t.view(-1))
                base = dev.data_ptr() + off
                off += t.numel()
            recs[j] = _lib.LbSrc(base, row_pitch, plane_pitch, LAYOUTS[layout], 0)
            rows.append(g.row())
        rows += [[0, H, W, 0, 0, 0, 0, 0]] * (self.batch - len(srcs))      # all border, reads nothing
        C.memmove(host.data_ptr(), recs, C.sizeof(recs))
        host[self.batch * REC:head].view(torch.int32).copy_(torch.tensor(rows, dtype=torch.int32).view(-1))
        with torch.cuda.device(self.dev):
            dev.copy_(host, non_blocking=True)      # the pinned block is reused only after this copy (torch's host allocator)
            canvas = torch.empty(self.batch, 3, H, W, dtype=torch.uint8, device=self.dev)
            letterbox_val_launch(dev[:self.batch * REC], dev[self.batch * REC:head], canvas)
        return canvas, targets, [g.shapes for g in geos], len(srcs)
