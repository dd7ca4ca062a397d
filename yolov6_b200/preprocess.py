"""Decoded frames in, source-pixel boxes out: the two steps of the reference's Inferer around the model.

`Inferer.process_image` (core/inferer.py:161-171) letterboxes each image on the host with cv2 (data/data_augment.py:29-58)
and `Inferer.rescale` (:173-188) maps the boxes back.  Here both run on the device for a whole batch per launch
(`yv6_letterbox`, `yv6_rescale_boxes`): images of any size -- OpenCV `imread` layout, uint8 HWC BGR -- are packed back to
back in one byte buffer, and a per-image int32 table carries the geometry the host computed with the reference's Python
expressions.  Because the geometry is data, a CUDA graph that contains these kernels serves any mix of image sizes.

Only letterbox(..., auto=False) is provided: it pads every image to the full H x W canvas, so a batch has one shape.
Inferer's own default, auto=True, pads to a stride multiple and gives each image its own shape; that does not fit a
fixed-shape batch.  Decoding (JPEG / PNG -> pixels) stays with the caller.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

GEO = 8      # int32 per image in the geometry table: src_off, h0, w0, nh, nw, top, left, 0 (YV6_LB_GEO)


def letterbox_geometry(h0, w0, H, W, scaleup=True):
    """The reference's letterbox numbers for an h0 x w0 image on an H x W canvas (data_augment.py:38-55, auto=False):
    (r, (nw, nh), top, left), new_unpad = (nw, nh) rounded half to even as Python's round() does."""
    r = min(H / h0, W / w0)
    if not scaleup:
        r = min(r, 1.0)
    nw, nh = int(round(w0 * r)), int(round(h0 * r))
    dw, dh = (W - nw) / 2, (H - nh) / 2
    return r, (nw, nh), int(round(dh - 0.1)), int(round(dw - 0.1))


def as_frame(im):
    """uint8 HWC 3-channel host image (numpy array or CPU tensor) -> contiguous uint8 CPU tensor; RuntimeError otherwise."""
    t = torch.from_numpy(np.ascontiguousarray(im)) if isinstance(im, np.ndarray) else im
    if not isinstance(t, torch.Tensor) or t.device.type != "cpu":
        raise RuntimeError(f"letterbox: frames must be host numpy arrays or CPU tensors, got {type(im).__name__}")
    if t.dtype != torch.uint8:
        raise RuntimeError(f"letterbox: frames must be uint8, got {t.dtype}")
    if t.dim() != 3 or t.shape[2] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
        raise RuntimeError(f"letterbox: frames must be HWC with 3 channels (BGR), got shape {tuple(t.shape)}")
    return t.contiguous()


class LetterboxMeta:
    """Per-image metadata of a letterboxed batch.
    geo: int32 [B, GEO] host table (the device copy is what the kernels read); n: number of real images (slots beyond n are
    all border); shapes: Evaler's `(h0, w0), ((h0 * r / h0, w0 * r / w0), (left, top))` per image (datasets.py:198), which
    `evalpost.convert_to_coco_format` takes as is."""

    def __init__(self, geo, n, H, W, shapes, geo_dev=None):
        self.geo, self.n, self.H, self.W, self.shapes, self.geo_dev = geo, n, H, W, shapes, geo_dev


def pack_frames(frames, B, H, W, scaleup, src_host, geo_host):
    """Validate `frames`, copy their bytes back to back into the pinned `src_host` and fill `geo_host` [B, GEO].
    Raises RuntimeError before anything is written when a frame is malformed or the bytes exceed the buffer.
    Returns (bytes used, shapes)."""
    frames = [as_frame(f) for f in frames]
    if not 1 <= len(frames) <= B:
        raise RuntimeError(f"letterbox: {len(frames)} frames for a batch of {B}")
    used = sum(f.numel() for f in frames)
    if used > src_host.numel():
        raise RuntimeError(f"letterbox: the frames hold {used} bytes, the staging buffer {src_host.numel()} (raise max_src_bytes)")
    rows, shapes, off = [], [], 0
    for f in frames:
        h0, w0 = int(f.shape[0]), int(f.shape[1])
        r, (nw, nh), top, left = letterbox_geometry(h0, w0, H, W, scaleup)
        src_host[off:off + f.numel()].copy_(f.view(-1))
        rows.append([off, h0, w0, nh, nw, top, left, 0])
        shapes.append(((h0, w0), ((h0 * r / h0, w0 * r / w0), (left, top))))
        off += f.numel()
    rows += [[0, H, W, 0, 0, 0, 0, 0]] * (B - len(frames))         # unused slots: all border, rescale well defined
    geo_host.copy_(torch.tensor(rows, dtype=torch.int32))
    return used, shapes


def letterbox_launch(src_dev, geo_dev, out, stream=None):
    """yv6_letterbox on device buffers: src_dev packed uint8 sources, geo_dev int32 [B, GEO], out uint8 [B, 3, H, W]."""
    B, _, H, W = out.shape
    _lib.check(_lib.lib().yv6_letterbox(_lib.handle(out.device.index or 0), C.c_void_p(src_dev.data_ptr()), C.c_void_p(geo_dev.data_ptr()),
                                        B, H, W, C.c_void_p(out.data_ptr()), _lib.stream_ptr(stream)))
    return out


def rescale_launch(out, count, geo_dev, H, W, res=None, stream=None):
    """yv6_rescale_boxes: NMS output out [B, max_det, 6] / count [B] -> res [B, max_det, 6] in source pixels (rows beyond
    count zeroed)."""
    B, max_det, _ = out.shape
    res = torch.empty_like(out) if res is None else res
    _lib.check(_lib.lib().yv6_rescale_boxes(_lib.handle(out.device.index or 0), C.c_void_p(out.data_ptr()), C.c_void_p(count.data_ptr()),
                                            C.c_void_p(geo_dev.data_ptr()), B, max_det, H, W, C.c_void_p(res.data_ptr()),
                                            _lib.stream_ptr(stream)))
    return res


def letterbox_batch(images, H, W, scaleup=True, out=None, device=None):
    """Letterbox a list of uint8 HWC BGR host images (numpy arrays or CPU tensors, any sizes) onto the uint8 NCHW RGB
    canvas [B, 3, H, W] on the device -- letterbox(im, (H, W), auto=False, scaleup) + HWC->CHW + BGR->RGB of
    Inferer.process_image, bit-exact against cv2.  `scaleup=True` is Inferer's setting, False the Evaler dataset's.
    Returns (canvas, LetterboxMeta).  `out` (uint8 [B, 3, H, W] CUDA tensor, B >= len(images)) is filled in place."""
    if out is None:
        out = torch.empty(len(images), 3, H, W, dtype=torch.uint8, device=device or torch.device("cuda", torch.cuda.current_device()))
    if out.device.type != "cuda" or out.dtype != torch.uint8 or tuple(out.shape[1:]) != (3, H, W):
        raise RuntimeError("letterbox_batch: out must be a uint8 CUDA tensor [B, 3, H, W]")
    B = out.shape[0]
    frames = [as_frame(f) for f in images]
    src_host = torch.empty(max(1, sum(f.numel() for f in frames)), dtype=torch.uint8).pin_memory()
    geo_host = torch.empty(B, GEO, dtype=torch.int32).pin_memory()
    used, shapes = pack_frames(frames, B, H, W, scaleup, src_host, geo_host)
    src_dev = src_host.to(out.device, non_blocking=True)
    geo_dev = geo_host.to(out.device, non_blocking=True)
    letterbox_launch(src_dev, geo_dev, out)
    torch.cuda.current_stream(out.device).synchronize()      # the pinned staging buffers die with this call
    return out, LetterboxMeta(geo_host.clone(), len(frames), H, W, shapes, geo_dev)


def rescale_boxes(out, count, meta):
    """Inferer.rescale(...) followed by .round() (inferer.py:103, 173-188) for every image of a batch: the NMS output
    out [B, max_det, 6] / count [B] of a letterboxed batch -> [B, max_det, 6] (x1, y1, x2, y2 in source pixels, conf, cls),
    rows beyond count zeroed.  Stays on the device, no host synchronisation."""
    if out.device.type != "cuda":
        raise RuntimeError("yolov6_b200.preprocess runs on CUDA tensors only (no CPU fallback)")
    geo = meta.geo_dev if meta.geo_dev is not None and meta.geo_dev.device == out.device else meta.geo.to(out.device)
    return rescale_launch(out.contiguous().float(), count.to(torch.int32).contiguous(), geo, meta.H, meta.W)
