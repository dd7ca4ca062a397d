"""Decoded frames in, source-pixel boxes out: the two steps of the reference's Inferer around the model.

`Inferer.process_image` (core/inferer.py:161-171) letterboxes each image on the host with cv2 (data/data_augment.py:29-58)
and `Inferer.rescale` (:173-188) maps the boxes back.  Here both run on the device for a whole batch per launch
(`yv6_letterbox_frames`, `yv6_rescale_boxes`): images of any size -- OpenCV `imread` layout, uint8 HWC BGR, or the RGB CHW
of torchvision's decoders -- are read where they lie: host images are packed back to back in one staging buffer, CUDA
tensors in place.  A per-image record table says where each image is and in which layout, and a per-image int32 table
carries the geometry the host computed with the reference's Python expressions.  Because both are data, a CUDA graph that
contains these kernels serves any mix of image sizes, layouts and locations.

Both of the reference's padding modes are provided.  auto=False pads every image to the full H x W canvas (the Evaler's
and a fixed-shape server's choice).  auto=True is Inferer's own default: the image is padded only up to the next multiple
of the stride, so a 1920 x 1080 frame at img_size 640 reaches the network as a 384 x 640 canvas.  Each source shape then
has its own canvas (`rect_canvas`); a batch takes one canvas, so frames whose canvases differ are refused before anything
is staged, and a caller serving mixed sources keeps one batch per canvas.  JPEGs are decoded on the device, with
cv2.imread's pixels, by `jpeg.JpegDecoder`, whose frames and `ready` event go straight into `DetectStream.submit`; other
formats, and the JPEG kinds it refuses, are decoded by the caller.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib

GEO = 8      # int32 per image in the geometry table: src_off, h0, w0, nh, nw, top, left, 0 (YV6_LB_GEO)


def inferer_stride(strides):
    """The stride Inferer pads and rounds img_size to: DetectBackend's max(model stride, 32) -- 32 for the P5 detectors,
    64 for the P6 and Lite ones."""
    return max(max(int(s) for s in strides), 32)


def inferer_size(img_size, stride):
    """Inferer.check_img_size: img_size (an int or (H, W)) with each side rounded up to a multiple of `stride`, as (H, W)."""
    H, W = (img_size, img_size) if isinstance(img_size, int) else img_size
    return math.ceil(H / stride) * stride, math.ceil(W / stride) * stride


def _resize_and_pad(h0, w0, H, W, scaleup, auto, stride):
    """data_augment.py:38-49: (r, (nw, nh), (dw, dh)), the total padding before it is split between the two sides."""
    r = min(H / h0, W / w0)
    if not scaleup:
        r = min(r, 1.0)
    nw, nh = int(round(w0 * r)), int(round(h0 * r))
    dw, dh = W - nw, H - nh
    if auto:                     # minimum rectangle: np.mod(dw, stride); dw >= 0, so Python's % is the same
        dw, dh = dw % stride, dh % stride
    return r, (nw, nh), (dw, dh)


def letterbox_geometry(h0, w0, H, W, scaleup=True, auto=False, stride=32):
    """The reference's letterbox numbers for an h0 x w0 image and new_shape (H, W) (data_augment.py:38-55):
    (r, (nw, nh), top, left), new_unpad = (nw, nh) rounded half to even as Python's round() does.  auto=False pads to the
    full H x W canvas, auto=True only up to the next multiple of `stride` (the canvas is `rect_canvas`)."""
    r, (nw, nh), (dw, dh) = _resize_and_pad(h0, w0, H, W, scaleup, auto, stride)
    return r, (nw, nh), int(round(dh / 2 - 0.1)), int(round(dw / 2 - 0.1))


def rect_canvas(h0, w0, img_size, stride, scaleup=True):
    """The canvas (H, W) Inferer.process_image(im, img_size, stride, half) gives an h0 x w0 image: letterbox with auto=True
    on img_size rounded up to the stride (`inferer_size`), i.e. (nh + dh, nw + dw) -- a multiple of `stride` on both sides.
    1080 x 1920 at 640 / stride 32 -> (384, 640); at 320 / stride 64 -> (192, 320)."""
    H, W = inferer_size(img_size, stride)
    _, (nw, nh), (dw, dh) = _resize_and_pad(h0, w0, H, W, scaleup, True, stride)
    return nh + dh, nw + dw


def common_canvas(srcs, H, W, scaleup, stride):
    """The rect canvas (`rect_canvas`) shared by checked frames (`check_frames`) at img_size (H, W); RuntimeError naming
    both shapes when two frames' canvases differ (one batch has one canvas)."""
    canvas = first = None
    for _, _, h0, w0, *_ in srcs:
        c = rect_canvas(h0, w0, (H, W), stride, scaleup)
        if canvas is None:
            canvas, first = c, (h0, w0)
        elif c != canvas:
            raise RuntimeError(f"letterbox: a {h0} x {w0} frame letterboxes to a {c[0]} x {c[1]} canvas, a {first[0]} x {first[1]} "
                               f"frame of the same batch to {canvas[0]} x {canvas[1]} (auto=True: one canvas per batch)")
    return canvas


class LetterboxMeta:
    """Per-image metadata of a letterboxed batch.
    geo: int32 [B, GEO] host table (the device copy is what the kernels read); n: number of real images (slots beyond n are
    all border); shapes: Evaler's `(h0, w0), ((h0 * r / h0, w0 * r / w0), (left, top))` per image (datasets.py:198), which
    `evalpost.convert_to_coco_format` takes as is."""

    def __init__(self, geo, n, H, W, shapes, geo_dev=None):
        self.geo, self.n, self.H, self.W, self.shapes, self.geo_dev = geo, n, H, W, shapes, geo_dev


LAYOUTS = {"bgr_hwc": _lib.LB_BGR_HWC, "rgb_chw": _lib.LB_RGB_CHW}
REC = C.sizeof(_lib.LbSrc)    # bytes per image in the yv6_lb_src record table


def source_pitches(shape, strides, layout):
    """(h0, w0, row_pitch, plane_pitch) of a uint8 frame with these sizes and element strides in `layout` ("bgr_hwc":
    [h0, w0, 3], pixel stride 3; "rgb_chw": [3, h0, w0]); RuntimeError when yv6_letterbox_frames cannot address it."""
    if layout not in LAYOUTS:
        raise RuntimeError(f"letterbox: layout must be one of {sorted(LAYOUTS)}, got {layout!r}")
    hwc = layout == "bgr_hwc"
    if len(shape) != 3 or shape[2 if hwc else 0] != 3:
        raise RuntimeError(f"letterbox: {layout} frames must be {'HWC with 3 channels last' if hwc else 'CHW with 3 channels first'}, "
                           f"got shape {tuple(shape)}")
    h0, w0 = (shape[0], shape[1]) if hwc else (shape[1], shape[2])
    if h0 < 1 or w0 < 1:
        raise RuntimeError(f"letterbox: empty frame, shape {tuple(shape)}")
    if strides[2] != 1:
        raise RuntimeError(f"letterbox: the unit-stride axis of a {layout} frame must be the innermost one, got strides {tuple(strides)}")
    if hwc and strides[1] != 3:
        raise RuntimeError(f"letterbox: a bgr_hwc frame needs a pixel stride of 3 bytes, got strides {tuple(strides)}")
    return int(h0), int(w0), int(strides[0] if hwc else strides[1]), 0 if hwc else int(strides[0])


def check_frame(im, layout, dev):
    """Validate one frame in `layout`; nothing is copied or enqueued.  A frame is a host numpy array or CPU tensor (staged:
    returned as a contiguous CPU tensor) or a uint8 tensor on `dev` (read in place).  Returns (tensor, on_device, h0, w0,
    row_pitch, plane_pitch); RuntimeError when the frame is unusable."""
    t = torch.from_numpy(np.ascontiguousarray(im)) if isinstance(im, np.ndarray) else im
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"letterbox: frames must be numpy arrays or tensors, got {type(im).__name__}")
    on_dev = t.device.type != "cpu"
    if on_dev and t.device != dev:
        raise RuntimeError(f"letterbox: a frame on {t.device}, the pipeline runs on {dev}")
    if t.dtype != torch.uint8:
        raise RuntimeError(f"letterbox: frames must be uint8, got {t.dtype}")
    if not on_dev:
        t = t.contiguous()
    return (t, on_dev) + source_pitches(tuple(t.shape), t.stride(), layout)


def check_frames(frames, B, layout, dev):
    """Validate 1..B frames for one letterbox launch (`check_frame` each); nothing is copied or enqueued.  Returns one
    (tensor, on_device, h0, w0, row_pitch, plane_pitch) per frame; RuntimeError when any frame is unusable."""
    if not 1 <= len(frames) <= B:
        raise RuntimeError(f"letterbox: {len(frames)} frames for a batch of {B}")
    return [check_frame(im, layout, dev) for im in frames]


def pack_sources(srcs, B, H, W, scaleup, layout, src_host, geo_host, rec_host, src_dev_ptr, auto=False, stride=32, canvas=None):
    """Lay out checked frames (`check_frames`) for yv6_letterbox_frames: copy the host frames back to back into `src_host`
    (the device buffer at `src_dev_ptr` receives these bytes before the launch), fill the geometry table `geo_host` [B, GEO]
    and the record table `rec_host` (B * REC bytes).  A device frame's record points at the frame itself.  (H, W) is the
    letterbox's new_shape; `canvas`, the shape of the device canvas, is (H, W) when not given.  With auto=True every frame's
    `rect_canvas` must equal `canvas`.  Raises RuntimeError before anything is written when a frame's canvas differs or
    the host frames exceed `src_host`.
    Returns (host bytes used, shapes, the device frames)."""
    canvas = tuple(canvas or (H, W))
    if auto:
        got = common_canvas(srcs, H, W, scaleup, stride)
        if got != canvas:
            h0, w0 = srcs[0][2:4]
            raise RuntimeError(f"letterbox: a {h0} x {w0} frame letterboxes to a {got[0]} x {got[1]} canvas at img_size {H} x {W}, "
                               f"stride {stride}; this batch's canvas is {canvas[0]} x {canvas[1]}")
    used = sum(t.numel() for t, on_dev, *_ in srcs if not on_dev)
    if used > src_host.numel():
        raise RuntimeError(f"letterbox: the host frames hold {used} bytes, the staging buffer {src_host.numel()} (raise max_src_bytes)")
    recs = (_lib.LbSrc * B)()
    rows, shapes, devs, off = [], [], [], 0
    for i, (t, on_dev, h0, w0, row_pitch, plane_pitch) in enumerate(srcs):
        r, (nw, nh), top, left = letterbox_geometry(h0, w0, H, W, scaleup, auto, stride)
        if on_dev:
            base, src_off = t.data_ptr(), 0
            devs.append(t)
        else:
            src_host[off:off + t.numel()].copy_(t.view(-1))
            base, src_off = src_dev_ptr + off, off
            off += t.numel()
        recs[i] = _lib.LbSrc(base, row_pitch, plane_pitch, LAYOUTS[layout], 0)
        rows.append([src_off, h0, w0, nh, nw, top, left, 0])
        shapes.append(((h0, w0), ((h0 * r / h0, w0 * r / w0), (left, top))))
    rows += [[0, canvas[0], canvas[1], 0, 0, 0, 0, 0]] * (B - len(srcs))     # unused slots: all border, rescale well defined
    geo_host.copy_(torch.tensor(rows, dtype=torch.int32))
    C.memmove(rec_host.data_ptr(), recs, C.sizeof(recs))
    return used, shapes, devs


def pack_frames(frames, B, H, W, scaleup, src_host, geo_host):
    """Validate host frames (uint8 HWC BGR), copy their bytes back to back into the pinned `src_host` and fill `geo_host`
    [B, GEO].  Raises RuntimeError before anything is written when a frame is malformed or the bytes exceed the buffer.
    Returns (bytes used, shapes)."""
    srcs = check_frames(frames, B, "bgr_hwc", torch.device("cpu"))
    used, shapes, _ = pack_sources(srcs, B, H, W, scaleup, "bgr_hwc", src_host, geo_host, torch.empty(B * REC, dtype=torch.uint8), 0)
    return used, shapes


def letterbox_frames_launch(rec_dev, geo_dev, out, stream=None):
    """yv6_letterbox_frames on device tables: rec_dev the B yv6_lb_src records, geo_dev int32 [B, GEO], out uint8 [B, 3, H, W]."""
    B, _, H, W = out.shape
    _lib.check(_lib.lib().yv6_letterbox_frames(_lib.handle(out.device.index or 0), C.c_void_p(rec_dev.data_ptr()),
                                               C.c_void_p(geo_dev.data_ptr()), B, H, W, C.c_void_p(out.data_ptr()), _lib.stream_ptr(stream)))
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


def letterbox_batch(images, H, W, scaleup=True, out=None, device=None, layout="bgr_hwc", auto=False, stride=32):
    """Letterbox a list of uint8 frames of any sizes onto the uint8 NCHW RGB canvas [B, 3, H, W] on the device --
    letterbox(im, (H, W), auto=False, scaleup) + HWC->CHW + BGR->RGB of Inferer.process_image, bit-exact against cv2.
    Each frame is a host numpy array or CPU tensor (staged through pinned memory) or a CUDA tensor on the canvas's device
    (read in place, in stream order after the work already on the current stream).  `layout` applies to every frame:
    "bgr_hwc" is cv2 imread's [h0, w0, 3] (rows may be padded, e.g. a crop view), "rgb_chw" torchvision's decoders'
    [3, h0, w0]; both give the canvas of the equivalent BGR HWC image.  `scaleup=True` is Inferer's setting, False the
    Evaler dataset's.  auto=True is Inferer.process_image(im, (H, W), stride, half) itself: (H, W) is img_size (rounded up
    to the stride) and the canvas is the frames' common `rect_canvas`; frames with different canvases raise RuntimeError
    before anything is staged.  Returns (canvas, LetterboxMeta).  `out` (uint8 [B, 3, h, w] CUDA tensor on that canvas,
    B >= len(images)) is filled in place."""
    dev = out.device if out is not None else device or torch.device("cuda", torch.cuda.current_device())
    if auto:
        H, W = inferer_size((H, W), stride)
    srcs = check_frames(images, out.shape[0] if out is not None else len(images), layout, dev)
    canvas = common_canvas(srcs, H, W, scaleup, stride) if auto else (H, W)
    if out is None:
        out = torch.empty(len(images), 3, *canvas, dtype=torch.uint8, device=dev)
    if out.device.type != "cuda" or out.dtype != torch.uint8 or tuple(out.shape[1:]) != (3, *canvas):
        raise RuntimeError("letterbox_batch: out must be a uint8 CUDA tensor [B, 3, H, W]")
    B = out.shape[0]
    nbytes = max(1, sum(t.numel() for t, on_dev, *_ in srcs if not on_dev))
    src_host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    geo_host = torch.empty(B, GEO, dtype=torch.int32).pin_memory()
    rec_host = torch.empty(B * REC, dtype=torch.uint8).pin_memory()
    src_dev = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
    _, shapes, _ = pack_sources(srcs, B, H, W, scaleup, layout, src_host, geo_host, rec_host, src_dev.data_ptr(), auto, stride,
                                canvas)
    src_dev.copy_(src_host, non_blocking=True)
    geo_dev = geo_host.to(out.device, non_blocking=True)
    rec_dev = rec_host.to(out.device, non_blocking=True)
    letterbox_frames_launch(rec_dev, geo_dev, out)
    torch.cuda.current_stream(out.device).synchronize()      # the pinned staging buffers die with this call
    return out, LetterboxMeta(geo_host.clone(), len(images), canvas[0], canvas[1], shapes, geo_dev)


def rescale_boxes(out, count, meta):
    """Inferer.rescale(...) followed by .round() (inferer.py:103, 173-188) for every image of a batch: the NMS output
    out [B, max_det, 6] / count [B] of a letterboxed batch -> [B, max_det, 6] (x1, y1, x2, y2 in source pixels, conf, cls),
    rows beyond count zeroed.  Stays on the device, no host synchronisation."""
    if out.device.type != "cuda":
        raise RuntimeError("yolov6_b200.preprocess runs on CUDA tensors only (no CPU fallback)")
    geo = meta.geo_dev if meta.geo_dev is not None and meta.geo_dev.device == out.device else meta.geo.to(out.device)
    return rescale_launch(out.contiguous().float(), count.to(torch.int32).contiguous(), geo, meta.H, meta.W)
