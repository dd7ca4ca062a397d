"""oracle/letterbox.py -- numpy restatement of the letterbox / rescale kernels (TEST INFRASTRUCTURE ONLY).

`resize_linear` states the sampling rule of yolov6_b200/csrc/yv6_letterbox.cu, which is OpenCV's uint8 INTER_LINEAR
cv2.resize: double-precision source coordinate, 11-bit coefficients, horizontal border taps clamped with a zero
fraction, vertical rows clamped with the unreset fraction, and the truncating vertical pass of OpenCV's SIMD kernel.
`letterbox` and `rescale` follow the reference's data_augment.letterbox (auto=False) + Inferer.process_image and
Inferer.rescale(...).round(); tests/golden/make_golden_letterbox.py pins all three against the live reference and cv2.
"""
import numpy as np
import torch


def geometry(h0, w0, H, W, scaleup=True):
    """data_augment.py:38-55 with auto=False: (r, (nw, nh), top, left)."""
    r = min(H / h0, W / w0)
    if not scaleup:
        r = min(r, 1.0)
    nw, nh = int(round(w0 * r)), int(round(h0 * r))
    dw, dh = (W - nw) / 2, (H - nh) / 2
    return r, (nw, nh), int(round(dh - 0.1)), int(round(dw - 0.1))


def _taps(src, dst, reset_border):
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    fr = (f - s.astype(np.float32)).astype(np.float32)
    if reset_border:
        lo, hi = s < 0, s >= src - 1
        fr = np.where(lo | hi, np.float32(0), fr)
        s = np.where(lo, 0, np.where(hi, src - 1, s))
    c0 = np.rint((np.float32(1) - fr) * np.float32(2048)).astype(np.int64)
    c1 = np.rint(fr * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), c0, c1


def resize_linear(im, nw, nh):
    """cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR) for uint8 HWC images."""
    h0, w0 = im.shape[:2]
    x0, x1, a0, a1 = _taps(w0, nw, True)
    y0, y1, b0, b1 = _taps(h0, nh, False)
    src = im.astype(np.int64)
    S = src[:, x0, :] * a0[None, :, None] + src[:, x1, :] * a1[None, :, None]        # [h0, nw, c]
    t = (((b0[:, None, None] * (S[y0] >> 4)) >> 16) + ((b1[:, None, None] * (S[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(t, 0, 255).astype(np.uint8)


def letterbox(im, H, W, scaleup=True):
    """letterbox(im, (H, W), auto=False, scaleup) + HWC->CHW + BGR->RGB (Inferer.process_image without the /255):
    uint8 [3, H, W]."""
    h0, w0 = im.shape[:2]
    _, (nw, nh), top, left = geometry(h0, w0, H, W, scaleup)
    body = im if (nw, nh) == (w0, h0) else resize_linear(im, nw, nh)
    out = np.full((H, W, 3), 114, np.uint8)
    out[top:top + nh, left:left + nw] = body
    return np.ascontiguousarray(out.transpose(2, 0, 1)[::-1])


def rescale(det, H, W, h0, w0):
    """Inferer.rescale((H, W), det[:, :4], (h0, w0)).round() in torch fp32 on the CPU; det [k, 6] float32."""
    b = torch.as_tensor(det, dtype=torch.float32).clone()
    ratio = min(H / h0, W / w0)
    padding = (W - w0 * ratio) / 2, (H - h0 * ratio) / 2
    boxes = b[:, :4]
    boxes[:, [0, 2]] -= padding[0]
    boxes[:, [1, 3]] -= padding[1]
    boxes[:, :4] /= ratio
    boxes[:, 0].clamp_(0, w0)
    boxes[:, 1].clamp_(0, h0)
    boxes[:, 2].clamp_(0, w0)
    boxes[:, 3].clamp_(0, h0)
    b[:, :4] = boxes.round()
    return b.numpy()


def synthetic_source(h0, w0, kind, seed):
    """Seeded uint8 HWC BGR test image: 'noise' (uniform bytes) or 'grad' (smooth ramps that expose coefficient errors)."""
    rng = np.random.default_rng(7000 + seed)
    if kind == "noise":
        return rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
    y = np.linspace(0, 1, h0)[:, None]
    x = np.linspace(0, 1, w0)[None, :]
    ph = rng.uniform(0, 1, 3)
    chans = [(255 * (0.5 + 0.5 * np.sin(2 * np.pi * (x * (1 + 2 * c) + y * (2 - c) + ph[c])))) for c in range(3)]
    return np.ascontiguousarray(np.stack(chans, -1).round().clip(0, 255).astype(np.uint8))


# (h0, w0, H, W, scaleup, kind): downscale, upscale, exact fit, odd sizes, extreme aspect ratios, 1x1 / 2x2, scaleup=False,
# noise and gradients; mostly small canvases, a few at 640.
CASES = [
    (138, 302, 320, 640, True, "noise"), (138, 302, 320, 640, True, "grad"),
    (1080, 1920, 192, 320, True, "grad"), (480, 640, 64, 64, True, "noise"),
    (320, 320, 320, 320, True, "noise"), (200, 320, 320, 320, True, "grad"),
    (333, 999, 128, 320, True, "noise"), (101, 77, 160, 128, True, "grad"),
    (17, 1000, 320, 320, True, "noise"), (1000, 17, 320, 320, True, "grad"),
    (1, 1, 64, 64, True, "noise"), (2, 2, 64, 64, True, "grad"), (2, 2, 64, 96, True, "noise"),
    (50, 100, 320, 320, True, "noise"), (3, 5, 192, 320, True, "grad"),
    (123, 457, 320, 320, False, "noise"), (900, 450, 320, 320, False, "grad"), (63, 31, 128, 64, False, "noise"),
    (640, 1280, 640, 640, True, "grad"), (360, 480, 640, 640, True, "noise"), (720, 1280, 640, 640, True, "grad"),
]


def synthetic_detections(H, W, seed, n=40):
    """Seeded NMS-like rows [n, 6] on an H x W canvas: boxes inside, on and beyond the borders, coordinates on quarter-pixel
    grid points (after rescaling, many of them land exactly on .5)."""
    rng = np.random.default_rng(9000 + seed)
    xy = rng.integers(-40, max(W, H) + 40, (n, 2)) + rng.integers(0, 4, (n, 2)) * 0.25
    wh = rng.integers(1, 200, (n, 2)) + rng.integers(0, 4, (n, 2)) * 0.25
    xy[:4] = [[0, 0], [-3.5, -0.5], [W - 0.5, H - 0.5], [W, H]]
    conf = rng.uniform(0.25, 1, (n, 1))
    cls = rng.integers(0, 80, (n, 1))
    return np.concatenate([xy, xy + wh, conf, cls], 1).astype(np.float32)


# (h0, w0, H, W): ratio 1, 2 and 1/2 (exact .5 rounding points), non-dyadic ratios, padding on either axis.
RESCALE_CASES = [(640, 640, 640, 640), (320, 320, 640, 640), (1280, 960, 640, 640), (1080, 1920, 640, 640), (138, 302, 320, 640),
                 (17, 1000, 320, 320), (1000, 17, 320, 320), (1, 1, 64, 64), (333, 999, 128, 320)]
