"""oracle/augment.py -- numpy restatement of the training augmentation kernels (TEST INFRASTRUCTURE ONLY; no cv2).

States the pixel rules of yolov6_b200/csrc/yv6_augment.cu, which are OpenCV's uint8 paths as the reference's
TrainValDataset.__getitem__ (yolov6/data/datasets.py:166-255) calls them:
  - `warp_affine`: cv2.warpAffine(img, M[:2], (W, H), INTER_LINEAR, BORDER_CONSTANT 114): M inverted in double, 10-bit
    fixed-point coordinates rounded to 5-bit fractions, the 32 x 32 bilinear table (every entry an exact integer, so its
    sum is 32768 without correction), (sum + 2^14) >> 15, an out-of-image tap reads 114;
  - `bgr_to_hsv` / `hsv_to_bgr`: cv2.cvtColor BGR2HSV (12-bit fixed point) and HSV2BGR (float32 with fused
    multiply-adds and a truncating store, as OpenCV's AVX2 kernel computes it);
  - `compose`: mosaic / letterbox canvas, affine, mixup, HSV, flips and HWC BGR -> CHW RGB for one sampler record, on top
    of oracle.letterbox.resize_linear.
tests/golden/make_golden_augment.py pins these against the live reference and cv2.
"""
import numpy as np

from oracle.letterbox import resize_linear

_F = np.float32


def warp_affine(img, M, W, H, border=114):
    """cv2.warpAffine(img, M[:2], dsize=(W, H), borderValue=(114,) * 3) for uint8 HWC images, M the forward 3x3 matrix."""
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
    x = np.arange(W, dtype=np.float64)
    y = np.arange(H, dtype=np.float64)
    adelta = np.rint(m[0] * x * 1024).astype(np.int64)
    bdelta = np.rint(m[3] * x * 1024).astype(np.int64)
    X0 = np.rint((m[1] * y + m[2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((m[4] * y + m[5]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, fx, sy, fy = X >> 5, X & 31, Y >> 5, Y & 31
    h0, w0 = img.shape[:2]
    src = img.astype(np.int64)

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < h0) & (xx >= 0) & (xx < w0)
        v = src[np.clip(yy, 0, h0 - 1), np.clip(xx, 0, w0 - 1)]
        return np.where(ok[..., None], v, border)

    w00 = ((32 - fx) * (32 - fy) * 32)[..., None]
    w01 = (fx * (32 - fy) * 32)[..., None]
    w10 = ((32 - fx) * fy * 32)[..., None]
    w11 = (fx * fy * 32)[..., None]
    acc = tap(sy, sx) * w00 + tap(sy, sx + 1) * w01 + tap(sy + 1, sx) * w10 + tap(sy + 1, sx + 1) * w11
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def _div_tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, np.rint((255 << 12) / i), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.rint((180 << 12) / (6.0 * i)), 0).astype(np.int64)
    return sdiv, hdiv


SDIV, HDIV = _div_tables()


def bgr_to_hsv(img):
    """cv2.cvtColor(img, COLOR_BGR2HSV) for uint8 [..., 3] BGR (hue in [0, 180))."""
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * SDIV[v] + (1 << 11)) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * HDIV[diff] + (1 << 11)) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def _fma(a, b, c):
    """float32 fused multiply-add: the float64 product of two float32 values is exact."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(_F)


_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hsv_to_bgr(hsv):
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) for uint8 [..., 3] HSV with hue < 180, as OpenCV's AVX2 kernel computes it: s and
    v scaled by 1/255f, h by 6/180f, sector = trunc(h), tab2 = v * fma(-s, f, 1), tab3 = v * fma(-s, 1 - f, 1), times 255f,
    truncated."""
    h = hsv[..., 0].astype(_F) * _F(6.0 / 180.0)
    s = hsv[..., 1].astype(_F) * _F(1.0 / 255.0)
    v = hsv[..., 2].astype(_F) * _F(1.0 / 255.0)
    pre = np.trunc(h)
    f = (h - pre).astype(_F)
    sector = pre.astype(np.int64) % 6
    one = np.ones_like(f)
    tab = np.stack([v, v * (one - s), v * _fma(-s, f, one), v * _fma(-s, (one - f).astype(_F), one)], -1)
    out = np.take_along_axis(tab, _SECTOR[sector], -1) * _F(255.0)
    return np.trunc(out).astype(np.uint8)


def hsv_luts(gains):
    """augment_hsv's three lookup tables (data_augment.py:20-23) for the drawn gains r (float64 [3])."""
    x = np.arange(0, 256, dtype=np.float64)
    return (((x * gains[0]) % 180).astype(np.uint8), np.clip(x * gains[1], 0, 255).astype(np.uint8),
            np.clip(x * gains[2], 0, 255).astype(np.uint8))


def augment_hsv(img, gains):
    """augment_hsv(img) with the drawn gains: BGR -> HSV -> three LUTs -> BGR."""
    lh, ls, lv = hsv_luts(gains)
    hsv = bgr_to_hsv(img)
    hsv = np.stack([lh[hsv[..., 0]], ls[hsv[..., 1]], lv[hsv[..., 2]]], -1)
    return hsv_to_bgr(hsv)


def load_resized(src, img_size):
    """TrainValDataset.load_image with augment=True (datasets.py:278-296): INTER_LINEAR to int(w0 * r), int(h0 * r)."""
    h0, w0 = src.shape[:2]
    ratio = img_size / max(h0, w0)
    if ratio != 1:
        return resize_linear(src, int(w0 * ratio), int(h0 * ratio))
    return src


def mosaic_canvas(imgs, yc, xc, H, W):
    """The img4 of mosaic_augmentation (data_augment.py:156-177) for four resized images."""
    img4 = np.full((H * 2, W * 2, 3), 114, np.uint8)
    for (y1a, y2a, x1a, x2a, y1b, x1b), img in zip(mosaic_tiles([im.shape[:2] for im in imgs], yc, xc, H, W), imgs):
        img4[y1a:y2a, x1a:x2a] = img[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
    return img4


def mosaic_tiles(hw, yc, xc, H, W):
    """Placement of the four tiles: (y1a, y2a, x1a, x2a, y1b, x1b) each, data_augment.py:162-175."""
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


def letterbox_canvas(img, H, W):
    """letterbox(img, (H, W), auto=False, scaleup=True) (data_augment.py:29-58), HWC BGR."""
    h, w = img.shape[:2]
    r = min(H / h, W / w)
    nw, nh = int(round(w * r)), int(round(h * r))
    top, left = int(round((H - nh) / 2 - 0.1)), int(round((W - nw) / 2 - 0.1))
    body = img if (nw, nh) == (w, h) else resize_linear(img, nw, nh)
    out = np.full((H, W, 3), 114, np.uint8)
    out[top:top + nh, left:left + nw] = body
    return out


# The golden dataset: (h0, w0, kind) per image -- COCO-like frames, sources far smaller than the canvas, 1x1, extreme
# aspect ratios, a frame whose load_image size truncates to 639 (so the letterbox resizes it again) and exact fits.
DATASET = [(480, 640, "noise"), (640, 480, "grad"), (333, 517, "noise"), (1, 1, "noise"), (17, 1000, "grad"),
           (1000, 17, "noise"), (100, 60, "grad"), (640, 640, "noise"), (720, 1280, "grad"), (1, 1, "grad"),
           (50, 50, "noise"), (427, 640, "grad"), (606, 450, "noise"), (200, 30, "grad")]
NO_LABELS = 3          # the image without labels


def synthetic_labels(i):
    """Seeded YOLO-format rows float32 [k, 5] (cls, cx, cy, w, h normalised) of dataset image i; image NO_LABELS has none."""
    if i == NO_LABELS:
        return np.zeros((0, 5), np.float32)
    rng = np.random.default_rng(500 + i)
    k = int(rng.integers(1, 12))
    wh = rng.uniform(0.02, 0.9, (k, 2))
    c = rng.uniform(wh / 2, 1 - wh / 2)
    cls = rng.integers(0, 80, (k, 1))
    return np.concatenate([cls, c, wh], 1).astype(np.float32)


def dataset_sources():
    from oracle.letterbox import synthetic_source
    return {i: synthetic_source(h, w, kind, 100 + i) for i, (h, w, kind) in enumerate(DATASET)}


# (name, hyp overrides of yolov6s, H, W, img_size, batch indices, seed)
CASES = [
    ("yolov6s_640_bs8", {}, 640, 640, 640, [0, 1, 2, 7, 8, 11, 12, 13], 1),
    ("yolov6l6_640_bs8", dict(scale=0.9, mixup=0.2), 640, 640, 640, [0, 2, 4, 6, 8, 10, 12, 1], 3),
    ("mixup_always_256", dict(scale=0.9, mixup=1.0), 256, 256, 256, [3, 5, 9], 4),
    ("degrees_shear_320", dict(degrees=10.0, shear=5.0), 320, 320, 320, [0, 4, 5, 10], 5),
    ("no_hsv_flipud_320", dict(hsv_h=0.0, hsv_s=0.0, hsv_v=0.0, flipud=1.0), 320, 320, 320, [1, 6, 9, 13], 6),
    ("letterbox_640", dict(mosaic=0.0, mixup=0.0), 640, 640, 640, [12, 0, 3, 4, 5, 8, 13, 10], 7),
    ("letterbox_affine_320", dict(mosaic=0.0, degrees=10.0, shear=5.0), 320, 320, 320, [12, 2, 6, 9], 8),
    ("rect_384x640", {}, 384, 640, 640, [0, 2, 8, 11], 9),
    ("rect_letterbox_384x640", dict(mosaic=0.0), 384, 640, 640, [0, 5, 8, 12], 10),
]


def compose(rec, sources, H, W, img_size):
    """One sample of TrainValDataset.__getitem__ from a sampler record (yolov6_b200.augment.Sample) and the decoded sources
    {index: uint8 HWC BGR}: uint8 [3, H, W] RGB."""
    def canvas_image(cv):
        imgs = [load_resized(sources[i], img_size) for i in cv.indices]
        if rec.mosaic:
            canvas = mosaic_canvas(imgs, cv.yc, cv.xc, H, W)
        else:
            canvas = letterbox_canvas(imgs[0], H, W)
        if (cv.M != np.eye(3)).any():
            return warp_affine(canvas, cv.M, W, H)
        return canvas

    img = canvas_image(rec.canvases[0])
    if rec.mix_r is not None:
        img2 = canvas_image(rec.canvases[1])
        img = (img * rec.mix_r + img2 * (1 - rec.mix_r)).astype(np.uint8)
    if rec.gains is not None:
        img = augment_hsv(img, rec.gains)
    if rec.flipud:
        img = img[::-1]
    if rec.fliplr:
        img = img[:, ::-1]
    return np.ascontiguousarray(img.transpose(2, 0, 1)[::-1])
