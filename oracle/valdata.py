"""oracle/valdata.py -- numpy restatement of yv6_letterbox_val (TEST INFRASTRUCTURE ONLY).

`resize_area` states OpenCV's uint8 INTER_AREA cv2.resize for a shrink, both of its paths:
  - resizeAreaFast_, when both scales 1 / (n / n0) are integers (is_area_fast): the int sum of each sx x sy box, then
    (sum + 2) >> 2 for 2 x 2 (ResizeAreaFastVec and its scalar tail) or saturate_cast<uchar>(sum * (1.f / area));
  - resizeArea_ otherwise: computeResizeAreaTab's (source, destination, float weight) table per axis, a float32
    horizontal accumulation per source row in table order, a float32 vertical accumulation per destination row
    (sum = beta * buf, then sum += beta * buf) and saturate_cast<uchar> (round half to even).  numpy never fuses a
    multiply into an add, so each float32 step rounds as OpenCV's does.
`load_image` / `val_canvas` compose it with oracle.letterbox.resize_linear into the Evaler's validation image.
tests/test_valdata.py pins resize_area against cv2 directly; tests/golden/make_golden_valdata.py pins the geometry and
canvases against the unmodified reference dataset.
"""
import math

import numpy as np

from .letterbox import resize_linear

DBL_EPSILON = 2.220446049250313e-16


def is_area_fast(h0, w0, nh, nw):
    sx, sy = 1.0 / (nw / w0), 1.0 / (nh / h0)
    return abs(sx - round(sx)) < DBL_EPSILON and abs(sy - round(sy)) < DBL_EPSILON


def area_tab(ssize, dsize):
    """computeResizeAreaTab(ssize, dsize, cn=1, scale): lists of (dst, src, float32 weight) in OpenCV's order."""
    scale = 1.0 / (dsize / ssize)
    tab = []
    for dx in range(dsize):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, ssize - fsx1)
        sx1, sx2 = math.ceil(fsx1), math.floor(fsx2)
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, np.float32((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, np.float32(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def _by_rank(tab, dsize):
    """The table as rank-ordered columns: for tap rank t, (dst indices, src indices, weights) of every dst with > t taps."""
    per = [[] for _ in range(dsize)]
    for d, s, a in tab:
        per[d].append((s, a))
    ranks = []
    for t in range(max(len(p) for p in per)):
        ds = [d for d in range(dsize) if len(per[d]) > t]
        ranks.append((np.array(ds), np.array([per[d][t][0] for d in ds]), np.array([per[d][t][1] for d in ds], np.float32)))
    return ranks


def resize_area(im, nw, nh):
    """cv2.resize(im, (nw, nh), interpolation=cv2.INTER_AREA) for a uint8 HWC shrink (nw <= w0, nh <= h0)."""
    h0, w0 = im.shape[:2]
    if is_area_fast(h0, w0, nh, nw):
        kx, ky = w0 // nw, h0 // nh
        s = im[:nh * ky, :nw * kx].astype(np.int64).reshape(nh, ky, nw, kx, -1).sum(axis=(1, 3))
        if kx == 2 and ky == 2:
            return ((s + 2) >> 2).astype(np.uint8)
        t = s.astype(np.float32) * (np.float32(1) / np.float32(kx * ky))
        return np.clip(np.rint(t), 0, 255).astype(np.uint8)
    src = im.astype(np.float32)
    buf = np.zeros((h0, nw, im.shape[2]), np.float32)
    for d, s, a in _by_rank(area_tab(w0, nw), nw):
        buf[:, d] = buf[:, d] + src[:, s] * a[None, :, None]
    acc = np.zeros((nh, nw, im.shape[2]), np.float32)
    for t, (d, s, a) in enumerate(_by_rank(area_tab(h0, nh), nh)):
        term = buf[s] * a[:, None, None]
        acc[d] = term if t == 0 else acc[d] + term
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def load_image(im, img_size, shrink_size=None):
    """TrainValDataset.load_image with augment=False (datasets.py:257-296) on a decoded BGR image: (img, (h0, w0), (h, w))."""
    h0, w0 = im.shape[:2]
    ratio = (img_size - shrink_size) / max(h0, w0) if shrink_size else img_size / max(h0, w0)
    if ratio != 1:
        nw, nh = int(w0 * ratio), int(h0 * ratio)
        if nw < 1 or nh < 1:
            raise ValueError(f"{h0} x {w0} loads to an empty {nh} x {nw}")
        if (nh, nw) != (h0, w0):
            im = resize_area(im, nw, nh) if ratio < 1 else resize_linear(im, nw, nh)
    return im, (h0, w0), im.shape[:2]


def val_canvas(im, H, W, img_size, shrink_size=None):
    """The Evaler's validation image of a BGR source on an H x W batch canvas: load_image, letterbox(auto=False,
    scaleup=False) -- a pad only -- and HWC->CHW + BGR->RGB: uint8 [3, H, W]."""
    img, _, (h, w) = load_image(im, img_size, shrink_size)
    assert h <= H and w <= W, "the canvas must hold the loaded image"
    top, left = int(round((H - h) / 2 - 0.1)), int(round((W - w) / 2 - 0.1))
    out = np.full((H, W, 3), 114, np.uint8)
    out[top:top + h, left:left + w] = img
    return np.ascontiguousarray(out.transpose(2, 0, 1)[::-1])


def synthetic_source(h0, w0, seed):
    """Seeded uint8 HWC BGR source: smooth ramps plus noise, so both area weights and rounding ties are exercised."""
    rng = np.random.default_rng(9100 + seed)
    y = np.linspace(0, 1, h0, dtype=np.float32)[:, None]
    x = np.linspace(0, 1, w0, dtype=np.float32)[None, :]
    ph = rng.uniform(0, 1, 3).astype(np.float32)
    chans = [127.5 + 100 * np.sin(np.float32(2 * np.pi) * (x * (1 + 2 * c) + y * (2 - c) + ph[c])) for c in range(3)]
    base = np.stack(chans, -1) + rng.integers(-27, 28, (h0, w0, 3)).astype(np.float32)
    return np.ascontiguousarray(base.round().clip(0, 255).astype(np.uint8))


def synthetic_labels(seed, n=None):
    """Seeded YOLO labels [k, 5] float32 (class, x, y, w, h normalised), some boxes reaching past the image edge."""
    rng = np.random.default_rng(9300 + seed)
    k = int(rng.integers(0, 7)) if n is None else n
    cls = rng.integers(0, 80, k)
    xy = rng.uniform(0.02, 0.98, (k, 2))
    wh = rng.uniform(0.01, 0.6, (k, 2))
    return np.concatenate([cls[:, None], xy, wh], 1).astype(np.float32)
