"""CPU checks of the validation-batch host side (yolov6_b200/valdata.py) and its oracle: the batch order and canvases,
each image's geometry, shapes and labels equal to what the reference's TrainValDataset(augment=False) produced
(tests/golden/valdata_cases.json), oracle/valdata.py's INTER_AREA byte-identical to cv2, the ctypes mirror of
yv6_letterbox_val against the header, and the refusals that happen before anything is written or enqueued."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import valdata as ov
from yolov6_b200 import _lib
from yolov6_b200.valdata import ValFeed, val_batches, val_geometry, val_labels

GOLDEN = os.path.join(ROOT, "tests", "golden")
CUDA0 = torch.device("cuda", 0)       # never touched: every refusal below happens before a CUDA call


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "valdata_cases.json")) as f:
        cases = json.load(f)
    return cases, dict(np.load(os.path.join(GOLDEN, "valdata.npz")))


def case_items(golden, name):
    """(settings, [(source index, shapes, labels_out)] in loader order)."""
    cases, arrays = golden
    c = cases["cases"][name]
    lab, off = arrays[f"{name}_labels"], arrays[f"{name}_offsets"]
    items = [(i, sh, lab[off[k]:off[k + 1]]) for k, (i, sh) in enumerate(zip(c["order"], c["shapes"]))]
    return c, items


def shapes_tuple(sh):
    h0, w0, rh, rw, pl, pt = sh
    return (h0, w0), ((rh, rw), (pl, pt))


NAMES = ["rect640", "rect320", "rect1280", "square640", "shrink640", "metric200"]


@pytest.mark.parametrize("name", NAMES)
def test_batches_geometry_and_labels_equal_the_reference(golden, name):
    c, items = case_items(golden, name)
    order, bidx, canvases = val_batches(c["sources"], c["img_size"], c["batch"], c["stride"], c["pad"], c["rect"])
    assert order.tolist() == c["order"]
    if c["rect"]:
        assert canvases.tolist() == c["batch_shapes"]
    else:
        assert (canvases == c["img_size"]).all()
    for k, (i, sh, lab) in enumerate(items):
        h0, w0 = c["sources"][i]
        g = val_geometry(h0, w0, canvases[bidx[k]], c["img_size"], c["shrink_size"])
        assert g.shapes == shapes_tuple(sh), (k, i)
        want = lab.copy()
        want[:, 0] = 0
        got = val_labels(ov.synthetic_labels(i), g)
        assert got.dtype == np.float32 and np.array_equal(got, want), (k, i)


def test_cases_cover_every_mode(golden):
    seen = set()
    for name in NAMES:
        c, _ = case_items(golden, name)
        order, bidx, canvases = val_batches(c["sources"], c["img_size"], c["batch"], c["stride"], c["pad"], c["rect"])
        for k, i in enumerate(order):
            g = val_geometry(*c["sources"][i], canvases[bidx[k]], c["img_size"], c["shrink_size"])
            fast = (g.h0 // g.h, g.w0 // g.w) if g.mode == _lib.VAL_AREA_FAST else None
            seen.add((g.mode, fast))
    modes = {m for m, _ in seen}
    assert modes == {_lib.VAL_COPY, _lib.VAL_LINEAR, _lib.VAL_AREA, _lib.VAL_AREA_FAST}
    assert {(2, 2), (3, 3), (4, 4)} <= {f for _, f in seen if f}


@pytest.mark.parametrize("name", ["rect640", "rect320", "shrink640"])
def test_oracle_canvases_hash_like_the_reference(golden, name):
    import hashlib
    c, items = case_items(golden, name)
    _, bidx, canvases = val_batches(c["sources"], c["img_size"], c["batch"], c["stride"], c["pad"], c["rect"])
    for k, (i, _, _) in enumerate(items):
        H, W = canvases[bidx[k]]
        im = ov.val_canvas(ov.synthetic_source(*c["sources"][i], i), H, W, c["img_size"], c["shrink_size"])
        assert hashlib.sha256(im.tobytes()).hexdigest() == c["sha256"][k], (k, i)


def test_oracle_inter_area_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    cases = [(480, 640, 240, 320), (360, 480, 120, 160), (1280, 960, 320, 240), (300, 200, 100, 100), (427, 640, 213, 320),
             (641, 640, 640, 639), (1000, 777, 320, 248), (7, 9, 1, 1), (17, 1000, 5, 320)]
    for _ in range(300):
        h0, w0 = int(rng.integers(2, 300)), int(rng.integers(2, 300))
        r = rng.uniform(0.02, 1.0)
        cases.append((h0, w0, max(1, min(h0, int(h0 * r))), max(1, min(w0, int(w0 * r)))))
    fast = 0
    for j, (h0, w0, nh, nw) in enumerate(cases):
        im = ov.synthetic_source(h0, w0, j)
        fast += ov.is_area_fast(h0, w0, nh, nw)
        assert np.array_equal(ov.resize_area(im, nw, nh), cv2.resize(im, (nw, nh), interpolation=cv2.INTER_AREA)), (h0, w0, nh, nw)
    assert fast >= 5


def test_letterbox_val_mirror_matches_the_header(tmp_path):
    with open(os.path.join(ROOT, "include", "yv6.h")) as f:
        hdr = f.read()
    proto = re.search(r"int yv6_letterbox_val\(([^)]*)\)", hdr).group(1)
    assert len(proto.split(",")) == len(_lib._SIGNATURES["yv6_letterbox_val"][1])
    assert "yv6_letterbox_val" in _lib.exported_symbols()
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "val.c"
    src.write_text('#include <stdio.h>\n#include "yv6.h"\nint main(){printf("%d %d %d %d %d\\n", YV6_VAL_COPY, YV6_VAL_LINEAR, '
                   'YV6_VAL_AREA, YV6_VAL_AREA_FAST, YV6_LB_GEO);return 0;}\n')
    exe = tmp_path / "val"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [_lib.VAL_COPY, _lib.VAL_LINEAR, _lib.VAL_AREA, _lib.VAL_AREA_FAST, 8]


def test_geometry_refusals(golden):
    cases, _ = golden
    for r in cases["refusals"]:
        assert r["reference_raised"]                       # cv2.resize raised in the reference's load_image
        with pytest.raises(RuntimeError, match="empty size"):
            val_geometry(r["h0"], r["w0"], (r["img_size"], r["img_size"]), r["img_size"], r["shrink_size"])
    with pytest.raises(RuntimeError, match="larger than its"):
        val_geometry(480, 640, (480, 608), 640)             # loads to 480 x 640
    with pytest.raises(RuntimeError, match="larger than its"):
        val_geometry(480, 640, (448, 640), 640)
    g = val_geometry(480, 640, (480, 640), 640)              # an exact fit is a plain copy with no border
    assert (g.mode, g.top, g.left, g.shapes) == (_lib.VAL_COPY, 0, 0, ((480, 640), ((1.0, 1.0), (0, 0))))


def test_feed_refuses_before_enqueueing():
    shapes = [(480, 640), (640, 480), (427, 640), (100, 100)]
    feed = ValFeed(2, 320, 32, shapes, device=CUDA0)
    b0, b1 = feed.batches()
    im = {i: np.zeros((*shapes[i], 3), np.uint8) for i in range(4)}
    lab = [np.zeros((0, 5), np.float32)] * 2
    bad = [
        ((list(b0), [im[b0[0]], im[b0[0]].astype(np.float32)], lab), "uint8"),
        ((list(b0), [im[b0[0]], im[b0[1]][:, :, :2]], lab), "3 channels"),
        ((list(b0), [im[b0[0]], torch.zeros(*shapes[b0[1]], 3, dtype=torch.uint8, device="meta")], lab), "a frame on meta"),
        ((list(b0), [im[b0[1]], im[b0[0]]] if shapes[b0[0]] != shapes[b0[1]] else [im[b0[0]], np.zeros((9, 9, 3), np.uint8)], lab),
         "entry in shapes_hw"),
        (([b0[0], b1[0]], [im[b0[0]], im[b1[0]]], lab), "span batches"),
        ((list(b0), [im[b0[0]], im[b0[1]]], lab[:1]), "label arrays"),
        (([b0[0]], [im[b0[0]], im[b0[1]]], lab), "indices for"),
        (([9], [im[0]], lab[:1]), "outside"),
        ((list(b0) + [b1[0]], [im[i] for i in list(b0) + [b1[0]]], lab + lab[:1]), "for a batch of 2"),
    ]
    for args, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            feed.feed(*args)
    small = ValFeed(2, 320, 32, shapes, max_src_bytes=1000, device=CUDA0)
    with pytest.raises(RuntimeError, match="max_src_bytes"):
        small.feed(list(b0), [im[i] for i in b0], lab)
    zero = ValFeed(2, 640, 32, shapes, shrink_size=640, device=CUDA0)
    with pytest.raises(RuntimeError, match="empty size"):
        zero.feed(list(b0), [im[i] for i in b0], lab)
    with pytest.raises(RuntimeError, match="CUDA"):
        ValFeed(2, 320, 32, shapes, device="cpu")
