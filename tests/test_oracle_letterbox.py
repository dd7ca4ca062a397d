"""CPU checks of the letterbox / rescale restatement against the reference's goldens (tests/golden/letterbox_cases.json: canvas
digests, tests/golden/letterbox.npz: rescaled rows; made by make_golden_letterbox.py from the unmodified reference and cv2), and
of the host-side geometry and frame validation."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import golden_json, golden_npz
from oracle import letterbox as ol
from yolov6_b200.preprocess import GEO, letterbox_geometry, pack_frames

G = golden_json("letterbox_cases.json")
NPZ = golden_npz("letterbox.npz")


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_cases_are_the_golden_ones():
    assert [(c["h0"], c["w0"], c["H"], c["W"], c["scaleup"], c["kind"]) for c in G["cases"]] == [tuple(c) for c in ol.CASES]
    assert [tuple(c) for c in G["rescale_cases"]] == [tuple(c) for c in ol.RESCALE_CASES]
    for c in G["cases"]:
        assert int(ol.synthetic_source(c["h0"], c["w0"], c["kind"], c["seed"]).astype(np.int64).sum()) == c["src_sum"]


@pytest.mark.parametrize("i", range(len(ol.CASES)))
def test_geometry_equals_reference(i):
    c = G["cases"][i]
    r, (nw, nh), top, left = letterbox_geometry(c["h0"], c["w0"], c["H"], c["W"], c["scaleup"])
    assert (r, top, left) == (c["r"], c["top"], c["left"])
    assert ol.geometry(c["h0"], c["w0"], c["H"], c["W"], c["scaleup"]) == (r, (nw, nh), top, left)
    canvas = ol.letterbox(ol.synthetic_source(c["h0"], c["w0"], c["kind"], c["seed"]), c["H"], c["W"], c["scaleup"])
    assert sha256(canvas) == c["canvas_sha256"]
    inside = canvas[:, top:top + nh, left:left + nw]
    assert inside.shape == (3, nh, nw)
    assert (canvas == 114).sum() >= 3 * (c["H"] * c["W"] - nh * nw)       # the border around new_unpad is all 114


@pytest.mark.parametrize("i", range(len(ol.CASES)))
def test_restatement_bit_exact_against_cv2(i):
    c = G["cases"][i]
    assert c["oracle_mismatch"] == 0
    im = ol.synthetic_source(c["h0"], c["w0"], c["kind"], c["seed"])
    canvas = ol.letterbox(im, c["H"], c["W"], c["scaleup"])
    assert canvas.dtype == np.uint8 and canvas.shape == (3, c["H"], c["W"])
    assert sha256(canvas) == c["canvas_sha256"]


@pytest.mark.parametrize("j", range(len(ol.RESCALE_CASES)))
def test_rescale_restatement_equals_reference(j):
    h0, w0, H, W = ol.RESCALE_CASES[j]
    assert np.array_equal(ol.rescale(NPZ[f"r{j}_det"], H, W, h0, w0), NPZ[f"r{j}_out"])


def test_pack_frames_layout_and_rejections():
    frames = [np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3), torch.full((5, 1, 3), 7, dtype=torch.uint8)]
    src, geo = torch.zeros(64, dtype=torch.uint8), torch.zeros(3, GEO, dtype=torch.int32)
    used, shapes = pack_frames(frames, 3, 32, 64, True, src, geo)
    assert used == 18 + 15
    assert src[:18].tolist() == list(range(18)) and src[18:33].tolist() == [7] * 15
    r, (nw, nh), top, left = letterbox_geometry(5, 1, 32, 64, True)
    assert geo[1].tolist() == [18, 5, 1, nh, nw, top, left, 0]
    assert geo[2].tolist() == [0, 32, 64, 0, 0, 0, 0, 0]                  # unused slot: all border
    assert shapes[1] == ((5, 1), ((5 * r / 5, 1 * r / 1), (left, top)))
    before = (src.clone(), geo.clone())
    bad = [
        [np.zeros((40, 1, 3), np.uint8)] * 1,         # 120 bytes > 64
        [np.zeros((2, 2, 3), np.float32)],
        [np.zeros((2, 2, 4), np.uint8)],
        [np.zeros((2, 2), np.uint8)],
        [np.zeros((2, 2, 3), np.uint8)] * 4,           # more frames than slots
        [],
    ]
    for b in bad:
        with pytest.raises(RuntimeError):
            pack_frames(b, 3, 32, 64, True, src, geo)
        assert torch.equal(src, before[0]) and torch.equal(geo, before[1])
