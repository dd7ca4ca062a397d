"""CPU checks of the training augmentation against the reference's goldens (tests/golden/augment_cases.json: what the
reference's __getitem__ drew and the digest of each output; tests/golden/augment.npz: its labels_out; both made by
make_golden_augment.py from the unmodified reference and cv2): the host sampler draws the same numbers, the label path
gives the same rows, and the numpy restatement of the kernels gives the same bytes."""
import hashlib
import random

import numpy as np
import pytest
import torch

from conftest import golden_json, golden_npz
from oracle import augment as oa
from yolov6_b200.augment import Sampler, check_labels, sample_labels

G = golden_json("augment_cases.json")
NPZ = golden_npz("augment.npz")
SRC = oa.dataset_sources()


def drawn(case):
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    return Sampler(len(oa.DATASET), case["H"], case["W"], case["hyp"], case["img_size"]).draw(case["batch"])


def test_goldens_match_cv2_and_cover_the_cases():
    assert G["bgr2hsv_mismatch"] == 0 and G["hsv2bgr_mismatch"] == 0
    assert [c["name"] for c in G["cases"]] == [c[0] for c in oa.CASES]
    assert [tuple(d) for d in G["dataset"]] == oa.DATASET
    for c in G["cases"]:
        assert not any(c["oracle_mismatch"]) and not any(c["warp_mismatch"]) and not any(c["hsv_mismatch"])
    kinds = {(bool(d["centres"]), d["mix_r"] is not None, d["gains"] is not None) for c in G["cases"] for d in c["draws"]}
    assert kinds >= {(True, False, True), (True, True, True), (False, False, True), (True, False, False)}


@pytest.mark.parametrize("ci", range(len(oa.CASES)))
def test_sampler_draws_what_the_reference_draws(ci):
    case = G["cases"][ci]
    plan = drawn(case)
    for rec, ref in zip(plan.samples, case["draws"], strict=True):
        assert rec.index == ref["index"]
        assert rec.sources() == ref["loaded"]
        assert [[cv.yc, cv.xc] for cv in rec.canvases if rec.mosaic] == ref["centres"]
        assert [cv.M.tolist() for cv in rec.canvases] == ref["M"]
        assert [cv.s for cv in rec.canvases] == ref["s"]
        assert rec.mix_r == ref["mix_r"]
        assert (None if rec.gains is None else rec.gains.tolist()) == ref["gains"]
        assert (rec.flipud, rec.fliplr) == (ref["flipud"], ref["fliplr"])
    assert plan.sources == list(dict.fromkeys(i for r in case["draws"] for i in r["loaded"]))


@pytest.mark.parametrize("ci", range(len(oa.CASES)))
def test_labels_equal_reference(ci):
    case = G["cases"][ci]
    shapes = {i: SRC[i].shape[:2] for i in SRC}
    labels = {i: oa.synthetic_labels(i) for i in SRC}
    for k, rec in enumerate(drawn(case).samples):
        got = sample_labels(rec, shapes, labels, case["H"], case["W"], case["img_size"])
        ref = NPZ[f"{case['name']}_{k}_labels"]
        assert got.dtype == torch.float32 and got.shape == ref.shape
        assert np.array_equal(got.numpy(), ref), f"{case['name']} sample {k}"


@pytest.mark.parametrize("ci", range(len(oa.CASES)))
def test_oracle_images_equal_reference(ci):
    case = G["cases"][ci]
    for k, rec in enumerate(drawn(case).samples):
        img = oa.compose(rec, SRC, case["H"], case["W"], case["img_size"])
        assert hashlib.sha256(img.tobytes()).hexdigest() == case["chw_sha256"][k], f"{case['name']} sample {k}"


def test_malformed_labels_raise():
    assert check_labels([], "x").shape == (0, 5)
    for bad in (np.zeros((2, 4)), np.full((1, 5), np.nan), np.array([[0, 0.5, 0.5, 1.2, 0.1]]), np.array([[-1, .5, .5, .1, .1]])):
        with pytest.raises(RuntimeError):
            check_labels(bad, "x")
