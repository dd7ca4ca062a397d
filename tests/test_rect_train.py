"""Training off the square on the host side, against the reference's goldens (tests/golden/make_golden_rect_train.py):
the Sampler's draws and labels_out for --specific-shape and --rect samples, and the --rect batch schedule of each rank."""
import random

import numpy as np
import pytest

from conftest import golden_json, golden_npz
from oracle import augment as oa
from oracle import valdata as ov
from yolov6_b200 import _lib
from yolov6_b200.augment import Sampler, rect_batches, sample_labels
from yolov6_b200.valdata import val_batches, val_geometry, val_labels

G = golden_json("rect_train_cases.json")
NPZ = golden_npz("rect_train.npz")
SRC_SHAPES = {i: (h, w) for i, (h, w, _) in enumerate(oa.DATASET)}
LABELS = {i: oa.synthetic_labels(i) for i in range(len(oa.DATASET))}


@pytest.mark.parametrize("case", G["samples"], ids=[c["name"] for c in G["samples"]])
def test_sampler_labels_equal_reference(case):
    H, W = case["H"], case["W"]
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    if case["target"] == "rect":       # a rect sampler is sized for the square; each batch names its canvas
        s = Sampler(len(oa.DATASET), case["img_size"], case["img_size"], case["hyp"], case["img_size"], target="rect")
        plan = s.draw(case["batch"], (H, W))
    else:
        s = Sampler(len(oa.DATASET), H, W, case["hyp"], case["img_size"], target="specific")
        plan = s.draw(case["batch"])
    assert (plan.H, plan.W) == (H, W)
    for k, rec in enumerate(plan.samples):
        got = sample_labels(rec, SRC_SHAPES, LABELS, H, W, case["img_size"], s.target).numpy()
        want = NPZ[f"{case['name']}_{k}_labels"]
        assert got.dtype == want.dtype and np.array_equal(got, want), f"{case['name']} sample {k}"
    # the box arithmetic's dtype follows the target (float64 for a batch_shapes row, float32 for a specific shape) even
    # where the original rule would not: the square rect_640x640 and the non-square specific letterbox cases pin it


@pytest.mark.parametrize("case", G["loaders"], ids=[c["name"] for c in G["loaders"]])
def test_rect_schedule_equals_reference_loader(case):
    for rank, want in enumerate(case["ranks"]):
        got = rect_batches(case["shapes"], case["img_size"], case["batch"], case["stride"], case["world"], rank)
        assert [[idx, list(c)] for idx, c in got] == want, f"{case['name']} rank {rank}"
        for _, (h, w) in got:
            assert h <= case["img_size"] and w <= case["img_size"]      # pad 0: every canvas fits the square step
    if case["world"] > 1:      # the DDP tail the sampler drops
        n = len(case["shapes"])
        assert sum(len(i) for r in case["ranks"] for i, _ in r) == n // case["world"] * case["world"]


def test_specific_shape_must_be_a_stride_multiple():
    from yolov6_b200.augment import HYP_YOLOV6S, AugmentFeed
    with pytest.raises(ValueError, match="stride"):
        AugmentFeed(2, 384, 608, HYP_YOLOV6S, 10, 1000, 640, target="specific", stride=64)
    with pytest.raises(ValueError):
        Sampler(10, 384, 640, HYP_YOLOV6S, 640, target="square")


VAL = G["val_cases"]


def val_items(name):
    """(settings, [(source index, shapes, labels_out)] in the reference loader's order) of a specific-shape validation case."""
    c = VAL[name]
    lab, off = NPZ[f"val_{name}_labels"], NPZ[f"val_{name}_offsets"]
    return c, [(i, sh, lab[off[k]:off[k + 1]]) for k, (i, sh) in enumerate(zip(c["order"], c["shapes"]))]


@pytest.mark.parametrize("name", list(VAL))
def test_specific_shape_validation_equals_reference(name):
    """Batch order (sorted when rect is on), one (height, width) canvas for every batch, load_image at min(W / w0, H / h0)
    whatever shrink_size says, the Evaler's shapes and labels_out."""
    c, items = val_items(name)
    H, W = c["specific_shape"]
    order, bidx, _ = val_batches(c["sources"], c["img_size"], c["batch"], c["stride"], c["pad"], c["rect"])
    assert order.tolist() == c["order"]
    for k, (i, sh, lab) in enumerate(items):
        h0, w0 = c["sources"][i]
        g = val_geometry(h0, w0, (H, W), c["img_size"], c["shrink_size"], specific_shape=True)
        (rh0, rw0), ((rh, rw), (pl, pt)) = g.shapes
        assert [rh0, rw0, rh, rw, pl, pt] == sh, (name, k, i)
        want = lab.copy()
        want[:, 0] = 0
        got = val_labels(ov.synthetic_labels(i), g)
        assert got.dtype == np.float32 and np.array_equal(got, want), (name, k, i)


def test_specific_shape_validation_cases_cover_every_load_mode():
    modes = {val_geometry(*VAL[n]["sources"][i], VAL[n]["specific_shape"], VAL[n]["img_size"], specific_shape=True).mode
             for n in VAL for i in range(len(VAL[n]["sources"]))}
    assert modes == {_lib.VAL_COPY, _lib.VAL_LINEAR, _lib.VAL_AREA_FAST, _lib.VAL_AREA}, modes
