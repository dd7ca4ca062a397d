"""The CPU oracle of the COCO box evaluation (oracle/cocoeval.py) against hand-worked cases, one per rule of pycocotools'
COCOeval (tests/golden/cocoeval_cases.json); the rounding that turns NMS rows into json rows; the ctypes mirror of
yv6_coco_state; and, where pycocotools imports, the oracle against pycocotools itself on fabricated sets."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import cocoeval as oc

GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "cocoeval_cases.json")) as f:
    CASES = json.load(f)


def select(arr, index):
    """index entries: int, '*' (whole axis) or [lo, hi) -- see tests/golden/make_golden_cocoeval.py."""
    return arr[tuple(slice(None) if i == "*" else slice(i[0], i[1]) if isinstance(i, list) else i for i in index)]


def check_expectations(case, stats, precision, recall, scores):
    arrays = {"stats": stats, "precision": precision, "recall": recall, "scores": scores}
    for name, index, value in case["expect"]:
        got = select(arrays[name], index)
        want = np.broadcast_to(np.asarray(value, np.float64), np.shape(got))
        assert np.array_equal(got, want), (name, index, got, value)


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_case(name):
    case = CASES[name]
    stats, precision, recall, scores = oc.evaluate(case["gt"], case["results"], case.get("img_ids"))
    K = len(case["gt"]["categories"])
    assert precision.shape == (10, 101, K, 4, 3) and recall.shape == (10, K, 4, 3) and scores.shape == precision.shape
    check_expectations(case, stats, precision, recall, scores)


def test_every_rule_has_a_case():
    assert {"perfect", "crowd_three_hits", "gt_id_zero", "tied_scores", "dets_120", "area_boundaries", "crowd_only_category",
            "absent_category", "string_image_ids", "off_the_end"} <= set(CASES)


def test_thresholds_are_params_linspaces():
    assert oc.IOU_THRS[0] == .5 and oc.IOU_THRS[5] == .75 and len(oc.IOU_THRS) == 10
    # 10 of the 101 recall thresholds are not i / 100; the device reads the host's table, never i / 100
    off = [i for i in range(101) if oc.REC_THRS[i] != i / 100]
    assert len(off) == 10 and oc.REC_THRS[35] == 0.35000000000000003


def test_load_res_rejects_unknown_images():
    case = CASES["perfect"]
    with pytest.raises(AssertionError):
        oc.load_res(case["gt"], [dict(case["results"][0], image_id=12345)])


def test_summarize_means_over_entries_above_minus_one():
    precision = -np.ones((10, 101, 2, 4, 3))
    recall = -np.ones((10, 2, 4, 3))
    precision[:, :, 0, 0, 2] = 0.5
    recall[:, 0, 0, 2] = 0.25
    s = oc.summarize(precision, recall)
    assert s[0] == 0.5 and s[1] == 0.5 and s[8] == 0.25 and s[3] == -1 and s[6] == -1


def device_round(v, scale):
    """The device formula of yv6_coco_update: rint((double)v * scale) / scale."""
    return np.rint(v.astype(np.float64) * scale) / scale


def test_device_rounding_equals_round_and_json():
    rng = np.random.default_rng(0)
    v = np.concatenate([(rng.random(200000) * 1300 - 10).astype(np.float32), rng.random(100000).astype(np.float32),
                        (rng.random(50000) * 1e-3).astype(np.float32)])
    # exact ties at the 4th / 6th decimal: k / 2^n with few enough bits to be exact in fp32
    ties = np.array([1.0625, 2.0625, 0.0625, 3.4375, 0.5625, 12.3125, 1.5 / 1024, 5 / 64, 0.03125, 0.00048828125], np.float32)
    v = np.concatenate([v, ties, -ties])
    for scale, nd in ((1e3, 3), (1e5, 5)):
        want = np.array(json.loads(json.dumps([round(x, nd) for x in v.tolist()])))
        got = device_round(v, scale)
        assert np.array_equal(got.view(np.int64), want.view(np.int64)), int((got != want).sum())
    assert device_round(np.array([1.0625], np.float32), 1e3)[0] == 1.062          # half to even


def test_ctypes_mirror_of_the_coco_state_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    from yolov6_b200 import _lib
    src = tmp_path / "coco.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yv6.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(yv6_coco_state), offsetof(yv6_coco_state, gt_off), '
                   'offsetof(yv6_coco_state, score), offsetof(yv6_coco_state, flags));return 0;}\n')
    exe = tmp_path / "coco"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    S = _lib.CocoState
    assert got == [C.sizeof(S), S.gt_off.offset, S.score.offset, S.flags.offset]


def test_library_exports_the_coco_entry_points():
    from yolov6_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    for n in ("yv6_coco_workspace_bytes", "yv6_coco_update", "yv6_coco_load", "yv6_coco_accumulate"):
        assert hasattr(lib, n) and n in _lib.exported_symbols()
    assert lib.yv6_coco_workspace_bytes(5000, 300, 80) > 5000 * 300 * 40


def test_fabricated_set_covers_the_rules():
    gt, batches, ids = oc.fabricate(1, 64, n_cats=12, B=16)
    area = np.array([a["area"] for a in gt["annotations"]])
    assert (area < 32 ** 2).any() and ((area > 32 ** 2) & (area < 96 ** 2)).any() and (area > 96 ** 2).any()
    assert any(a["id"] == 0 for a in gt["annotations"])
    assert len(gt["categories"]) == 11 and ids[-1] not in {c["id"] for c in gt["categories"]}
    assert sum(len(b[3]) for b in batches) == 64 and max(int(b[1].max()) for b in batches) == 300


def _pycocotools():
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
    except ImportError:
        return None
    if not hasattr(COCOeval, "evaluate"):                   # a stand-in module, not pycocotools
        return None
    return COCO, COCOeval


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_matches_pycocotools(seed, tmp_path):
    pc = _pycocotools()
    if pc is None:
        pytest.skip("pycocotools is not installed")
    COCO, COCOeval = pc
    gt, batches, ids = oc.fabricate(seed, 120, n_cats=20, gts_per_image=6, crowd=0.05, B=16)
    rows = oc.rows_of(batches, ids)
    cases = [(gt, rows, None)] + [(c["gt"], c["results"], c.get("img_ids")) for c in CASES.values()]
    for g, r, img_ids in cases:
        with open(tmp_path / "gt.json", "w") as f:
            json.dump(g, f)
        coco = COCO(str(tmp_path / "gt.json"))
        ev = COCOeval(coco, coco.loadRes(r), "bbox")
        if img_ids is not None:
            ev.params.imgIds = img_ids
        ev.evaluate()
        ev.accumulate()
        ev.summarize()
        stats, precision, recall, scores = oc.evaluate(g, r, img_ids)
        assert np.array_equal(precision, ev.eval["precision"]) and np.array_equal(recall, ev.eval["recall"])
        assert np.array_equal(scores, ev.eval["scores"]) and np.array_equal(stats, ev.stats)
