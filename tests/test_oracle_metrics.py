"""The CPU oracle of the PR metric (oracle/metrics.py) against goldens of the unmodified reference Evaler
(tests/golden/make_golden_metrics.py), and the tie / interpolation rules it states."""
import json
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import metrics as om

GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "metrics_cases.json")) as f:
    CASES = json.load(f)


def golden_batches(g, name):
    meta = CASES[name]
    out = []
    for bi in range(meta["n_batches"]):
        rows, count, targets = g[f"{name}/b{bi}/rows"], g[f"{name}/b{bi}/count"], g[f"{name}/b{bi}/targets"]
        preds = np.split(rows, np.cumsum(count)[:-1])
        shapes = [((s[0][0], s[0][1]), ((s[1][0], s[1][1]), (s[2][0], s[2][1]))) for s in meta["shapes"][bi]]
        out.append((preds, targets, shapes, (meta["H"], meta["W"])))
    return out


def check_against_golden(res, g, name, tol=1e-12):
    """res: dict with the oracle's / PRMetric's fields.  Flags, classes, counts, matrix and i* exact; values to tol."""
    meta = CASES[name]
    assert np.array_equal(np.asarray(res["nt"]), np.array(meta["nt"])), name
    assert np.array_equal(res["matrix"], g[f"{name}/matrix"]), name
    assert bool(res["ok"]) == meta["ok"], name
    if not meta["ok"]:
        assert res["map50"] == 0.0 and res["map"] == 0.0
        return
    assert np.array_equal(res["ap_class"], g[f"{name}/ap_class"]), name
    for k in ("p", "r", "ap", "f1"):
        assert res[k].shape == g[f"{name}/{k}"].shape, (name, k)
        err = float(np.abs(res[k] - g[f"{name}/{k}"]).max()) if res[k].size else 0.0
        assert err <= tol, (name, k, err)
    assert res["best"] == meta["best"], name
    for k in ("map50", "map", "mp", "mr"):
        assert abs(res[k] - meta[k]) <= tol, (name, k, res[k], meta[k])


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "metrics.npz"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference(golden, name):
    res = om.evaluate(golden_batches(golden, name), CASES[name]["nc"])
    assert np.array_equal(res["correct"], golden[f"{name}/correct"]), name
    assert np.array_equal(res["conf"], golden[f"{name}/conf"]) and np.array_equal(res["pcls"], golden[f"{name}/pcls"])
    assert np.array_equal(res["tcls"], golden[f"{name}/tcls"])
    check_against_golden(res, golden, name)


def test_exact_threshold_ious(golden):
    """0.5, 0.75 and 55/100 sit exactly on iouv entries: `>=` makes them correct at that threshold and not the next."""
    c = golden["exact/correct"]
    assert c[0].tolist() == [True] + [False] * 9                          # IoU 0.5
    assert c[1].tolist() == [True] * 6 + [False] * 4                      # IoU 0.75 = iouv[5]
    assert c[2].tolist() == [True, True] + [False] * 8                    # 55/100 == iouv[1] in fp32
    assert c[3].tolist() == [False] * 10                                  # same label, higher row index
    assert np.float32(55) / np.float32(100) == om.IOUV[1]


def test_interp_repeated_points_take_the_last():
    assert om.interp([0.5], [0, .5, .5, 1], [1, .8, .6, 0], left=1)[0] == 0.6
    rng = np.random.default_rng(0)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        xp = np.sort(rng.integers(0, 8, n) / 7.0)                        # many repeats
        fp = rng.random(n)
        x = np.concatenate([rng.uniform(-0.2, 1.2, 50), xp])
        for left in (0.0, 1.0):
            assert np.array_equal(om.interp(x, xp, fp, left), np.interp(x, xp, fp, left=left))


def test_compute_ap_equals_trapz_of_np_interp():
    rng = np.random.default_rng(1)
    for _ in range(50):
        tp = rng.random(int(rng.integers(1, 60))) < 0.5
        tpc = np.cumsum(tp).astype(np.float64)
        recall, precision = tpc / (int(tp.sum()) + 3 + 1e-16), tpc / np.arange(1, len(tp) + 1)
        mrec = np.concatenate(([0.], recall, [recall[-1] + 0.01]))
        mpre = np.flip(np.maximum.accumulate(np.flip(np.concatenate(([1.], precision, [0.])))))
        x = np.linspace(0, 1, 101)
        want = np.sum(np.diff(x) * (np.interp(x, mrec, mpre)[1:] + np.interp(x, mrec, mpre)[:-1]) / 2.0)
        assert om.compute_ap(recall, precision) == want


def test_tie_rules():
    # two labels with the same IoU to one detection: the lower label index is L(d); a second detection on that label
    # is then not correct, one on the other label is
    iou = np.array([[0.8, 0.8, 0.0], [0.8, 0.0, 0.9]], np.float32)
    lcls, dcls = np.zeros(2, np.float32), np.zeros(3, np.float32)
    c = om.correct_flags(iou, lcls, dcls)
    assert c[:, 0].tolist() == [True, False, True]
    # process_batch keeps the lowest detection index per label, not the highest IoU
    iou = np.array([[0.6, 0.95]], np.float32)
    c = om.correct_flags(iou, np.zeros(1, np.float32), np.zeros(2, np.float32))
    assert c[:, 0].tolist() == [True, False]
    assert c[1].tolist() == (om.IOUV > np.float32(0.6)).tolist()          # where the first is no candidate, the second counts
    # the confusion matrix keeps the highest IoU per label (the re-sort of metrics.py:198 is applied)
    m = np.zeros((3, 3))
    om.confusion_update(m, np.array([[0.6, 0.95]], np.float32), np.zeros(1, np.float32), np.array([0.9, 0.9], np.float32),
                        np.array([0, 1], np.float32), 2)
    assert m[1, 0] == 1 and m[0, 2] == 1 and m.sum() == 2
