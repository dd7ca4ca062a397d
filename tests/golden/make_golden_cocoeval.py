"""Writes tests/golden/cocoeval_cases.json: small COCO box-evaluation cases, one per rule of pycocotools' COCOeval
(bbox, default Params), with the expected values worked out by hand in the comments below (nothing here runs an
evaluator).  Each expectation is (array, index, value): index entries are an int, "*" for a whole axis or [lo, hi) for a
range; every selected entry must equal value exactly.  Arrays: precision / scores [T,R,K,A,M], recall [T,K,A,M], stats.

    python tests/golden/make_golden_cocoeval.py

Recurring numbers (eps = np.spacing(1)): 1 / (1 + eps) = 0.9999999999999998; 2 / (2 + eps) = 1; 1 / (2 + eps) = 0.5;
1 / (100 + eps) = 0.01.  Recall thresholds 25, 33, 50 are exactly 0.25, 0.33, 0.5.
"""
import json
import os

ONE_EPS = 0.9999999999999998            # 1 / (1 + eps): the precision of a lone first tp
ALL, SMALL, MEDIUM, LARGE = 0, 1, 2, 3


def img(i):
    return {"id": i, "height": 1000, "width": 1000}


def ann(i, image, cat, box, area=None, crowd=0):
    return {"id": i, "image_id": image, "category_id": cat, "bbox": box, "area": box[2] * box[3] if area is None else area,
            "iscrowd": crowd}


def det(image, cat, box, score):
    return {"image_id": image, "category_id": cat, "bbox": box, "score": score}


def cats(*ids):
    return [{"id": c, "name": f"c{c}"} for c in ids]


CASES = {}

# perfect detections of two small (100) and two large (40000) gts.  Every range holding gts sees its tps first or after
# ignored dets only, so the envelope is 1 everywhere; medium has no gt: -1.  AR@1: only the top det per image, 1 of 4.
CASES["perfect"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(1, 1, 1, [10, 10, 10, 10]), ann(2, 1, 1, [300, 300, 200, 200]), ann(3, 1, 1, [30, 10, 10, 10]),
                        ann(4, 1, 1, [600, 600, 200, 200])]},
    results=[det(1, 1, [10, 10, 10, 10], 0.9), det(1, 1, [300, 300, 200, 200], 0.8), det(1, 1, [30, 10, 10, 10], 0.7),
             det(1, 1, [600, 600, 200, 200], 0.6)],
    expect=[["stats", ["*"], [1, 1, 1, 1, -1, 1, 0.25, 1, 1, 1, -1, 1]],
            ["precision", ["*", "*", 0, MEDIUM, "*"], -1], ["recall", ["*", 0, MEDIUM, "*"], -1],
            ["precision", ["*", "*", 0, SMALL, 2], 1.0], ["precision", ["*", "*", 0, LARGE, 2], 1.0]])

# three dets inside one crowd gt (crowd IoU = inter / det area = 1) all match it and are ignored, never fps; the two
# regular gts are then found: all-range precision 1 everywhere at maxDet 10 and 100 (at maxDet 1 the one det kept is an
# ignored one: 0).  small and large hold no counted gt: -1.
CASES["crowd_three_hits"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(1, 1, 1, [0, 0, 40, 40]), ann(2, 1, 1, [100, 0, 40, 40]), ann(3, 1, 1, [300, 300, 200, 200], crowd=1)]},
    results=[det(1, 1, [310, 310, 50, 50], 0.95), det(1, 1, [400, 400, 60, 60], 0.94), det(1, 1, [320, 420, 30, 30], 0.93),
             det(1, 1, [0, 0, 40, 40], 0.9), det(1, 1, [100, 0, 40, 40], 0.8)],
    expect=[["precision", ["*", "*", 0, ALL, [1, 3]], 1.0], ["precision", ["*", "*", 0, MEDIUM, 2], 1.0],
            ["precision", ["*", "*", 0, ALL, 0], 0.0],
            ["recall", ["*", 0, ALL, 2], 1.0], ["precision", ["*", "*", 0, SMALL, "*"], -1],
            ["precision", ["*", "*", 0, LARGE, "*"], -1], ["stats", [0], 1.0]])

# the gt with id 0 (area field 1000, box 32x32) is matched by det A (33x33, IoU 1024/1089 = 0.94; unmatched at 0.95)
# and A is scored as a false positive in 'all': tp = [0, 1], fp = [1, 1], pr = [0, 0.5] -> 0.5 up to recall 0.5, then
# off the end.  In 'small' A's area 1089 is out of range and dtm == 0, so A is ignored: pr = [_, 1/(1+eps)].
CASES["gt_id_zero"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(0, 1, 1, [0, 0, 32, 32], area=1000), ann(1, 1, 1, [100, 100, 20, 20])]},
    results=[det(1, 1, [0, 0, 33, 33], 0.9), det(1, 1, [100, 100, 20, 20], 0.8)],
    expect=[["precision", ["*", [0, 51], 0, ALL, 2], 0.5], ["precision", ["*", [51, 101], 0, ALL, 2], 0.0],
            ["recall", ["*", 0, ALL, 2], 0.5], ["precision", ["*", [0, 51], 0, SMALL, 2], ONE_EPS],
            ["precision", ["*", [51, 101], 0, SMALL, 2], 0.0], ["recall", ["*", 0, SMALL, 2], 0.5],
            ["stats", [0], 0.2524752475247525], ["stats", [1], 0.2524752475247525]])   # 255 / 1010 and 25.5 / 101

# all scores tie at 0.5.  Category 1: image 1 lists its fp before its tp, and the per-image sort keeps that order.
# Category 2: image 2's tp comes first in the results but image 1's fp first in sorted-imgId order, which the
# accumulate sort keeps.  Both: [fp, tp] with 2 gts -> precision 0.5 up to recall 0.5 ([tp, fp] would give 1/(1+eps)).
CASES["tied_scores"] = dict(
    gt={"images": [img(1), img(2)], "categories": cats(1, 2),
        "annotations": [ann(1, 1, 1, [0, 0, 50, 50]), ann(2, 1, 2, [200, 200, 50, 50]), ann(3, 2, 1, [0, 0, 50, 50]),
                        ann(4, 2, 2, [0, 0, 50, 50])]},
    results=[det(2, 2, [0, 0, 50, 50], 0.5), det(1, 1, [400, 400, 50, 50], 0.5), det(1, 1, [0, 0, 50, 50], 0.5),
             det(1, 2, [400, 400, 50, 50], 0.5)],
    expect=[["precision", ["*", [0, 51], "*", ALL, 2], 0.5], ["precision", ["*", [51, 101], "*", ALL, 2], 0.0],
            ["scores", ["*", [0, 51], "*", ALL, 2], 0.5], ["recall", ["*", "*", ALL, 2], 0.5]])

# 120 dets in one (image, category): 100 fps score above the only tp (listed first in the results), 19 below.  The tp
# ranks 101st and is dropped: no tp at any maxDet; precision 0 (r = 0 reads the envelope at the first det, 0), scores
# hold the top score at r = 0 and 0 beyond (searchsorted runs off the end).
CASES["dets_120"] = dict(
    gt={"images": [img(1)], "categories": cats(1), "annotations": [ann(1, 1, 1, [0, 0, 50, 50])]},
    results=[det(1, 1, [0, 0, 50, 50], 0.3)] + [det(1, 1, [900, 900, 10, 10], round(0.9 - i * 0.001, 3)) for i in range(100)]
    + [det(1, 1, [900, 900, 10, 10], 0.2) for _ in range(19)],
    expect=[["recall", ["*", 0, ALL, "*"], 0.0], ["precision", ["*", "*", 0, ALL, "*"], 0.0],
            ["scores", ["*", 0, 0, ALL, "*"], 0.9], ["scores", ["*", [1, 101], 0, ALL, "*"], 0.0],
            ["stats", [0], 0.0], ["stats", [8], 0.0]])

# areas exactly 1024 and 9216 belong to both neighbouring ranges.  medium counts both (two tps: precision 1);
# small counts only A and large only B, each a lone tp beside an ignored det: 1/(1+eps) everywhere; recall 1 in all.
CASES["area_boundaries"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(1, 1, 1, [0, 0, 32, 32]), ann(2, 1, 1, [100, 100, 96, 96])]},
    results=[det(1, 1, [0, 0, 32, 32], 0.9), det(1, 1, [100, 100, 96, 96], 0.8)],
    expect=[["recall", ["*", 0, "*", 2], 1.0], ["precision", ["*", "*", 0, MEDIUM, 2], 1.0],
            ["precision", ["*", "*", 0, SMALL, 2], ONE_EPS], ["precision", ["*", "*", 0, LARGE, 2], ONE_EPS],
            ["stats", [4], 1.0], ["stats", [9], 1.0], ["stats", [10], 1.0], ["stats", [11], 1.0]])

# category 2 has only a crowd gt: npig = 0 in every range, so all its entries stay -1 and the means skip it.
CASES["crowd_only_category"] = dict(
    gt={"images": [img(1)], "categories": cats(1, 2),
        "annotations": [ann(1, 1, 1, [0, 0, 50, 50]), ann(2, 1, 1, [100, 0, 50, 50]), ann(3, 1, 2, [200, 200, 100, 100], crowd=1)]},
    results=[det(1, 1, [0, 0, 50, 50], 0.9), det(1, 1, [100, 0, 50, 50], 0.8), det(1, 2, [210, 210, 50, 50], 0.95)],
    expect=[["precision", ["*", "*", 1, "*", "*"], -1], ["recall", ["*", 1, "*", "*"], -1], ["scores", ["*", "*", 1, "*", "*"], -1],
            ["stats", [0], 1.0], ["stats", [8], 1.0]])

# a det of category 99, absent from the gt json, is dropped: category 1 stays perfect.
CASES["absent_category"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(1, 1, 1, [0, 0, 50, 50]), ann(2, 1, 1, [100, 0, 50, 50])]},
    results=[det(1, 99, [0, 0, 50, 50], 0.99), det(1, 1, [0, 0, 50, 50], 0.9), det(1, 1, [100, 0, 50, 50], 0.8)],
    expect=[["precision", ["*", "*", 0, ALL, 2], 1.0], ["stats", [0], 1.0]])

# string image ids (the reference's generated labels) sort as strings: 'a10' < 'a9' < 'b'.  a10 holds the tp, a9 an fp
# of the same score: [tp, fp] with 3 gts -> 1/(1+eps) up to recall 1/3 (r <= 33), then off the end.
CASES["string_image_ids"] = dict(
    gt={"images": [img("b"), img("a10"), img("a9")], "categories": cats(1),
        "annotations": [ann(1, "a9", 1, [0, 0, 50, 50]), ann(2, "a10", 1, [0, 0, 50, 50]), ann(3, "b", 1, [0, 0, 50, 50])]},
    results=[det("a9", 1, [300, 300, 50, 50], 0.5), det("a10", 1, [0, 0, 50, 50], 0.5)],
    expect=[["precision", ["*", [0, 34], 0, ALL, 2], ONE_EPS], ["precision", ["*", [34, 101], 0, ALL, 2], 0.0]])

# four gts, one tp then one fp: rc = [0.25, 0.25]; searchsorted runs off the end for every threshold above 0.25.
CASES["off_the_end"] = dict(
    gt={"images": [img(1)], "categories": cats(1),
        "annotations": [ann(i + 1, 1, 1, [100 * i, 0, 40, 40]) for i in range(4)]},
    results=[det(1, 1, [0, 0, 40, 40], 0.9), det(1, 1, [500, 500, 40, 40], 0.8)],
    expect=[["precision", ["*", [0, 26], 0, ALL, 2], ONE_EPS], ["precision", ["*", [26, 101], 0, ALL, 2], 0.0],
            ["scores", ["*", [0, 26], 0, ALL, 2], 0.9], ["scores", ["*", [26, 101], 0, ALL, 2], 0.0],
            ["recall", ["*", 0, ALL, 2], 0.25]])

# params.imgIds = [1]: image 2 (only fps) is left out, image 1's two perfect dets give 1.
CASES["img_ids_subset"] = dict(
    gt={"images": [img(1), img(2)], "categories": cats(1),
        "annotations": [ann(1, 1, 1, [0, 0, 50, 50]), ann(2, 1, 1, [100, 0, 50, 50]), ann(3, 2, 1, [0, 0, 50, 50])]},
    results=[det(2, 1, [500, 500, 50, 50], 0.99), det(1, 1, [0, 0, 50, 50], 0.9), det(1, 1, [100, 0, 50, 50], 0.8)],
    img_ids=[1],
    expect=[["precision", ["*", "*", 0, ALL, 2], 1.0], ["stats", [0], 1.0]])

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cocoeval_cases.json")
    with open(path, "w") as f:
        json.dump(CASES, f, indent=1)
    print("wrote", path)
