"""tests/golden/make_golden_valdata.py -- golden validation batches from the UNMODIFIED reference's
TrainValDataset(augment=False) (yolov6/data/datasets.py:166-296, 498-520: sort_files_shapes, load_image, letterbox and
the label code) and the cv2 it calls, on seeded synthetic sources (build container only, CPU).

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_valdata.py

Each source is written as a lossless PNG with its labels; the dataset object is a stand-in built without __init__ (which
would scan a directory and cache image checks): it gets the paths, labels and PIL shapes __init__ would have found, the
Evaler's hyp {"shrink_size": ...}, and for rect=True the reference's own batch_indices expression and sort_files_shapes.
Then __getitem__ runs unchanged for every index and the collate's image index is ignored (column 0 stays 0).

Writes valdata_cases.json (per case: settings, the loader's source order, batch_shapes, each item's shapes and the SHA-256
of its [3, H, W] image; the refusal cases and what the reference raised) and valdata.npz (labels_out of every item,
concatenated per case, with offsets).  The oracle's canvas for each item is checked against the reference's on the way.
"""
import hashlib
import json
import os
import sys
import tempfile
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(HERE, "refshim"), "/root/reference", ROOT]
warnings.filterwarnings("ignore")

import cv2  # noqa: E402
from PIL import Image  # noqa: E402
from yolov6.data.datasets import TrainValDataset  # noqa: E402

from oracle import valdata as ov  # noqa: E402

# (h0, w0) of the shared sources, chosen for the modes they reach at 320 / 640 / 1280:
#   480x640 (2x at 320), 1080x1920 (3x at 640, 6x at 320), 1280x960 (4x at 320), 427x640 (generic, y scale 2.0047 at 320),
#   1000x777, 2000x3000, 641x640 (640 x 639 at 640), 640x512 and 640x480 (r == 1 at 640), 300x400 and 500x500 (INTER_LINEAR
#   at 640 / 1280), 20x1000, 1000x24 and 12x900 (extreme aspect ratios), 360x480 (3x at 160 with shrink).
SOURCES = [(480, 640), (1080, 1920), (1280, 960), (427, 640), (1000, 777), (2000, 3000), (641, 640), (640, 512), (640, 480),
           (300, 400), (500, 500), (20, 1000), (1000, 24), (12, 900), (360, 480)]

# name -> (img_size, batch, stride, rect, pad, shrink_size): every case leaves a partial last batch
CASES = {
    "rect640": (640, 4, 32, True, 0.5, None),
    "rect320": (320, 6, 32, True, 0.5, None),
    "rect1280": (1280, 4, 64, True, 0.5, None),
    "square640": (640, 4, 32, False, 0.0, None),
    "shrink640": (640, 4, 32, True, 0.5, 480),
}

# the fabricated set the metric test runs: 200 sources of COCO-like and odd sizes at img_size 320, batch 32
METRIC_SET = {"name": "metric200", "n": 200, "img_size": 320, "batch": 32, "stride": 32, "seed": 5}

# (h0, w0, img_size, shrink_size): a loaded size that truncates to 0 -- cv2.resize raises, so must yv6's host geometry
REFUSALS = [(10, 4000, 320, None), (480, 640, 640, 640)]


def metric_sources():
    """The (h0, w0) of METRIC_SET's sources: mostly COCO's 640x480 / 480x640 / 427x640 / 640x427, some others."""
    rng = np.random.default_rng(METRIC_SET["seed"])
    common = [(480, 640), (640, 480), (427, 640), (640, 427), (360, 640), (500, 375)]
    out = []
    for _ in range(METRIC_SET["n"]):
        if rng.uniform() < 0.75:
            out.append(common[int(rng.integers(len(common)))])
        else:
            out.append((int(rng.integers(40, 700)), int(rng.integers(40, 700))))
    return out


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def stand_in(tmp, tag, sources, img_size, batch, stride, rect, pad, shrink):
    d = TrainValDataset.__new__(TrainValDataset)
    d.img_size, d.batch_size, d.stride, d.pad, d.rect, d.augment = img_size, batch, stride, pad, rect, False
    d.hyp = {"shrink_size": shrink}
    d.specific_shape, d.cache_ram = False, False
    d.img_paths, labels = [], []
    for i, (h0, w0) in enumerate(sources):
        p = os.path.join(tmp, f"{tag}_{i:03d}.png")
        if not os.path.exists(p):
            cv2.imwrite(p, ov.synthetic_source(h0, w0, i))
        d.img_paths.append(p)
        labels.append(ov.synthetic_labels(i))
    d.labels = labels
    shapes = []
    for p in d.img_paths:
        im = Image.open(p)
        shapes.append((im.height, im.width))            # check_image's (height, width)
    if rect:
        d.shapes = np.array(shapes, dtype=np.float64)
        d.batch_indices = np.floor(np.arange(len(shapes)) / batch).astype(np.int_)
        d.sort_files_shapes()
    return d


def run_case(tmp, tag, sources, img_size, batch, stride, rect, pad, shrink):
    d = stand_in(tmp, tag, sources, img_size, batch, stride, rect, pad, shrink)
    index = {p: i for i, p in enumerate(sorted(d.img_paths))}
    order, shapes, sha, labels, mism = [], [], [], [], 0
    for k in range(len(d.img_paths)):
        img, labels_out, path, sh = d[k]
        i = index[path]
        order.append(i)
        (h0, w0), ((rh, rw), (pl, pt)) = sh
        shapes.append([int(h0), int(w0), float(rh), float(rw), int(pl), int(pt)])
        im = img.numpy()
        sha.append(sha256(im))
        labels.append(labels_out.numpy().astype(np.float32))
        H, W = im.shape[1:]
        src = cv2.imread(path)
        mism += int(not np.array_equal(ov.val_canvas(src, H, W, img_size, shrink), im))
    rec = {"img_size": img_size, "batch": batch, "stride": stride, "rect": rect, "pad": pad, "shrink_size": shrink,
           "sources": [list(s) for s in sources], "order": order, "shapes": shapes, "sha256": sha, "oracle_mismatches": mism}
    if rect:
        rec["batch_shapes"] = np.asarray(d.batch_shapes).astype(int).tolist()
    off = np.cumsum([0] + [len(x) for x in labels])
    return rec, np.concatenate(labels, 0), off


def main():
    out_json, arrays = {"cases": {}, "refusals": []}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (img_size, batch, stride, rect, pad, shrink) in CASES.items():
            rec, lab, off = run_case(tmp, "src", SOURCES, img_size, batch, stride, rect, pad, shrink)
            out_json["cases"][name] = rec
            arrays[f"{name}_labels"], arrays[f"{name}_offsets"] = lab, off
            print(name, "items", len(rec["order"]), "oracle mismatches", rec["oracle_mismatches"], "canvases",
                  sorted({tuple(s) for s in rec.get("batch_shapes", [])}))
        m = METRIC_SET
        rec, lab, off = run_case(tmp, "metric", metric_sources(), m["img_size"], m["batch"], m["stride"], True, 0.5, None)
        out_json["cases"][m["name"]] = rec
        arrays[f"{m['name']}_labels"], arrays[f"{m['name']}_offsets"] = lab, off
        print(m["name"], "oracle mismatches", rec["oracle_mismatches"], "distinct canvases", len({tuple(s) for s in rec["batch_shapes"]}))
        for h0, w0, img_size, shrink in REFUSALS:
            d = TrainValDataset.__new__(TrainValDataset)
            d.img_size, d.augment, d.specific_shape, d.cache_ram = img_size, False, False, False
            p = os.path.join(tmp, f"refuse_{h0}_{w0}.png")
            cv2.imwrite(p, ov.synthetic_source(h0, w0, 0))
            d.img_paths = [p]
            try:
                d.load_image(0, shrink)
                raised = None
            except cv2.error as e:
                raised = type(e).__name__
            out_json["refusals"].append({"h0": h0, "w0": w0, "img_size": img_size, "shrink_size": shrink, "reference_raised": raised})
            print("refusal", h0, w0, img_size, shrink, "->", raised)
    with open(os.path.join(HERE, "valdata_cases.json"), "w") as f:
        json.dump(out_json, f, indent=1)
    np.savez_compressed(os.path.join(HERE, "valdata.npz"), **arrays)


if __name__ == "__main__":
    main()
