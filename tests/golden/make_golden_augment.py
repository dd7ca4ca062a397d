"""tests/golden/make_golden_augment.py -- golden training samples from the UNMODIFIED reference
(yolov6/data/datasets.py:166-255 `TrainValDataset.__getitem__`, its `get_mosaic`, `load_image` and `general_augment`, and
data_augment.py) and the cv2 it calls, on the seeded dataset of oracle/augment.py (build container only).

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_augment.py

The dataset object is a stand-in built without __init__ (which would scan a directory): its `cache_ram` slots hold what
the reference's own `load_image` returns for each source written as a PNG, so `__getitem__` runs unchanged.  For each case
`random` and `np.random` are seeded and __getitem__ is called for every index of the batch.  The calls the reference makes
are observed, without changing its draws, to record what it drew: indices loaded, mosaic centres, M and s, the mixup
ratio, the HSV gains and the flips.

Writes augment_cases.json (per case: the drawn parameters and the SHA-256 of each CHW output; the oracle's mismatches
against cv2 for each output, for warpAffine and the HSV round trip on their own, and for HSV -> BGR over the whole
180 x 256 x 256 cube and BGR -> HSV over all 2^24 colours: all must be 0) and augment.npz (labels_out per sample).
"""
import hashlib
import json
import os
import random
import sys
import tempfile
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(HERE, "refshim"), "/root/reference", ROOT]
warnings.filterwarnings("ignore")

import cv2  # noqa: E402
import yolov6.data.data_augment as da  # noqa: E402
import yolov6.data.datasets as ds  # noqa: E402
from yolov6.data.datasets import TrainValDataset  # noqa: E402

from oracle import augment as oa  # noqa: E402
from yolov6_b200.augment import HYP_YOLOV6S, Sampler  # noqa: E402


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def stand_in(tmp, img_size, H, W, hyp):
    d = TrainValDataset.__new__(TrainValDataset)
    d.augment, d.hyp, d.img_size = True, hyp, img_size
    d.specific_shape, d.cache_ram = False, False
    d.rect = H != W
    d.target_height, d.target_width = H, W
    d.batch_shapes, d.batch_indices = np.array([[H, W]]), np.zeros(len(oa.DATASET), np.int64)
    src = oa.dataset_sources()
    d.img_paths = []
    for i in range(len(oa.DATASET)):
        p = os.path.join(tmp, f"{i:03d}.png")
        cv2.imwrite(p, src[i])
        d.img_paths.append(p)
    d.labels = [oa.synthetic_labels(i) for i in range(len(oa.DATASET))]
    loaded = [d.load_image(i) for i in range(len(oa.DATASET))]    # the reference's own load_image, then its RAM cache
    for i, (im, _, _) in enumerate(loaded):
        assert np.array_equal(cv2.imread(d.img_paths[i]), src[i])
    d.imgs = [x[0] for x in loaded]
    d.imgs_hw0 = [x[1] for x in loaded]
    d.imgs_hw = [x[2] for x in loaded]
    d.cache_ram = True
    return d, src


class Recorder:
    """Observes the reference's calls.  Peeks replay a draw from a saved generator state and restore it, so the reference's
    own draws are untouched."""

    def __init__(self, d):
        self.rec = []
        self.d = d
        orig_load, orig_mosaic, orig_gtm, orig_general = d.load_image, ds.mosaic_augmentation, da.get_transform_matrix, TrainValDataset.general_augment
        orig_beta = np.random.beta

        def load_image(index, shrink_size=None):
            self.cur["loaded"].append(int(index))
            return orig_load(index, shrink_size)

        def mosaic_augmentation(shape, *a, **k):
            st = random.getstate()
            th, tw = (shape if isinstance(shape, (list, np.ndarray)) else (shape, shape))
            yc, xc = (int(random.uniform(x // 2, 3 * x // 2)) for x in (th, tw))
            random.setstate(st)
            self.cur["centres"].append([yc, xc])
            return orig_mosaic(shape, *a, **k)

        def get_transform_matrix(*a, **k):
            M, s = orig_gtm(*a, **k)
            self.cur["M"].append(M.tolist())
            self.cur["s"].append(float(s))
            return M, s

        def beta(a, b, size=None):
            r = orig_beta(a, b, size)
            self.cur["mix_r"] = float(r)
            return r

        def general_augment(obj, img, labels):
            h = obj.hyp
            st, nst = random.getstate(), np.random.get_state()
            if h["hsv_h"] or h["hsv_s"] or h["hsv_v"]:
                self.cur["gains"] = (np.random.uniform(-1, 1, 3) * [h["hsv_h"], h["hsv_s"], h["hsv_v"]] + 1).tolist()
            self.cur["flipud"] = random.random() < h["flipud"]
            self.cur["fliplr"] = random.random() < h["fliplr"]
            random.setstate(st)
            np.random.set_state(nst)
            return orig_general(obj, img, labels)

        d.load_image = load_image
        ds.mosaic_augmentation = mosaic_augmentation
        da.get_transform_matrix = get_transform_matrix
        np.random.beta = beta
        TrainValDataset.general_augment = general_augment

    def get(self, index):
        self.cur = dict(index=int(index), loaded=[], centres=[], M=[], s=[], mix_r=None, gains=None)
        img, labels_out, _, _ = self.d.__getitem__(index)
        self.rec.append(self.cur)
        return img.numpy(), labels_out.numpy()


def color_checks():
    """Exhaustive: BGR -> HSV over all 2^24 colours, HSV -> BGR over every hue < 180 and all s, v, in 1024-pixel rows
    (OpenCV's vector path, which every row of a width that is a multiple of 32 takes)."""
    c = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([c & 255, (c >> 8) & 255, c >> 16], -1).astype(np.uint8).reshape(-1, 1024, 3)
    bad_fwd = int((cv2.cvtColor(bgr, cv2.COLOR_BGR2HSV) != oa.bgr_to_hsv(bgr)).any(-1).sum())
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([h, s, v], -1).astype(np.uint8).reshape(-1, 1024, 3)
    bad_inv = int((cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR) != oa.hsv_to_bgr(hsv)).any(-1).sum())
    return bad_fwd, bad_inv


if __name__ == "__main__":
    bad_fwd, bad_inv = color_checks()
    print("BGR->HSV mismatches over 2^24 colours:", bad_fwd, " HSV->BGR mismatches over 180x256x256:", bad_inv)
    store, cases = {}, []
    ref_gtm, ref_mosaic, ref_general, ref_beta = da.get_transform_matrix, ds.mosaic_augmentation, TrainValDataset.general_augment, np.random.beta
    with tempfile.TemporaryDirectory() as tmp:
        for ci, (name, over, H, W, img_size, batch, seed) in enumerate(oa.CASES):
            hyp = dict(HYP_YOLOV6S, **over)
            d, src = stand_in(tmp, img_size, H, W, hyp)
            rec = Recorder(d)
            random.seed(seed)
            np.random.seed(seed)
            outs = [rec.get(i) for i in batch]
            da.get_transform_matrix, ds.mosaic_augmentation, TrainValDataset.general_augment, np.random.beta = ref_gtm, ref_mosaic, ref_general, ref_beta
            # the oracle on the host sampler's records for the same seeds
            random.seed(seed)
            np.random.seed(seed)
            plan = Sampler(len(oa.DATASET), H, W, hyp, img_size).draw(batch)
            digests, mism, warp_mism, hsv_mism = [], [], [], []
            for k, ((img, lab), r) in enumerate(zip(outs, plan.samples)):
                assert img.shape == (3, H, W), img.shape
                mine = oa.compose(r, src, H, W, img_size)
                mism.append(int((mine != img).any(0).sum()))
                digests.append(sha256(img))
                store[f"{name}_{k}_labels"] = lab
                # warpAffine and the HSV round trip on their own, on this sample's first canvas
                cv = r.canvases[0]
                imgs = [oa.load_resized(src[i], img_size) for i in cv.indices]
                canvas = oa.mosaic_canvas(imgs, cv.yc, cv.xc, H, W) if r.mosaic else oa.letterbox_canvas(imgs[0], H, W)
                ref_w = cv2.warpAffine(canvas, cv.M[:2], dsize=(W, H), borderValue=(114, 114, 114))
                warp_mism.append(int((ref_w != oa.warp_affine(canvas, cv.M, W, H)).any(-1).sum()))
                if r.gains is not None:      # augment_hsv's cv2 calls (data_augment.py:17-26) with the drawn gains
                    lh, ls, lv = oa.hsv_luts(r.gains)
                    hue, sat, val = cv2.split(cv2.cvtColor(ref_w, cv2.COLOR_BGR2HSV))
                    ref_h = cv2.cvtColor(cv2.merge((cv2.LUT(hue, lh), cv2.LUT(sat, ls), cv2.LUT(val, lv))), cv2.COLOR_HSV2BGR)
                    hsv_mism.append(int((ref_h != oa.augment_hsv(ref_w, r.gains)).any(-1).sum()))
            print(ci, name, (H, W), "mosaic" if plan.samples[0].mosaic else "letterbox",
                  "mixup", sum(s.mix_r is not None for s in plan.samples), "oracle mismatches", mism, "warp", warp_mism, "hsv", hsv_mism)
            cases.append(dict(name=name, hyp=hyp, H=H, W=W, img_size=img_size, batch=batch, seed=seed, draws=rec.rec,
                              chw_sha256=digests, oracle_mismatch=mism, warp_mismatch=warp_mism, hsv_mismatch=hsv_mism))
    np.savez_compressed(os.path.join(HERE, "augment.npz"), **store)
    with open(os.path.join(HERE, "augment_cases.json"), "w") as f:
        json.dump(dict(cv2=cv2.__version__, bgr2hsv_mismatch=bad_fwd, hsv2bgr_mismatch=bad_inv,
                       dataset=[list(x) for x in oa.DATASET], cases=cases), f, indent=1)
