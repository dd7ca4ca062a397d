"""tests/golden/make_golden_rect_train.py -- golden training samples off the square from the UNMODIFIED reference:
`TrainValDataset.__getitem__` with specific_shape=True (--specific-shape) and with a rect batch_shapes row (--rect), and the
train loader's batches with rect=True (create_dataloader's DataLoader and DistributedSampler over `sort_files_shapes`), and
validation batches with specific_shape=True (`TrainValDataset(augment=False)` as the Evaler and the Trainer's val loader
build it with --specific-shape).
Build container only:

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_rect_train.py

Samples use the seeded dataset of oracle/augment.py and the dataset stand-in of make_golden_augment.py; for specific-shape
cases the stand-in's RAM cache is refilled by the reference's own load_image with specific_shape set.  Loader cases run
the reference's sort_files_shapes on a stand-in whose shapes are fabricated, then the DataLoader with the sampler
create_dataloader builds for a rank of `world`.

Validation cases use the sources and the stand-in of make_golden_valdata.py with specific_shape, target_height and
target_width set.

Writes rect_train_cases.json (per sample case: the SHA-256 of each CHW output; per loader case: each rank's batches as
(dataset indices, canvas); per validation case, in make_golden_valdata.py's format: the loader's source order, each item's
shapes and the SHA-256 of its image) and rect_train.npz (labels_out per sample; labels_out and offsets per validation
case, keys prefixed val_)."""
import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE]
from make_golden_augment import oa, sha256, stand_in  # noqa: E402  (also puts the reference and refshim on sys.path)
import make_golden_valdata as mv  # noqa: E402

import torch  # noqa: E402
from torch.utils.data import DataLoader, Dataset  # noqa: E402
from torch.utils.data.distributed import DistributedSampler  # noqa: E402
from yolov6.data.datasets import TrainValDataset  # noqa: E402

from yolov6_b200.augment import HYP_YOLOV6S  # noqa: E402

# name, hyp overrides, target ("specific" / "rect"), canvas (H, W), img_size, dataset indices, seed
SAMPLE_CASES = [
    ("specific_384x640_mosaic", {}, "specific", (384, 640), 640, [0, 1, 2, 7, 8, 11], 21),
    ("specific_640x384_mosaic", {}, "specific", (640, 384), 640, [1, 4, 5, 9, 12, 13], 22),
    ("specific_384x640_mixup", dict(scale=0.9, mixup=1.0), "specific", (384, 640), 640, [3, 5, 9, 10], 23),
    ("specific_640x384_degrees_shear", dict(degrees=10.0, shear=5.0), "specific", (640, 384), 640, [0, 4, 6, 10], 24),
    ("specific_384x640_letterbox", dict(mosaic=0.0), "specific", (384, 640), 640, [12, 0, 3, 4, 5, 8], 25),
    ("specific_640x384_letterbox_affine", dict(mosaic=0.0, degrees=10.0, shear=5.0), "specific", (640, 384), 640,
     [12, 2, 6, 9, 1, 13], 26),
    ("rect_384x640_mosaic", {}, "rect", (384, 640), 640, [0, 2, 8, 11], 31),
    ("rect_640x448_letterbox", dict(mosaic=0.0), "rect", (640, 448), 640, [1, 4, 12, 7], 32),
    ("rect_640x640_letterbox", dict(mosaic=0.0), "rect", (640, 640), 640, [0, 5, 8, 12], 33),
    ("rect_448x640_mixup", dict(scale=0.9, mixup=1.0), "rect", (448, 640), 640, [3, 6, 9, 13], 34),
]

# name, aspect-ratio family, n images, batch per rank, stride
LOADER_CASES = [(f"{fam}_n{n}_b{b}_s{st}", fam, n, b, st)
                for fam in ("tall", "wide", "mixed") for n, b in ((37, 4), (50, 3)) for st in (32, 64)]
WORLDS = (1, 2, 4)
# name -> (height, width), img_size, batch, stride, rect, pad, shrink_size: the Trainer's val loader (rect, pad 0.5) and the
# Evaler's default (no rect); shrink_size is set in two cases, where load_image ignores it under specific_shape
VAL_CASES = {
    "specific_384x640_rect": ((384, 640), 640, 4, 32, True, 0.5, None),
    "specific_640x384": ((640, 384), 640, 4, 32, False, 0.0, 480),
    "specific_256x320_rect": ((256, 320), 320, 6, 32, True, 0.5, 160),
    "specific_640x480_rect": ((640, 480), 640, 4, 32, True, 0.5, None),     # the 640x480 source loads as it is
}
IMG_SIZE = 640


def fabricated_shapes(fam, n, seed):
    """(h0, w0) of n images whose aspect ratios w0 / h0 are all below 1, all above 1, or both, with ties."""
    r = np.random.RandomState(seed)
    long = r.randint(200, 1400, n)
    ar = {"tall": r.uniform(0.3, 0.99, n), "wide": r.uniform(1.01, 3.0, n), "mixed": r.uniform(0.4, 2.5, n)}[fam]
    ar[::7] = ar[0]                               # ties: argsort's order among equal ratios counts
    w = np.where(ar >= 1, long, np.maximum(1, (long * ar).astype(int)))
    h = np.where(ar >= 1, np.maximum(1, (long / ar).astype(int)), long)
    return [(int(a), int(b)) for a, b in zip(h, w)]


def loader_batches(shapes, batch, stride, world):
    """Each rank's batches from the reference: __init__'s rect branch and sort_files_shapes on a stand-in, then the
    DataLoader create_dataloader builds (DistributedSampler(shuffle=False, drop_last=world > 1) when world > 1)."""
    d = TrainValDataset.__new__(TrainValDataset)
    d.img_size, d.stride, d.pad, d.batch_size, d.cache_ram = IMG_SIZE, stride, 0.0, batch, False
    d.img_paths = list(range(len(shapes)))            # dataset indices stand in for the paths
    d.labels = [None] * len(shapes)
    d.shapes = np.array(shapes, dtype=np.float64)
    sample_batch_size = batch * world                 # datasets.py:89-95 under DDP
    d.batch_indices = np.floor(np.arange(len(shapes)) / sample_batch_size).astype(np.int_)
    d.sort_files_shapes()

    class Items(Dataset):
        def __len__(self):
            return len(d.img_paths)

        def __getitem__(self, index):
            return d.img_paths[index], tuple(int(v) for v in d.batch_shapes[d.batch_indices[index]])

    out = []
    bs = min(batch, len(shapes))
    for rank in range(world):
        sampler = None if world == 1 else DistributedSampler(Items(), num_replicas=world, rank=rank, shuffle=False, drop_last=True)
        dl = DataLoader(Items(), batch_size=bs, shuffle=False, sampler=sampler, num_workers=0, collate_fn=lambda b: b)
        batches = []
        for b in dl:
            canv = {c for _, c in b}
            assert len(canv) == 1, canv                # collate_fn's torch.stack needs one shape per batch
            batches.append([[int(i) for i, _ in b], list(canv.pop())])
        out.append(batches)
    return out


def sample_case(tmp, name, over, target, canvas, img_size, batch, seed, store):
    H, W = canvas
    hyp = dict(HYP_YOLOV6S, **over)
    d, _ = stand_in(tmp, img_size, H, W, hyp)
    if target == "specific":
        d.specific_shape, d.rect, d.cache_ram = True, False, False
        loaded = [d.load_image(i) for i in range(len(oa.DATASET))]       # the reference's load_image at min(W / w0, H / h0)
        d.imgs, d.imgs_hw0, d.imgs_hw = [x[0] for x in loaded], [x[1] for x in loaded], [x[2] for x in loaded]
        d.cache_ram = True
    else:
        d.rect = True
        d.batch_shapes = np.array([[H, W]]).astype(np.int_)               # a numpy row, as sort_files_shapes makes
    random.seed(seed)
    np.random.seed(seed)
    digests = []
    for k, i in enumerate(batch):
        img, labels_out, _, _ = d.__getitem__(i)
        assert tuple(img.shape) == (3, H, W), img.shape
        digests.append(sha256(img.numpy()))
        store[f"{name}_{k}_labels"] = labels_out.numpy()
    print(name, (H, W), [len(store[f"{name}_{k}_labels"]) for k in range(len(batch))])
    return dict(name=name, hyp=hyp, target=target, H=H, W=W, img_size=img_size, batch=batch, seed=seed, chw_sha256=digests)


def val_case(tmp, name, canvas, img_size, batch, stride, rect, pad, shrink, store):
    d = mv.stand_in(tmp, "val", mv.SOURCES, img_size, batch, stride, rect, pad, shrink)
    d.specific_shape, (d.target_height, d.target_width) = True, canvas
    index = {p: i for i, p in enumerate(sorted(d.img_paths))}
    order, shapes, sha, labels = [], [], [], []
    for k in range(len(d.img_paths)):
        img, labels_out, path, sh = d[k]
        assert tuple(img.shape[1:]) == tuple(canvas)
        order.append(index[path])
        (h0, w0), ((rh, rw), (pl, pt)) = sh
        shapes.append([int(h0), int(w0), float(rh), float(rw), int(pl), int(pt)])
        sha.append(sha256(img.numpy()))
        labels.append(labels_out.numpy().astype(np.float32))
    store[f"val_{name}_labels"] = np.concatenate(labels, 0)
    store[f"val_{name}_offsets"] = np.cumsum([0] + [len(x) for x in labels])
    print("val", name, "items", len(order))
    return {"img_size": img_size, "batch": batch, "stride": stride, "rect": rect, "pad": pad, "shrink_size": shrink,
            "specific_shape": list(canvas), "sources": [list(s) for s in mv.SOURCES], "order": order, "shapes": shapes,
            "sha256": sha}


if __name__ == "__main__":
    store, samples, loaders, val = {}, [], [], {}
    with tempfile.TemporaryDirectory() as tmp:
        for case in SAMPLE_CASES:
            samples.append(sample_case(tmp, *case, store))
        for name, case in VAL_CASES.items():
            val[name] = val_case(tmp, name, *case, store)
    for ci, (name, fam, n, b, st) in enumerate(LOADER_CASES):
        shapes = fabricated_shapes(fam, n, 100 + ci)
        for world in WORLDS:
            loaders.append(dict(name=f"{name}_w{world}", shapes=shapes, batch=b, stride=st, world=world, img_size=IMG_SIZE,
                                ranks=loader_batches(shapes, b, st, world)))
    np.savez_compressed(os.path.join(HERE, "rect_train.npz"), **store)
    with open(os.path.join(HERE, "rect_train_cases.json"), "w") as f:
        json.dump(dict(torch=torch.__version__, samples=samples, loaders=loaders, val_cases=val), f, indent=1)
