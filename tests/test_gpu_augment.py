"""GPU parity of the training augmentation (yv6_aug_resize, yv6_augment, AugmentFeed) against the reference's goldens
(tests/golden/augment_cases.json: digests of __getitem__'s CHW outputs; tests/golden/augment.npz: its labels_out), and of
a TrainStep fed by AugmentFeed against the same step loaded with the oracle's batch."""
import hashlib
import random

import numpy as np
import pytest
import torch

from conftest import golden_json, golden_keys, golden_npz
from oracle import augment as oa
from oracle import fabricate as fab

pytestmark = pytest.mark.gpu

G = golden_json("augment_cases.json")
NPZ = golden_npz("augment.npz")
SRC = oa.dataset_sources()
LABELS = {i: oa.synthetic_labels(i) for i in SRC}
MAX_SRC = sum(s.nbytes for s in SRC.values())


def feed_for(case, **kw):
    from yolov6_b200.augment import AugmentFeed
    return AugmentFeed(len(case["batch"]), case["H"], case["W"], case["hyp"], len(oa.DATASET), MAX_SRC, case["img_size"],
                       device=torch.device("cuda:0"), **kw)


def seeded_plan(feed, case):
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    return feed.draw(case["batch"])


@pytest.mark.parametrize("ci", range(len(oa.CASES)))
def test_feed_byte_identical_to_reference(ci):
    """Each golden case is one batch: its sources have mixed sizes, and the two launches serve all of them."""
    case = G["cases"][ci]
    feed = feed_for(case)
    plan = seeded_plan(feed, case)
    targets = feed.submit(plan, SRC, LABELS)
    feed.wait()
    got = feed.images.cpu().numpy()
    for k, rec in enumerate(plan.samples):
        if hashlib.sha256(np.ascontiguousarray(got[k]).tobytes()).hexdigest() != case["chw_sha256"][k]:
            ref = oa.compose(rec, SRC, case["H"], case["W"], case["img_size"])      # carries the golden digest (CPU test)
            diff = np.abs(got[k].astype(np.int64) - ref.astype(np.int64))
            pytest.fail(f"{case['name']} sample {k}: {int((diff > 0).sum())} bytes differ, max {int(diff.max())}")
    ref_t = []
    for k in range(len(case["batch"])):
        lab = NPZ[f"{case['name']}_{k}_labels"].copy()
        lab[:, 0] = k
        ref_t.append(lab)
    ref_t = np.concatenate(ref_t, 0)
    assert np.array_equal(targets.numpy(), ref_t)
    n = ref_t.shape[0]
    dev_t = feed.targets.cpu().numpy()
    assert np.array_equal(dev_t[:n], ref_t) and (dev_t[n:] == -1).all()


def test_feed_drives_trainstep_like_load():
    """Two steps of a TrainStep fed by AugmentFeed return the same loss tensor as TrainStep.load with the oracle's batch."""
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.step import TrainStep
    from yolov6_b200.augment import AugmentFeed
    H = W = 256
    B = 4
    hyp = dict(G["cases"][1]["hyp"], mixup=0.5)
    sd = fab.fabricate_state_dict(golden_keys("yolov6n"), seed=0)
    m = build_model("yolov6n", 80, torch.device("cuda:0"))
    m.load_state_dict(sd)
    crit = ComputeLoss(num_classes=80, ori_img_size=H, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    step = TrainStep(m.train(), crit, B, H, W, in_dtype=torch.uint8)
    feed = AugmentFeed(B, H, W, hyp, len(oa.DATASET), MAX_SRC, step=step)
    for it, batch in enumerate(([0, 1, 2, 3], [8, 11, 12, 13])):
        random.seed(40 + it)
        np.random.seed(40 + it)
        plan = feed.draw(batch)
        targets = feed.submit(plan, SRC, LABELS)
        feed.wait()
        fed = step.run().clone()
        imgs = torch.from_numpy(np.stack([oa.compose(r, SRC, H, W, H) for r in plan.samples])).pin_memory()
        step.load(imgs, targets)
        loaded = step.run().clone()
        assert torch.equal(fed, loaded), (it, fed.tolist(), loaded.tolist())
        assert float(fed[0]) > 0


def test_bad_input_raises_before_enqueue():
    case = G["cases"][2]
    feed = feed_for(case)
    plan = seeded_plan(feed, case)
    i = plan.sources[0]
    bad = [
        ({**SRC, i: SRC[i].astype(np.float32)}, LABELS),                 # not uint8
        ({**SRC, i: SRC[i][..., :2]}, LABELS),                           # 2 channels
        ({**SRC, i: SRC[i][..., 0]}, LABELS),                            # not HWC
        ({k: v for k, v in SRC.items() if k != i}, LABELS),              # missing source
        (SRC, {**LABELS, i: np.zeros((2, 4), np.float32)}),              # malformed label rows
        (SRC, {**LABELS, i: np.array([[0, 0.5, 0.5, 1.5, 0.1]], np.float32)}),
    ]
    for frames, labels in bad:
        with pytest.raises(RuntimeError):
            feed.submit(plan, frames, labels)
    from yolov6_b200.augment import AugmentFeed
    small = AugmentFeed(len(case["batch"]), case["H"], case["W"], case["hyp"], len(oa.DATASET), 100, case["img_size"])
    with pytest.raises(RuntimeError, match="max_src_bytes"):
        small.submit(plan, SRC, LABELS)
    assert feed.ready is None and small.ready is None
    with pytest.raises(RuntimeError):
        feed.draw(case["batch"] + [0])
