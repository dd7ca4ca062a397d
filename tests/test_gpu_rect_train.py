"""Training off the square on the GPU: the augmentation feed in the --specific-shape and --rect modes against the reference's
goldens (tests/golden/make_golden_rect_train.py), every training launch at non-square shapes against float64 (the checks of
test_gpu_forward_launches.py and test_gpu_backward_launches.py, run at those shapes), a single-shape TrainStep at 384 x 640
against the autograd path, and a multi-shape TrainStep against fresh single-shape steps.

Also specific-shape validation canvases (ValFeed) against the reference's SHA-256, and the assignment and loss launches at
640 x 384 and on P6 rect maps against float64.

Bars are the existing ones: loss 1e-4 relative and every gradient 5e-3 relative L2 against the autograd path (fp32 atomics
reorder the accumulation, test_gpu_step.py); a multi-shape step's loss tensor is bit-identical to a fresh step's and its
flat gradient within 1e-5 relative L2 of it (two runs differ only by fp32-atomic reordering, about 1e-7)."""
import hashlib
import random

import numpy as np
import pytest
import torch

import test_gpu_backward_launches as bwd
import test_gpu_forward_launches as fwd
import test_gpu_loss_launches as ll
import test_gpu_valdata as gv
import test_loss_launch_cases as ll_cases
from conftest import golden_json, golden_npz
from oracle import augment as oa
from oracle import fabricate as fab
from oracle import loss as oloss

pytestmark = pytest.mark.gpu

G = golden_json("rect_train_cases.json")
NPZ = golden_npz("rect_train.npz")
SRC = oa.dataset_sources()
LABELS = {i: oa.synthetic_labels(i) for i in SRC}
MAX_SRC = sum(s.nbytes for s in SRC.values())
B = 2


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def feed_of(case, **kw):
    from yolov6_b200.augment import AugmentFeed
    full = (case["img_size"],) * 2 if case["target"] == "rect" else (case["H"], case["W"])
    return AugmentFeed(len(case["batch"]), *full, case["hyp"], len(oa.DATASET), MAX_SRC, case["img_size"],
                       device=torch.device("cuda:0"), target=case["target"], **kw)


def submit_case(feed, case):
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    plan = feed.draw(case["batch"], (case["H"], case["W"]) if case["target"] == "rect" else None)
    targets = feed.submit(plan, SRC, LABELS)
    feed.wait()
    return targets


def check_case(feed, case, targets):
    got = feed.images.cpu().numpy()
    assert got.shape[2:] == (case["H"], case["W"])
    bad = [k for k in range(len(case["batch"])) if sha(got[k]) != case["chw_sha256"][k]]
    assert not bad, f"{case['name']}: samples {bad} differ from the reference"
    ref = []
    for k in range(len(case["batch"])):
        lab = NPZ[f"{case['name']}_{k}_labels"].copy()
        lab[:, 0] = k
        ref.append(lab)
    assert np.array_equal(targets.numpy(), np.concatenate(ref, 0))


@pytest.mark.parametrize("ci", range(len(G["samples"])), ids=[c["name"] for c in G["samples"]])
def test_feed_byte_identical_to_reference(ci):
    case = G["samples"][ci]
    feed = feed_of(case)
    check_case(feed, case, submit_case(feed, case))


def test_one_feed_changes_canvas_between_batches():
    """One rect feed, sized once for 640 x 640, takes the four rect cases in a row: each batch on its own canvas (and with
    its case's augmentation settings)."""
    cases = [c for c in G["samples"] if c["target"] == "rect"]
    feed = feed_of(cases[0])
    for case in cases + cases[:1]:
        feed.sampler.hyp = dict(case["hyp"])
        check_case(feed, case, submit_case(feed, case))


# ---------------------------------------------------------------------------------------------------- specific-shape validation
@pytest.mark.parametrize("how", ["host", "rgb_chw", "mix"])
@pytest.mark.parametrize("name", list(G["val_cases"]))
def test_specific_shape_validation_canvases_equal_the_reference(name, how):
    """ValFeed(specific_shape=(H, W)) through the checks of test_gpu_valdata.py: every canvas's SHA-256, shapes, targets."""
    from oracle import valdata as ov
    from yolov6_b200.valdata import ValFeed
    c = G["val_cases"][name]
    lab, off = NPZ[f"val_{name}_labels"], NPZ[f"val_{name}_offsets"]
    items = [(i, sh, lab[off[k]:off[k + 1]]) for k, (i, sh) in enumerate(zip(c["order"], c["shapes"]))]
    feed = ValFeed(c["batch"], c["img_size"], c["stride"], c["sources"], pad=c["pad"], rect=c["rect"],
                   shrink_size=c["shrink_size"], device=torch.device("cuda:0"), specific_shape=c["specific_shape"])
    sources = [ov.synthetic_source(h0, w0, i) for i, (h0, w0) in enumerate(c["sources"])]
    results = gv.run(c, feed, how, sources)
    assert all(tuple(canvas.shape[2:]) == tuple(c["specific_shape"]) for canvas, *_ in results)
    gv.check_case(c, items, results)


# ---------------------------------------------------------------------------------------------------- launches at rect shapes
LAUNCH_SHAPES = [("yolov6n", 384, 640), ("yolov6n", 640, 384), ("yolov6s", 384, 640), ("yolov6s", 640, 384),
                 ("yolov6m", 384, 640), ("yolov6m", 640, 384), ("yolov6n6", 768, 1280), ("yolov6n6", 1280, 768)]
LAUNCH_IDS = [f"{c}_{h}x{w}" for c, h, w in LAUNCH_SHAPES]


@pytest.fixture
def rect_images(monkeypatch):
    """Makes the launch tests' synthetic image batch H x W whatever square size they ask for."""
    calls = []

    def use(H, W):
        real = fab.synthetic_images

        def images(n, h, w, seed=0):
            calls.append((H, W))
            return real(n, H, W, seed=seed)
        monkeypatch.setattr(fab, "synthetic_images", images)
    yield use
    assert calls, "the launch test planned its engine without the rect image batch"


@pytest.mark.parametrize("cfg,H,W", LAUNCH_SHAPES, ids=LAUNCH_IDS)
def test_training_forward_launches_at_rect_shape(cfg, H, W, rect_images, monkeypatch):
    name = f"{cfg}_{H}x{W}_rect"
    rect_images(H, W)
    monkeypatch.setitem(fwd.TRAIN_CONFIGS, name, (cfg, H, B, False))
    fwd.test_every_training_forward_launch_matches_float64(name)


@pytest.mark.parametrize("cfg,H,W", LAUNCH_SHAPES, ids=LAUNCH_IDS)
def test_training_backward_launches_at_rect_shape(cfg, H, W, rect_images, monkeypatch):
    name = f"{cfg}_{H}x{W}_rect"
    rect_images(H, W)
    monkeypatch.setitem(bwd.MODELS, name, dict(cfg=cfg, size=H, batch=B))
    bwd.test_every_backward_launch_record_matches_float64_autograd(name)


# ---------------------------------------------------------------------------------------------------- assignment and loss launches
# name -> the loss-launch configuration (test_gpu_loss_launches.CONFIGS format) and its det_loss variants: the 640 x 384
# orientation on P5 (384 x 640 is its n_rect), and P6 rect maps in both orientations under both assigner branches
LOSS_RECT = {
    "n_rect_640x384": (dict(strides=ll_cases.P5, R=4, H=640, W=384, assign="tal", topk=13), [("siou", 0, 1.0)]),
    "n6_rect_768x1280_tal": (dict(strides=ll_cases.P6, R=4, H=768, W=1280, assign="tal", topk=13), [("siou", 0, 1.0)]),
    "n6_rect_1280x768_tal": (dict(strides=ll_cases.P6, R=4, H=1280, W=768, assign="tal", topk=13), [("giou", 1, 0.37)]),
    "n6_rect_768x1280_atss": (dict(strides=ll_cases.P6, R=4, H=768, W=1280, assign="atss", topk=9), [("siou", 0, 1.0)]),
    "n6_rect_1280x768_atss": (dict(strides=ll_cases.P6, R=4, H=1280, W=768, assign="atss", topk=9), [("giou", 0, 1.0)]),
}


@pytest.mark.parametrize("name", list(LOSS_RECT))
def test_assignment_and_loss_launches_at_rect_shape(name, monkeypatch):
    """targets_pad, box decode, the assigner (TAL or ATSS), its expansion and det_loss at a rect map, each checked against
    float64 by the checks of test_gpu_loss_launches.py."""
    cfg, variants = LOSS_RECT[name]
    monkeypatch.setitem(ll.CONFIGS, name, cfg)
    monkeypatch.setitem(ll.LOSS_VARIANTS, name, variants)
    ll.test_pad_decode_and_assign_launches(name)
    ll.test_assign_expand_launch(name)
    for iou, ngz, gscale in variants:
        ll.test_det_loss_launch(name, iou, ngz, gscale)


# ---------------------------------------------------------------------------------------------------- TrainStep off the square
def make_model(seed=0, **kw):
    from yolov6_b200.model import build_model
    m = build_model("yolov6n", 80, torch.device("cuda:0"), **kw)
    sd = fab.fabricate_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    for k in sd:
        if (".cls_preds" in k or ".reg_preds" in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
    m.load_state_dict(sd)
    return m.train()


def losses(fuse_ab=False):
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.loss_fuseab import ComputeLoss as ComputeLossAB
    kw = dict(num_classes=80, ori_img_size=640, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    return ComputeLoss(**kw), (ComputeLossAB(**kw) if fuse_ab else None)


def batch(H, W, seed=3):
    return fab.synthetic_images(B, H, W, seed=seed).cuda(), oloss.synthetic_targets(B, seed=seed + 1).cuda()


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def check_grads(ref, flat, what):
    worst = 0.0
    for n, g in ref.items():
        if float(g.norm()) < 1e-12:
            continue
        e = rel(flat.grad_view(n), g)
        worst = max(worst, e)
        assert e < 5e-3, f"{what}: {n}: {e:.3e}"
    return worst


@pytest.mark.parametrize("mode", ["plain", "fuse_ab"])
def test_single_shape_step_matches_autograd_path_at_384x640(mode):
    from yolov6_b200.step import TrainStep
    H, W = 384, 640
    x, targets = batch(H, W)
    fuse_ab = mode == "fuse_ab"
    m1, m2 = make_model(fuse_ab=fuse_ab), make_model(fuse_ab=fuse_ab)
    (c1, c1ab), (c2, c2ab) = losses(fuse_ab), losses(fuse_ab)
    preds, _ = m1(x)
    if fuse_ab:
        l_af, _ = c1((preds[0], preds[3], preds[4]), targets, 0, 0, H, W)
        l_ab, _ = c1ab(preds[:3], targets, 0, 0, H, W)
        loss = l_af + l_ab
    else:
        loss, _ = c1(preds, targets, 0, 0, H, W)
    loss.backward()
    ref = {n: p.grad.detach().clone() for n, p in m1.named_parameters() if p.grad is not None}
    step = TrainStep(m2, c2, B, H, W, max_gt=64, compute_loss_ab=c2ab)
    step.load(x, targets)
    out = step.run(epoch_num=0).clone()
    torch.cuda.synchronize()
    assert abs(float(out[0]) - float(loss)) <= 1e-4 * abs(float(loss)), (float(out[0]), float(loss))
    print(f"{mode} 384x640: worst gradient rel err vs autograd path {check_grads(ref, step.eng.flat, mode):.2e}")


def test_single_shape_distill_step_matches_autograd_path_at_384x640():
    from yolov6_b200 import loss_distill
    from yolov6_b200.step import TrainStep
    H, W, T, MAX_EPOCH, epoch = 384, 640, 20.0, 300, 10
    x, targets = batch(H, W)
    crit = lambda: loss_distill.ComputeLoss(num_classes=80, ori_img_size=640, warmup_epoch=0, use_dfl=False, reg_max=0,  # noqa: E731
                                            iou_type="siou", distill_weight={"class": 1.0, "dfl": 1.0})
    student, teacher, c = make_model(0), make_model(1), crit()
    preds, s_feats = student(x)
    with torch.no_grad():
        t_preds, t_feats = teacher(x)
    loss, _ = c(preds, t_preds, s_feats, t_feats, targets, epoch, MAX_EPOCH, T, 0, H, W)
    loss.backward()
    ref = {n: p.grad.detach().clone() for n, p in student.named_parameters() if p.grad is not None}
    step = TrainStep(make_model(0), crit(), B, H, W, max_gt=64, teacher=make_model(1), temperature=T, max_epoch=MAX_EPOCH)
    step.load(x, targets)
    out = step.run(epoch_num=epoch).clone()
    torch.cuda.synchronize()
    assert abs(float(out[0]) - float(loss)) <= 1e-4 * abs(float(loss)), (float(out[0]), float(loss))
    print(f"distill 384x640: worst gradient rel err vs autograd path {check_grads(ref, step.eng.flat, 'distill'):.2e}")


@pytest.mark.parametrize("mode", ["plain", "fuse_ab"])
def test_multi_shape_step_equals_fresh_single_shape_steps(mode):
    """Shapes A, B, C, A through one step: each step's loss tensor is bit-identical to a fresh single-shape step's from the
    same weights, and its flat gradient is within the tolerance of two runs (the weight-gradient reductions use fp32
    atomics, so their order is not fixed).  The fourth step replays A's graphs: nothing is captured."""
    from yolov6_b200.step import TrainStep
    fuse_ab = mode == "fuse_ab"
    visits = [(384, 640), (640, 384), (640, 640), (384, 640)]
    c, cab = losses(fuse_ab)
    multi = TrainStep(make_model(fuse_ab=fuse_ab), c, B, 640, 640, max_gt=64, compute_loss_ab=cab, shapes=visits[:3])
    captures, report = [], []
    for k, (H, W) in enumerate(visits):
        x, targets = batch(H, W, seed=3 + k)
        multi.load(x, targets)
        got = multi.run(epoch_num=0).clone()
        g_multi = multi.eng.flat.gflat.clone()
        captures.append(multi.captures)
        fc, fcab = losses(fuse_ab)
        fresh = TrainStep(make_model(fuse_ab=fuse_ab), fc, B, H, W, max_gt=64, compute_loss_ab=fcab)
        fresh.load(x, targets)
        want = fresh.run(epoch_num=0).clone()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{mode} {H}x{W} (step {k}): {got.tolist()} vs {want.tolist()}"
        g_fresh = fresh.eng.flat.gflat
        bits = torch.equal(g_multi, g_fresh)
        e = rel(g_multi, g_fresh)
        report.append(f"{H}x{W}: gradient {'bit-identical' if bits else f'rel {e:.2e}'}")
        assert e < 1e-5, f"{mode} {H}x{W}: flat gradient rel {e:.3e}"   # fp32-atomic reordering only: ~1e-7
        del fresh
    assert captures == [1, 2, 3, 3], captures
    print(f"{mode}: " + "; ".join(report))


def test_multi_shape_refusals():
    from yolov6_b200 import loss_distill
    from yolov6_b200.step import TrainStep
    c, _ = losses()
    with pytest.raises(ValueError, match="fit inside"):
        TrainStep(make_model(), c, B, 640, 640, shapes=[(384, 704)])
    crit = loss_distill.ComputeLoss(num_classes=80, ori_img_size=640, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou")
    with pytest.raises(ValueError, match="distillation over several shapes"):
        TrainStep(make_model(0), crit, B, 640, 640, teacher=make_model(1), max_epoch=300, shapes=[(384, 640)])
    step = TrainStep(make_model(), c, B, 640, 640, shapes=[(384, 640)])
    with pytest.raises(ValueError, match="not one of"):
        step.use_shape(640, 384)


def test_feed_switches_a_multi_shape_step():
    """A rect AugmentFeed writes each batch into the step's input view at that batch's canvas; the step trains it as
    TrainStep.load of the same images does."""
    from yolov6_b200.augment import AugmentFeed, HYP_YOLOV6S
    from yolov6_b200.step import TrainStep
    c, _ = losses()
    canvases = [(384, 640), (640, 448), (384, 640)]
    step = TrainStep(make_model(), c, 4, 640, 640, in_dtype=torch.uint8, max_gt=64, shapes=canvases)
    feed = AugmentFeed(4, 640, 640, HYP_YOLOV6S, len(oa.DATASET), MAX_SRC, 640, step=step, target="rect")
    for k, canvas in enumerate(canvases):
        random.seed(50 + k)
        np.random.seed(50 + k)
        plan = feed.draw([0, 2, 8, 11], canvas)
        targets = feed.submit(plan, SRC, LABELS)
        feed.wait()
        assert step.images.shape[2:] == canvas
        imgs = step.images.clone()
        fed = step.run().clone()
        step.load(imgs, targets)
        loaded = step.run().clone()
        assert torch.equal(fed, loaded), (canvas, fed.tolist(), loaded.tolist())
        assert float(fed[0]) > 0
