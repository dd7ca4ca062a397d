"""The self-distillation recipe in the CUDA-graph TrainStep (step.py, `teacher=`) against the compatible autograd path on the same
batch: student(x), teacher(x) under no_grad, loss_distill.ComputeLoss[NS], loss.backward() (core/engine.py:153-159).

Bars: loss and the items (iou, dfl, cls, cwd) 1e-4 relative; every student gradient 5e-3 relative L2 (the bar of
test_gpu_fuseab.py::test_fuseab_train_step_graph_equals_autograd_path: fp32 atomics reorder the accumulation); the teacher's
head tensors 1e-4 relative L2 (same kernels, but the BatchNorm sums are float64 atomics, so a bf16 activation can differ by one
rounding step)."""
import math

import numpy as np
import pytest
import torch

from oracle import fabricate as fab
from oracle import loss as oloss

pytestmark = pytest.mark.gpu

B, T, MAX_EPOCH = 2, 20.0, 300


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def make_model(cfg, seed, **kw):
    """A training-mode model with fabricated weights (pred weights scaled by 0.1, as in test_gpu_fuseab.py)."""
    from yolov6_b200.model import build_model
    m = build_model(cfg, 80, torch.device("cuda:0"), **kw)
    sd = fab.fabricate_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    for k in sd:
        if (".cls_preds" in k or ".reg_preds" in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
    m.load_state_dict(sd)
    return m.train()


def ns_cfg():
    from yolov6_b200 import configs
    cfg = configs.get_config("yolov6n")
    cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16       # the N / S recipe, as test_gpu_fuseab.py:209-210
    return cfg


# recipe -> (student config and options, teacher options, loss class, loss options, image size)
RECIPES = {
    "ns": (ns_cfg, dict(distill_ns=True), dict(fuse_ab=True), "ComputeLossNS",
           dict(warmup_epoch=0, use_dfl=True, reg_max=16, iou_type="siou"), 128),
    "m_feat": (lambda: "yolov6m", {}, dict(fuse_ab=True), "ComputeLoss",
               dict(warmup_epoch=0, use_dfl=True, reg_max=16, iou_type="giou", distill_feat=True), 128),
    "n6": (lambda: "yolov6n6", {}, {}, "ComputeLoss",
           dict(fpn_strides=[8, 16, 32, 64], warmup_epoch=4, use_dfl=False, reg_max=0, iou_type="siou"), 256),
}


def recipe(name):
    from yolov6_b200 import loss_distill
    cfg, s_kw, t_kw, loss_cls, loss_kw, S = RECIPES[name]
    crit = lambda: getattr(loss_distill, loss_cls)(num_classes=80, ori_img_size=S, distill_weight={"class": 1.0, "dfl": 1.0},  # noqa: E731
                                                   **loss_kw)
    # teacher weights of their own seed: with the student's, the class KL and channel-wise terms would vanish
    return (lambda: make_model(cfg(), 0, **s_kw)), (lambda: make_model(cfg(), 1, **t_kw)), crit, S


def batch(S):
    return fab.synthetic_images(B, S, S, seed=3).cuda(), oloss.synthetic_targets(B, seed=4).cuda()


def compatible_path(name, epoch):
    """loss, items, student gradients and the teacher's (scores, distributions) of the autograd path."""
    student_f, teacher_f, crit_f, S = recipe(name)
    student, teacher, crit = student_f(), teacher_f(), crit_f()
    x, targets = batch(S)
    feat = crit.distill_feat
    student.return_featmaps = teacher.return_featmaps = feat
    preds, s_feats = student(x)
    with torch.no_grad():
        t_preds, t_feats = teacher(x)
    loss, items = crit(preds, t_preds, s_feats, t_feats, targets, epoch, MAX_EPOCH, T, 0, S, S)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().clone() for n, p in student.named_parameters() if p.grad is not None}
    return float(loss.detach()), items.cpu().double().numpy(), grads, (t_preds[-2].detach().clone(), t_preds[-1].detach().clone())


def distill_step(name, graph=True, **kw):
    from yolov6_b200.step import TrainStep
    student_f, teacher_f, crit_f, S = recipe(name)
    x, targets = batch(S)
    step = TrainStep(student_f(), crit_f(), B, S, S, max_gt=64, graph=graph, teacher=teacher_f(), temperature=T, max_epoch=MAX_EPOCH, **kw)
    step.load(x, targets)
    return step


def items_of(out):
    return out[[1, 2, 3, 6]].cpu().double().numpy()


def check_against_compatible(name, step, out, epoch):
    loss, items, grads, (t_cls, t_reg) = compatible_path(name, epoch)
    got = float(out[0])
    print(f"{name} epoch {epoch}: step loss {got} vs compatible path {loss}; items {items_of(out)} vs {items}")
    assert abs(got - loss) <= 1e-4 * abs(loss)
    np.testing.assert_allclose(items_of(out), items, rtol=1e-4, atol=1e-9)
    fl, worst = step.eng.flat, 0.0
    for n, g in grads.items():
        if float(g.norm()) < 1e-12:
            continue
        e = rel(fl.grad_view(n), g)
        worst = max(worst, e)
        assert e < 5e-3, f"{name}: {n}: {e:.3e}"
    e_cls, e_reg = rel(step.teng.cls, t_cls), rel(step.teng.reg, t_reg)
    print(f"{name}: worst gradient rel err {worst:.2e}; teacher heads rel err {e_cls:.2e} / {e_reg:.2e}")
    assert e_cls < 1e-4 and e_reg < 1e-4
    return grads


@pytest.mark.parametrize("name,epoch", [("ns", 10), ("m_feat", 10), ("n6", 2)])
def test_distill_step_matches_compatible_path(name, epoch):
    """(a) N / S recipe: distill_ns student, fuse_ab teacher, ComputeLossNS.  (b) M student with feature distillation: the
    neck-output gradients reach the student's backward.  (c) N6 student and plain N6 teacher at an ATSS epoch: four levels,
    class KL only (no DFL)."""
    step = distill_step(name)
    out = step.run(epoch_num=epoch).clone()
    torch.cuda.synchronize()
    assert not step.overflowed()
    if name == "m_feat":
        assert float(out[6]) > 0
    check_against_compatible(name, step, out, epoch)


def test_kl_decay_follows_the_epoch():
    """(d) epoch 0 then 150 of 300 on one step object and batch: each matches the compatible path at its epoch, the graphs were
    recaptured, and the class-KL terms are in the ratio of the decays (loss_distill.py:196)."""
    step = distill_step("ns")
    fl = step.eng.flat
    saved = fl.pflat.clone(), fl.iflat.clone()
    kl = {}
    for epoch in (0, 150):
        fl.pflat.copy_(saved[0])
        fl.iflat.copy_(saved[1])
        out = step.run(epoch_num=epoch).clone()
        torch.cuda.synchronize()
        assert list(step.graphs) == [(False, epoch)]
        kl[epoch] = float(step.state["keep_distill"][2][0])
        check_against_compatible("ns", step, out, epoch)
    decay = lambda e: ((1 - math.cos(e * math.pi / MAX_EPOCH)) / 2) * (0.01 - 1) + 1      # noqa: E731
    print("class KL at epochs 0 / 150:", kl, "decay ratio", decay(150) / decay(0))
    assert kl[0] > 0 and abs(kl[150] / kl[0] - decay(150) / decay(0)) <= 1e-6


def test_teacher_is_frozen_and_student_statistics_move_as_in_plain_step():
    """(e) Three steps, the capture warm-ups included, leave every teacher tensor bit-identical; the student's running
    statistics and batch counters end where a plain TrainStep's do."""
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.step import TrainStep
    student_f, teacher_f, crit_f, S = recipe("ns")
    x, targets = batch(S)
    teacher = teacher_f()
    before = {k: v.detach().clone() for k, v in teacher.state_dict().items()}
    step = TrainStep(student_f(), crit_f(), B, S, S, max_gt=64, teacher=teacher, temperature=T, max_epoch=MAX_EPOCH)
    plain = TrainStep(student_f(), ComputeLoss(num_classes=80, ori_img_size=S, warmup_epoch=0, use_dfl=False, reg_max=0, iou_type="siou"),
                      B, S, S, max_gt=64)
    for s in (step, plain):
        s.load(x, targets)
        for _ in range(3):
            s.run(epoch_num=10)
    torch.cuda.synchronize()
    after = teacher.state_dict()
    for k, v in before.items():
        assert torch.equal(after[k], v), f"teacher {k} changed"
    init = student_f().state_dict()
    got, want = step.model.state_dict(), plain.model.state_dict()
    for k in want:
        if k.endswith("num_batches_tracked"):
            assert int(got[k]) == int(want[k]) == 3, k
        elif k.endswith(("running_mean", "running_var")):
            assert rel(got[k], want[k]) < 1e-4, k
            assert not torch.equal(got[k], init[k]), f"student {k} did not move"


def test_eager_step_matches_graph_step():
    """(f) graph=False gives the graph step's loss and its gradients within the bar of (a)."""
    g_step, e_step = distill_step("ns", graph=True), distill_step("ns", graph=False)
    g_out, e_out = g_step.run(epoch_num=10).clone(), e_step.run(epoch_num=10).clone()
    torch.cuda.synchronize()
    assert abs(float(e_out[0]) - float(g_out[0])) <= 1e-4 * abs(float(g_out[0]))
    np.testing.assert_allclose(items_of(e_out), items_of(g_out), rtol=1e-4, atol=1e-9)
    worst = 0.0
    for n in g_step.eng.flat.names:
        g = g_step.eng.flat.grad_view(n)
        if float(g.norm()) < 1e-12:
            continue
        e = rel(e_step.eng.flat.grad_view(n), g)
        worst = max(worst, e)
        assert e < 5e-3, f"{n}: {e:.3e}"
    print("eager vs graph distillation step: worst gradient rel err", worst)
