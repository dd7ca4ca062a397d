"""The captured training step (step.TrainStep: CUDA graph, weight gradients on the side stream) started on poisoned memory,
against a serial eager step of the same engine on clean memory.

The backward pass does not clear the gradient buffers: the first writer of each channel slice assigns and later writers add
(train._resolve_first_writers), and weight gradients run on a side stream that reads one dc scratch pair while the main
stream refills the other (train.TrainEngine.backward).  Both are right only if no launch reads memory before this step
wrote it.  Here, for YOLOv6-S at 640, batch 32, uint8 input and YOLOv6-M at 640, batch 8 (the shapes bench.py trains), and
for N-QA and N with the neck outputs as differentiable outputs (external_feat_grads) at 128 px:
  * reference: one eager step with overlap_wgrad = False on clean memory; the flat gradient buffer, the loss items and the
    flat parameter buffer (the updated running statistics) are kept on the host;
  * compared run: a TrainStep with the graph and the side stream on, on the same weights, batch and targets.  After its graph
    is captured, the parameter buffer is put back to its state before the step, and every tensor the step writes before it
    reads is poisoned: activations, gradient buffers, dc / quadrant / pool scratch, head tensors and their gradients,
    statistics and coefficients, patches, QA and fuse_ab tensors and the flat gradient buffer hold 2^100, the zero arena
    holds bytes 0x7e (about 8e37 as fp32, 1e303 as float64).  Then the graph replays once.
The gradient of every parameter slot, the loss items and every slot of the parameter buffer must match the reference: a
read of poisoned memory puts about 1e25 (or inf / NaN) into some slot.  Weight gradients and the BatchNorm sums use float
atomics, so two serial steps are not bit-identical: the test measures that noise floor (two serial steps on the same
engine) and the bar is 8 x the floor, at least 1e-6, per slot as relative L2 error.  Measured on an H100 80GB HBM3 (700 W
power limit), the worst slot's floor was 6.2e-7 for S at 640 batch 32, 5.2e-7 for M at 640 batch 8, 0.9e-7 and 1.6e-7 for
N-QA and N at 128 px; the poisoned captured step differed from the serial one by 8.7e-7, 5.8e-7, 0.9e-7 and 1.1e-7, the
loss items and the parameter buffer (running statistics) not at all.

The 4-element pads of the flat gradient buffer (every slot starts on a 16-byte boundary) are never written by a step: the
gradient unpack covers the slots only, and the pads keep the zeros FlatState allocated.  The fused SGD reads them (it works
on float4 lanes), but lane by lane, so a pad value only reaches the pad lanes of the parameter, momentum and EMA buffers,
which no view of any parameter covers.  The test checks that the pads still hold the poison after the step, and that every
slot matched the reference regardless (YOLOv6-S and -N have no pad elements; M has 72).

N with distill_ns is not among the configurations: TrainStep computes no distillation loss, so in a TrainStep nothing
writes the gradient of the distillation head's extra output, and its first-writer plan is pinned by tests/test_train_plan.py.

Harness (test_poisoned_step_catches_a_first_writer_that_accumulates): one bn_bwd that assigns a gradient slice as its first
writer is made to add to it instead; the compared run must then be off by more than 1e10."""
import gc

import pytest
import torch

import test_gpu_backward_launches as bwd
from conftest import golden_keys
from oracle import fabricate as fab
from oracle import loss as oloss

pytestmark = pytest.mark.gpu

ARENA_POISON = 0x7E
# name -> model config, image size, batch, uint8 input, external_feat_grads
CONFIGS = {
    "yolov6s_640_b32_u8": ("yolov6s", 640, 32, True, False), "yolov6m_640_b8": ("yolov6m", 640, 8, False, False),
    "yolov6n_qa_128": ("yolov6n_qa", 128, 2, False, False), "yolov6n_feat_128": ("yolov6n", 128, 2, False, True),
}


def make(cfg, size, feat):
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    m = build_model(cfg, 80, torch.device("cuda:0"))
    if cfg in bwd.GOLDEN_KEYS:
        sd = fab.fabricate_state_dict(golden_keys(cfg), seed=0)
        for k in sd:                 # moderate head logits, as tests/test_gpu_step.py
            if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
                sd[k] = sd[k] * 0.1
        m.load_state_dict(sd)
    else:
        randomize_(m, seed=0)
    m.train()
    eng = m.train_engine(n_buckets=1)
    eng.external_feat_grads = feat
    g = m.graph
    dfl = bool(g.use_dfl and g.reg_max)
    loss = ComputeLoss(num_classes=80, ori_img_size=size, warmup_epoch=0, use_dfl=dfl, reg_max=g.reg_max if dfl else 0,
                       iou_type="giou" if dfl else "siou")
    return m, loss


def batch(size, n, u8):
    x = fab.synthetic_images(n, size, size, seed=5)
    if u8:
        x = (x * 255).round().to(torch.uint8)
    return x.cuda(), oloss.synthetic_targets(n, seed=6).cuda()


def poison(eng):
    mem = bwd.engine_mem(eng)
    for _, _, tag, t in mem.ts:
        if tag == "arena":
            t.fill_(ARENA_POISON)
        elif tag not in bwd.REST_EXEMPT:
            t.fill_(bwd.SENTINEL)


def slot_errors(fl, got_g, want_g, got_p, want_p):
    """Worst relative L2 error over the gradient slots and over the parameter-buffer slots (NaN counts as infinite)."""
    def worst(got, want, slots):
        w = 0.0
        for o, k, _ in slots:
            a, b = got[o:o + k].double(), want[o:o + k].double()
            e = float((a - b).norm() / (b.norm() + 1e-30))
            w = max(w, e if e == e else float("inf"))
        return w
    grads = [fl.slots[n] for n in fl.names]
    return worst(got_g, want_g, grads), worst(got_p, want_p, list(fl.slots.values()))


def serial_reference(name, repeat=2):
    """Eager steps with the weight gradients on the main stream, from the same state each time: [(gflat, loss items, pflat)]."""
    from yolov6_b200.step import TrainStep
    cfg, size, n, u8, feat = CONFIGS[name]
    m, loss = make(cfg, size, feat)
    x, t = batch(size, n, u8)
    step = TrainStep(m, loss, n, size, size, in_dtype=torch.uint8 if u8 else torch.float32, graph=False)
    step.eng.overlap_wgrad = False
    fl = step.eng.flat
    p0, i0 = fl.pflat.clone(), fl.iflat.clone()
    out = []
    for _ in range(repeat):
        fl.pflat.copy_(p0)
        fl.iflat.copy_(i0)
        step.load(x, t)
        items = step.run(epoch_num=1)[:4].clone()
        torch.cuda.synchronize()
        out.append((fl.gflat.cpu(), items.cpu(), fl.pflat.cpu()))
    del step, m
    gc.collect()
    torch.cuda.empty_cache()
    return out


def poisoned_run(name, flip=False):
    """The captured step with the side stream, replayed on poisoned memory.  `flip`: the first gradient slice a bn_bwd
    assigns as its first writer is accumulated into instead (harness check).  Returns (gflat, loss items, pflat, pads still poisoned)."""
    from yolov6_b200.step import TrainStep
    cfg, size, n, u8, feat = CONFIGS[name]
    m, loss = make(cfg, size, feat)
    x, t = batch(size, n, u8)
    step = TrainStep(m, loss, n, size, size, in_dtype=torch.uint8 if u8 else torch.float32, graph=True)
    eng = step.eng
    assert eng.overlap_wgrad, "the side stream is off (YV6_WGRAD_OVERLAP=0)"
    if flip:                 # the first first-writer slice of a bn_bwd: assign(False) changes nothing on an accumulating write
        def state(d):
            return list(d.accumulate), d.dres_assign
        flipped = False
        for c in (c for c in eng.bwd_calls if c.kind == "bn_bwd"):
            for w in c.writes:
                before = state(c.desc)
                w.assign(False)
                if state(c.desc) != before:
                    flipped = True
                    break
            if flipped:
                break
        assert flipped, "no bn_bwd assigns a gradient slice"
    fl = eng.flat
    p0, i0 = fl.pflat.clone(), fl.iflat.clone()
    step.load(x, t)
    step.run(epoch_num=1)                          # captures the graph (and replays it once)
    torch.cuda.synchronize()
    fl.pflat.copy_(p0)
    fl.iflat.copy_(i0)
    poison(eng)
    fl.gflat.fill_(bwd.SENTINEL)
    step.load(x, t)
    items = step.run(epoch_num=1)[:4].clone()
    torch.cuda.synchronize()
    pads = torch.ones(fl.n_train, dtype=torch.bool, device=fl.gflat.device)
    for o, k, _ in (fl.slots[nm] for nm in fl.names):
        pads[o:o + k] = False
    pads_kept = bool((fl.gflat[pads] == bwd.SENTINEL).all())
    out = (fl.gflat.cpu(), items.cpu(), fl.pflat.cpu(), pads_kept, int(pads.sum()))
    del step, eng, m
    gc.collect()
    torch.cuda.empty_cache()
    return out, fl


def items_error(got, want):
    e = float(((got - want).abs() / want.abs().clamp_min(1e-30)).max())
    return e if e == e else float("inf")


@pytest.mark.parametrize("name", list(CONFIGS))
def test_captured_step_on_poisoned_memory_matches_a_serial_step(name):
    (g0, it0, p0), (g1, it1, p1) = serial_reference(name)
    (g, it, p, pads_kept, npads), fl = poisoned_run(name)
    floor_g, floor_p = slot_errors(fl, g1, g0, p1, p0)
    floor = max(floor_g, floor_p, items_error(it1, it0))
    bar = max(8 * floor, 1e-6)
    err_g, err_p = slot_errors(fl, g, g0, p, p0)
    err_i = items_error(it, it0)
    print(f"\n{name}: noise floor of two serial steps {floor:.2e} (gradients {floor_g:.2e}, parameter buffer {floor_p:.2e}); "
          f"poisoned captured step: gradients {err_g:.2e}, loss items {err_i:.2e}, parameter buffer {err_p:.2e}, bar {bar:.2e}; "
          f"{npads} gradient pad elements kept the poison: {pads_kept}")
    assert floor <= 1e-4, f"two serial steps differ by {floor:.2e}: not rounding noise"
    assert err_g <= bar, f"gradients differ from the serial step by {err_g:.2e} (bar {bar:.2e})"
    assert err_i <= bar, f"loss items differ by {err_i:.2e}"
    assert err_p <= bar, f"parameter buffer (running statistics) differs by {err_p:.2e}"
    assert pads_kept, "a step wrote the pads of the flat gradient buffer"


def test_poisoned_step_catches_a_first_writer_that_accumulates():
    """Harness: one shortcut-gradient slice whose first writer adds to the buffer instead of assigning reads the poison."""
    name = "yolov6n_feat_128"
    (g0, it0, p0), = serial_reference(name, repeat=1)
    (g, it, p, _, _), fl = poisoned_run(name, flip=True)
    err_g, _ = slot_errors(fl, g, g0, p, p0)
    assert err_g > 1e10, f"an accumulating first writer went unnoticed (gradient error {err_g:.2e})"
