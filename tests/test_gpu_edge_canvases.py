"""Every launch against float64 on degenerate canvases: top-level maps one pixel tall, wide or both, 32- and 64-pixel
strips, and head levels with fewer anchors than ATSS's per-level top-k.

The engine takes any H and W that are multiples of the largest stride, and real callers make such shapes: letterbox
auto=True of a 100 x 2000 panorama at img_size 640 gives a 32 x 640 canvas (P5 1 x 20), a validation batch of aspect
1:20 a 64 x 640 canvas, rect training a 32 x 640 one, and a 32 x 32 image gives 1 x 1 P5 maps.  There the conv's halo box
is clipped at the top and bottom at once, every M tile has a dead upper half, TMA boxes are larger than the tensor, the
SPPF pool's vertical taps are all padding, SE averages 2 x 2 pixels (the Lite graph's smallest map), a head level has one
anchor, BatchNorm statistics run over batch x 1 x 1 pixels and ATSS picks min(topk, 1) anchors of a level.
tests/test_edge_canvas_coverage.py proves on the CPU that the configurations below reach those edges.

The checks are the existing per-launch harnesses, run at these shapes (each with its own sentinels, spans and bars):
  * inference: tests/test_gpu_forward_launches.py Part 1 (bf16 and fp32 modes) and tests/test_gpu_fp16.py's fp16 fixture;
  * training forward and backward: test_gpu_forward_launches.py Part 3 and tests/test_gpu_backward_launches.py, with the
    synthetic image batch made H x W as tests/test_gpu_rect_train.py does;
  * assignment and loss: tests/test_gpu_loss_launches.py on crowded targets scaled to the canvas (`crowded_targets`: up to
    70 ground truths per image on 21 to 420 anchors, duplicates, nested boxes, boxes over the edge, degenerate rows);
and two end-to-end checks of the plumbing around the launches: a DetectPipeline fed a 100 x 2000 frame lands on the 32 x
640 canvas and returns the eager chain's rows bit for bit, and a TrainStep at 32 x 640 matches the autograd path."""
import numpy as np
import pytest
import torch

import test_gpu_backward_launches as bwd
import test_gpu_fp16 as f16
import test_gpu_forward_launches as fwd
import test_gpu_loss_launches as ll
import test_gpu_rect as rect
import test_gpu_rect_train as rt
import test_loss_launch_cases as ll_cases
from test_gpu_fp16 import fp16_harness  # noqa: F401  (fixture)
from test_gpu_rect_train import rect_images  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

# name -> test_gpu_forward_launches.CONFIGS entry (model config, batch, height, width, precision, uint8 input)
INFER = {
    "yolov6n_32x32_b1": dict(cfg="yolov6n", N=1, H=32, W=32),
    "yolov6s_32x640_b2_u8_bf16": dict(cfg="yolov6s", N=2, H=32, W=640, u8=True),
    "yolov6s_32x640_b2_u8_fp32": dict(cfg="yolov6s", N=2, H=32, W=640, u8=True, precision="fp32"),
    "yolov6s_640x32_b2": dict(cfg="yolov6s", N=2, H=640, W=32),
    "yolov6m_64x640_b2": dict(cfg="yolov6m", N=2, H=64, W=640),
    "yolov6l6_64x64_b2": dict(cfg="yolov6l6", N=2, H=64, W=64),
    "yolov6n6_64x1280_b2": dict(cfg="yolov6n6", N=2, H=64, W=1280),
    "yolov6s_mbla_32x64_b2": dict(cfg="yolov6s_mbla", N=2, H=32, W=64),
    "yolov6n_qa_32x64_b2": dict(cfg="yolov6n_qa", N=2, H=32, W=64),
    "yolov6lite_s_64x64_b2": dict(cfg="yolov6lite_s", N=2, H=64, W=64),
    "yolov6lite_s_64x640_b2": dict(cfg="yolov6lite_s", N=2, H=64, W=640),
}
# the same harness in the fp16 mode (test_gpu_fp16.CONFIGS entries)
INFER_FP16 = {
    "yolov6s_640x32_b2": dict(cfg="yolov6s", N=2, H=640, W=32),
    "yolov6lite_s_64x64_b2": dict(cfg="yolov6lite_s", N=2, H=64, W=64),
    "yolov6lite_s_64x640_b2": dict(cfg="yolov6lite_s", N=2, H=64, W=640),
}
# name -> (model config, H, W, batch, fuse_ab head)
TRAIN = {
    "yolov6n_32x32": ("yolov6n", 32, 32, 2, False),
    "yolov6s_32x640": ("yolov6s", 32, 640, 2, False),
    "yolov6m_640x32": ("yolov6m", 640, 32, 2, False),
    "yolov6n6_64x1280": ("yolov6n6", 64, 1280, 2, False),
    "yolov6n_qa_32x64": ("yolov6n_qa", 32, 64, 2, False),
    "yolov6n_fuse_ab_32x640": ("yolov6n", 32, 640, 2, True),
}
# name -> (test_gpu_loss_launches.CONFIGS entry, det_loss variants (iou type, norm_gt_zero, grad_scale))
LOSS = {
    "p5_32x32_tal": (dict(strides=ll_cases.P5, R=4, H=32, W=32, assign="tal", topk=13), [("siou", 0, 1.0), ("giou", 1, 0.37)]),
    "p5_32x32_atss": (dict(strides=ll_cases.P5, R=68, H=32, W=32, assign="atss", topk=9), [("giou", 0, 1.0)]),
    "p5_32x32_ab_tal": (dict(strides=ll_cases.P5, R=4, H=32, W=32, assign="tal", topk=26, ab=True), [("giou", 1, 1.0)]),
    "p5_32x640_tal": (dict(strides=ll_cases.P5, R=68, H=32, W=640, assign="tal", topk=13), [("ciou", 0, 1.0)]),
    "p5_32x640_atss": (dict(strides=ll_cases.P5, R=4, H=32, W=640, assign="atss", topk=9), [("siou", 0, 2.5)]),
    "p6_64x64_tal": (dict(strides=ll_cases.P6, R=68, H=64, W=64, assign="tal", topk=13), [("giou", 0, 0.37)]),
    "p6_64x64_atss": (dict(strides=ll_cases.P6, R=68, H=64, W=64, assign="atss", topk=9), [("diou", 0, 1.0)]),
}


# ---------------------------------------------------------------------------------------------------------------- inference
@pytest.mark.parametrize("config", list(INFER))
def test_every_inference_launch_matches_float64_at_edge_canvas(config, monkeypatch):
    monkeypatch.setitem(fwd.CONFIGS, config, INFER[config])
    fwd.test_every_inference_launch_record_matches_float64(config)


@pytest.mark.parametrize("config", list(INFER_FP16))
def test_every_fp16_launch_matches_float64_at_edge_canvas(config, fp16_harness, monkeypatch):  # noqa: F811
    monkeypatch.setitem(f16.CONFIGS, config, INFER_FP16[config])
    f16.test_every_fp16_launch_record_matches_float64(config, fp16_harness)


# ---------------------------------------------------------------------------------------------------------------- training
@pytest.mark.parametrize("name", list(TRAIN))
def test_training_forward_launches_at_edge_canvas(name, rect_images, monkeypatch):  # noqa: F811
    cfg, H, W, B, fuse_ab = TRAIN[name]
    rect_images(H, W)
    monkeypatch.setitem(fwd.TRAIN_CONFIGS, name, (cfg, H, B, fuse_ab))
    fwd.test_every_training_forward_launch_matches_float64(name)


@pytest.mark.parametrize("name", list(TRAIN))
def test_training_backward_launches_at_edge_canvas(name, rect_images, monkeypatch):  # noqa: F811
    cfg, H, W, B, fuse_ab = TRAIN[name]
    rect_images(H, W)
    monkeypatch.setitem(bwd.MODELS, name, dict(cfg=cfg, size=H, batch=B, fuse_ab=fuse_ab))
    bwd.test_every_backward_launch_record_matches_float64_autograd(name)


# ---------------------------------------------------------------------------------------------------------------- assignment and loss
def crowded_targets(B, H, W, seed, nc=ll_cases.NC):
    """[n, 6] rows (img, cls, cx, cy, w, h; x normalised by W, y by H) for a canvas too small for
    test_loss_launch_cases.coco_like_targets, in a seeded shuffled order: image 0 has 70 rows (more than MAX_GT), image 1
    exactly 64, image 2 none, the others 10-40 -- tens of ground truths for 21 to 420 anchors.  Each image holds an exact
    duplicate, the same box with another class, a nested box, a box over the whole canvas, a box across the canvas edge, a
    zero-width and a zero-height row, a box around one stride-8 anchor centre and one between them, and labels 0 and nc - 1."""
    g = np.random.default_rng(seed)
    rows = []

    def box(img, cls, cx, cy, w, h):
        rows.append((img, cls, cx / W, cy / H, w / W, h / H))

    for img in range(B):
        if img == 2:
            continue
        want = 70 if img == 0 else 64 if img == 1 else int(g.integers(3, 41))
        start = len(rows)
        cls = int(g.integers(0, nc))
        cx, cy, w, h = g.uniform(0.3 * W, 0.7 * W), g.uniform(0.3 * H, 0.7 * H), g.uniform(6, 0.8 * W), g.uniform(6, 0.8 * H)
        box(img, cls, cx, cy, w, h)
        box(img, cls, cx, cy, w, h)
        box(img, (cls + 1) % nc, cx, cy, w, h)
        box(img, 0, cx + 0.1 * w, cy - 0.1 * h, 0.5 * w, 0.5 * h)
        box(img, nc - 1, W / 2, H / 2, float(W), float(H))
        box(img, cls, g.uniform(0, 4), g.uniform(0.2 * H, 0.8 * H), g.uniform(8, 0.5 * W), g.uniform(4, 0.5 * H))
        box(img, cls, g.uniform(0.2 * W, 0.8 * W), g.uniform(0.2 * H, 0.8 * H), 0.0, g.uniform(2, H / 2))
        box(img, cls, g.uniform(0.2 * W, 0.8 * W), g.uniform(0.2 * H, 0.8 * H), g.uniform(2, W / 2), 0.0)
        ax, ay = 8 * int(g.integers(0, W // 8)) + 4, 8 * int(g.integers(0, H // 8)) + 4
        box(img, int(g.integers(0, nc)), ax, ay, 3.0, 3.0)
        box(img, int(g.integers(0, nc)), ax + 4.0 if ax + 4 < W else ax - 4.0, ay, 2.0, 2.0)
        while len(rows) - start < want:
            w, h = g.uniform(2, W), g.uniform(2, H)
            box(img, int(g.integers(0, nc)), g.uniform(w / 4, W - w / 4), g.uniform(h / 4, H - h / 4), w, h)
    t = np.array(rows, dtype=np.float64)
    t = t[g.permutation(len(t))]
    return torch.from_numpy(t).float()


@pytest.mark.parametrize("name", list(LOSS))
def test_assignment_and_loss_launches_at_edge_canvas(name, monkeypatch):
    """targets_pad, box decode (or the anchor-aided boxes), TAL / ATSS, the expansion and det_loss against float64 on maps of
    21 (32 x 32, P5; 63 with three anchors per cell), 420 (32 x 640) and 85 (64 x 64, P6) anchors, whose top level holds one
    anchor per image row -- one in all at 32 x 32 and 64 x 64."""
    cfg, variants = LOSS[name]
    monkeypatch.setitem(ll.CONFIGS, name, cfg)
    monkeypatch.setitem(ll.LOSS_VARIANTS, name, variants)
    monkeypatch.setattr(ll.cases, "coco_like_targets", crowded_targets)
    ll.test_pad_decode_and_assign_launches(name)
    ll.test_assign_expand_launch(name)
    for iou, ngz, gscale in variants:
        ll.test_det_loss_launch(name, iou, ngz, gscale)
    _, _, _, _, gi, fg, _, _ = ll.checked_assignment(name)
    print(f"\n{name}: {int(fg.sum())} positive anchors of {fg.numel()} over {ll.B} images; "
          f"gts with a positive anchor per image: max {max(int(gi[b][fg[b].bool()].unique().numel()) for b in range(ll.B))}")
    assert int(fg.sum()) > 0, f"{name}: no positive anchor"


# ---------------------------------------------------------------------------------------------------------------- end to end
def test_pipeline_on_a_panorama_lands_on_32x640_and_equals_eager(monkeypatch):
    """A 100 x 2000 frame at img_size 640, letterbox auto=True: the 32 x 640 canvas (P5 1 x 20), host and CUDA frames, both
    layouts, through DetectPipeline against letterbox_batch -> model -> non_max_suppression -> rescale_boxes, bit for bit.
    The seeded model scores these canvases below test_gpu_rect's 0.03; the validation threshold 0.001 keeps rows to compare."""
    from yolov6_b200.pipeline import DetectPipeline
    from yolov6_b200.preprocess import rect_canvas
    assert rect_canvas(100, 2000, 640, 32) == (32, 640)
    monkeypatch.setattr(rect, "KW", dict(rect.KW, conf_thres=0.001))
    m, dev = rect.model("yolov6n"), torch.device("cuda:0")
    p = DetectPipeline(m, 2, 640, 640, raw_input=True, auto=True, source_shape=(100, 2000), **rect.KW)
    assert p.canvas == (32, 640)
    total = 0
    for layout, on_dev, seed in (("bgr_hwc", False, 0), ("rgb_chw", True, 10)):
        frs = rect.frames_of((100, 2000), 2, seed, layout, dev if on_dev else None)
        total += rect.check_rows(p(frs, layout=layout), rect.eager(m, frs, 640, 32, layout))
    print(f"\n32 x 640 pipeline: {total} rows equal the eager chain's")
    assert total > 0


def test_single_shape_step_matches_autograd_path_at_32x640():
    """TrainStep at 32 x 640 (rect training of a 1:20 batch) against the model's autograd path: the loss within 1e-4
    relative, every parameter gradient within 5e-3 relative L2 (the bars of tests/test_gpu_rect_train.py)."""
    from yolov6_b200.step import TrainStep
    H, W = 32, 640
    x, targets = rt.batch(H, W)
    m1, m2 = rt.make_model(), rt.make_model()
    (c1, _), (c2, _) = rt.losses(), rt.losses()
    preds, _ = m1(x)
    loss, _ = c1(preds, targets, 0, 0, H, W)
    loss.backward()
    ref = {n: p.grad.detach().clone() for n, p in m1.named_parameters() if p.grad is not None}
    step = TrainStep(m2, c2, rt.B, H, W, max_gt=64)
    step.load(x, targets)
    out = step.run(epoch_num=0).clone()
    torch.cuda.synchronize()
    assert abs(float(out[0]) - float(loss)) <= 1e-4 * abs(float(loss)), (float(out[0]), float(loss))
    assert float(out[5]) > 0, "no positive anchor at 32 x 640"
    print(f"\n32x640 step: loss {float(loss):.4f}, {int(out[5])} positives, worst gradient rel err vs autograd path "
          f"{rt.check_grads(ref, step.eng.flat, '32x640'):.2e}")
