"""Throughput of every built-in model on one GPU: bf16 inference images/s and the CUDA-graph training step.

    python tools/bench_models.py [--steps 30] [--warmup 10] [--models yolov6n,yolov6s_mbla,...] [--no-train]

Inference runs bench.py's own `bench_infer` (the DetectFarm pipeline bench.py times: one CUDA graph per batch -- network,
decode and batched NMS at the Evaler's settings -- from device-resident inputs, seeded synthetic weights): 640 px batch 32
for the P5 models, 1280 px batch 8 for the P6 ones, and 320 px (the Lite models' deploy size) at batch 32 and batch 1 for
YOLOv6Lite.  For each Lite model two more lines: the device time of every launch of one bf16 forward timed on its own,
summed per kind (wgmma convs against the depthwise / squeeze-excite / shuffle / upsample kernels), and the same network run
eagerly through PyTorch / cuDNN (oracle/lite.py in bf16, channels_last) on the same GPU, as the comparison point.  Each line also carries the conv GFLOP per image of the graph (2 x MACs
of every conv, transposed conv and prediction conv at that size).  The training step (TrainStep, CUDA graph, TAL or ATSS by
the config's atss_warmup_epoch at epoch 0, no optimizer) is timed for YOLOv6-S-MBLA (640, bs32), YOLOv6-N6 (1280, bs8) and
YOLOv6-S-QA next to YOLOv6-S (640, bs32).  For those two a further line splits one training step into its launches, each run
alone and summed per kind, with the achieved bandwidth of the QA kernels (yv6_qa_fwd / yv6_qa_bwd) over the bytes their shapes
imply, against the H100 SXM data-sheet 3.35 TB/s.
One JSON line per measurement; the first line names the card, its power limit and its maximum SM clock, read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from yolov6_b200 import configs  # noqa: E402
from yolov6_b200.arch import build_graph, is_lite  # noqa: E402

TRAIN_CASES = [("yolov6s_mbla", 640, 32), ("yolov6n6", 1280, 8), ("yolov6s_qa", 640, 32), ("yolov6s", 640, 32)]
SPLIT_CASES = [("yolov6s_qa", 640, 32), ("yolov6s", 640, 32)]
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def native(name):
    """[(size, batch)] of the measurements: 640 / 32 for P5 models, 1280 / 8 for P6 models, 320 / 32 and 320 / 1 for Lite."""
    if is_lite(configs.CONFIGS[name]):
        return [(320, 32), (320, 1)]
    return [(1280, 8) if len(configs.CONFIGS[name]["head"]["strides"]) == 4 else (640, 32)]


def conv_gflop_per_image(g, size):
    """2 x multiply-accumulates of every conv of graph g (inference forward, eval head) on one size x size image (or one
    H x W image when size is (H, W))."""
    H, W = (size, size) if isinstance(size, int) else size
    flop = 0
    for op in g.ops:
        if op.kind in ("pool", "se", "shuffle", "up") or (op.kind == "pred" and op.head[0] not in ("cls", "reg")):
            continue
        if op.kind == "stem":
            lvl = 1
        elif op.kind == "pred":
            lvl = g.bufs[op.src.buf].level
        else:
            lvl = g.bufs[op.dst.buf].level
        hw = (H >> lvl) * (W >> lvl)
        k = 2 if op.kind == "convT" else op.k        # a 2x2 stride-2 transposed conv: 4 taps per input pixel = 1 per output pixel
        flop += 2 * hw * op.cout * (1 if op.kind == "dw" else op.cin) * (1 if op.kind == "convT" else k * k)
    return flop / 1e9


def lite_split(name, size, batch, dev):
    """Device ms of one bf16 forward, every launch timed alone: wgmma convs (stem included) against the Lite kernels."""
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    eng = randomize_(build_model(name, 80, dev), seed=0).eval().set_precision("bf16").engine()
    x = torch.rand(batch, 3, size, size, device=dev)
    rows = eng.profile_calls(x)
    per_kind = {}
    for kind, _, ms in rows:
        per_kind[kind] = per_kind.get(kind, 0.0) + ms
    top = sorted(rows, key=lambda r: -r[2])[:8]
    return {"model": name, "mode": "launch split bf16", "size": size, "batch": batch, "launches": len(rows),
            "ms_by_kind": {k: round(v, 4) for k, v in per_kind.items()}, "slowest": [[k, n, round(ms, 4)] for k, n, ms in top]}


def lite_eager(name, size, batch, steps, warmup, dev):
    """The same network eagerly through PyTorch / cuDNN: oracle/lite.py's forward up to the head outputs (train-form weights,
    BN applied as its own ops; no decode and no NMS, which the kernel path's figure includes) in bf16, channels_last, seeded
    synthetic weights."""
    from oracle import fabricate as fab
    from oracle import lite
    from yolov6_b200.arch import param_specs
    keys = [(k, shape) for k, shape, _ in param_specs(build_graph(configs.get_config(name), 80))]
    sd = {k: v.to(dev, torch.bfloat16) if v.is_floating_point() else v for k, v in fab.fabricate_state_dict(keys).items()}
    sd = {k: v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v for k, v in sd.items()}
    x = torch.rand(batch, 3, size, size, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    with torch.no_grad():
        ms = bench.timed(lambda i: lite.forward(sd, lite.CONFIGS[name], x, train_outputs=True), steps, warmup, 1, dev)
    return {"model": name, "mode": "eager PyTorch/cuDNN bf16 channels_last, network only", "size": size, "batch": batch, "ms_per_step": ms,
            "images_per_s": batch / (ms * 1e-3)}


def bench_train_step(name, size, batch, steps, warmup, dev):
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.step import TrainStep
    from yolov6_b200.synth import synthetic_targets
    torch.manual_seed(0)
    model = build_model(name, 80, dev).train()
    hd = configs.CONFIGS[name]["head"]
    crit = ComputeLoss(fpn_strides=hd["strides"], num_classes=80, ori_img_size=size, warmup_epoch=hd["atss_warmup_epoch"],
                       use_dfl=hd["use_dfl"], reg_max=hd["reg_max"], iou_type=hd["iou_type"])
    step = TrainStep(model, crit, batch, size, size, in_dtype=torch.uint8, max_gt=64, graph=True)
    g = torch.Generator().manual_seed(1)
    step.load((torch.rand(batch, 3, size, size, generator=g) * 255).to(torch.uint8), synthetic_targets(batch, seed=100))
    ms = bench.timed(lambda i: step.run(epoch_num=0), steps, warmup, 1, dev)
    assert not step.overflowed()
    return {"model": name, "mode": "train", "size": size, "batch": batch, "ms_per_step": ms, "images_per_s": batch / (ms * 1e-3),
            "assigner": "ATSS" if hd["atss_warmup_epoch"] > 0 else "TAL", "step": "TrainStep (CUDA graph), no optimizer"}


def train_split(name, size, batch, dev, reps=5):
    """Device ms of every launch of one training step (the training engine's forward and backward call lists), each run alone
    after the per-step accumulators are cleared, median of `reps`, summed per kind.  yv6_qa_fwd moves u, v, t and (with the
    identity branch) x once each, yv6_qa_bwd dt and dx (read too when it accumulates): 2 bytes per element."""
    from yolov6_b200 import _lib
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    model = randomize_(build_model(name, 80, dev), seed=0).train()
    eng = model.train_engine()
    x = torch.rand(batch, 3, size, size, device=dev)
    cls, reg = eng.forward(x)
    eng.backward(torch.randn_like(cls) * 1e-3, torch.randn_like(reg) * 1e-3)
    torch.cuda.synchronize()
    sp = _lib.stream_ptr()

    def timed(fn):
        ts = []
        for _ in range(reps):
            eng.zero_arena.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return sorted(ts)[reps // 2]

    fwd_ms, bwd_ms, qa = {}, {}, {"qa_fwd": [0.0, 0], "qa_bwd": [0.0, 0]}
    calls = eng.fwd_calls
    try:
        for c in calls:
            eng.fwd_calls = [c]
            ms = timed(lambda: eng.run_forward(sp))
            fwd_ms[c.kind] = fwd_ms.get(c.kind, 0.0) + ms
            if c.kind == "qa":
                d = c.desc
                qa["qa_fwd"][0] += ms
                qa["qa_fwd"][1] += 2 * d.N * d.H * d.W * d.C * (3 + (1 if d.x else 0))
    finally:
        eng.fwd_calls = calls
    for j, c in enumerate(eng.bwd_calls):
        if c.bucket is not None:
            continue
        ms = timed(lambda: eng.backward(None, None, first=j, last=j + 1))
        bwd_ms[c.kind] = bwd_ms.get(c.kind, 0.0) + ms
        if c.kind == "qa_bwd":
            d = c.desc
            qa["qa_bwd"][0] += ms
            qa["qa_bwd"][1] += 2 * d.N * d.H * d.W * d.C * (2 + d.accumulate)
    out = {"model": name, "mode": "train launch split", "size": size, "batch": batch,
           "fwd_ms_by_kind": {k: round(v, 4) for k, v in fwd_ms.items()}, "bwd_ms_by_kind": {k: round(v, 4) for k, v in bwd_ms.items()}}
    for k, (ms, nbytes) in qa.items():
        if ms:
            out[k] = {"ms": round(ms, 4), "bytes": nbytes, "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                      "frac_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--models", default=",".join(configs.CONFIGS))
    ap.add_argument("--no-train", action="store_true")
    ap.add_argument("--train-only", action="store_true", help="skip the inference sweep")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"gpu": bench.gpu_info(0)}), flush=True)
    for name in ([] if args.train_only else args.models.split(",")):
        for size, batch in native(name):
            r = bench.bench_infer(name, batch, size, args.steps, args.warmup, 0, 1, dev, precision="bf16", e2e=False, roofline=False)
            print(json.dumps({"model": name, "mode": "infer bf16", "size": size, "batch": batch, "images_per_s": r["value"],
                              "ms_per_step": r["ms_per_step"], "launches_per_step": r["launches_per_step"],
                              "conv_gflop_per_image": conv_gflop_per_image(build_graph(configs.get_config(name), 80), size)}), flush=True)
            del r
            torch.cuda.empty_cache()
            if is_lite(configs.CONFIGS[name]):
                print(json.dumps(lite_eager(name, size, batch, args.steps, args.warmup, dev)), flush=True)
                print(json.dumps(lite_split(name, size, batch, dev)), flush=True)
                torch.cuda.empty_cache()
    if not args.no_train:
        for name, size, batch in TRAIN_CASES:
            print(json.dumps(bench_train_step(name, size, batch, args.steps, args.warmup, dev)), flush=True)
            torch.cuda.empty_cache()
        for name, size, batch in SPLIT_CASES:
            print(json.dumps(train_split(name, size, batch, dev)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
