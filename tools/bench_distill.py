"""Self-distillation step timing: YOLOv6-S (default) or -M, 640 px, batch 32, uint8 input, TAL.  The N / S recipe distils a
`distill_ns` student from a fuse_ab teacher with ComputeLossNS, the M / L recipe a plain student with ComputeLoss; both models
use the DFL head (use_dfl=True, reg_max=16).  Seeded synthetic weights and the synthetic targets of tools/bench_train.py.

Each phase builds its own models and is measured alone (its peak device memory too):
  distill_step    the distillation TrainStep (teacher forward on its own stream next to the student's forward, KL terms)
  plain_step      the same student's TrainStep with the detection loss only
  teacher_fwd     the teacher's forward-only plan alone (arena clear + pack + forward, replayed as one CUDA graph)
  fuseab_step     step 1 of the recipe: the fuse_ab teacher architecture's own TrainStep (anchor-free + anchor-aided losses)
  compatible      student(x), teacher(x) under no_grad, loss_distill loss, backward through autograd (eager launches)
teacher_hidden_ms = plain_step + teacher_fwd - distill_step: the teacher time that does not add to the step (the distillation
terms of the loss are counted against it).  Prints one JSON line.
usage: python tools/bench_distill.py [--model yolov6s|yolov6m] [--batch 32] [--size 640] [--steps 20] [--warmup 3]"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yolov6_b200 import _lib, configs  # noqa: E402
from yolov6_b200.loss import ComputeLoss  # noqa: E402
from yolov6_b200.loss_distill import ComputeLoss as DistillLoss  # noqa: E402
from yolov6_b200.loss_distill import ComputeLossNS  # noqa: E402
from yolov6_b200.loss_fuseab import ComputeLoss as ComputeLossAB  # noqa: E402
from yolov6_b200.model import build_model  # noqa: E402
from yolov6_b200.step import TrainStep  # noqa: E402
from yolov6_b200.synth import randomize_  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="yolov6s", choices=["yolov6s", "yolov6m"])
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--size", type=int, default=640)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()
B, S, name = args.batch, args.size, args.model
ns = name == "yolov6s"              # N / S recipe: distill_ns student + ComputeLossNS (core/engine.py:311-322)
EPOCH, MAX_EPOCH, T = 10, 300, 20.0
dev = torch.device("cuda:0")
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                     capture_output=True, text=True, check=True).stdout.strip().split(", ")
cfg = configs.get_config(name)
cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
iou = cfg["head"]["iou_type"]


def model(seed, **kw):
    return randomize_(build_model(cfg, 80, dev, **kw), seed=seed).train()   # random pred weights too: every loss term is non-zero


g = torch.Generator().manual_seed(1)
x = torch.randint(0, 256, (B, 3, S, S), generator=g, dtype=torch.uint8).to(dev)
rows = []
for b in range(B):                       # n ~ clip(Poisson(7.3), 1, 60) boxes per image (tools/bench_train.py)
    n = int(torch.poisson(torch.tensor([7.3]), generator=g).clamp(1, 60).item())
    wh = torch.rand(n, 2, generator=g) * 0.58 + 0.02
    cxy = wh / 2 + torch.rand(n, 2, generator=g) * (1 - wh)
    rows.append(torch.cat([torch.full((n, 1), float(b)), torch.randint(0, 80, (n, 1), generator=g).float(), cxy, wh], 1))
targets = torch.cat(rows).to(dev)
kw_dfl = dict(num_classes=80, ori_img_size=S, warmup_epoch=0, use_dfl=True, reg_max=16, iou_type=iou)


def distill_loss():
    return (ComputeLossNS if ns else DistillLoss)(**kw_dfl)


def student():
    return model(0, distill_ns=ns)


def teacher():
    return model(1, fuse_ab=True)


def timed(fn):
    """ms per call over args.steps calls after args.warmup, and the last call's output."""
    for _ in range(args.warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps, out


def phase(build):
    """Runs build() -> step function in a fresh memory window; returns (ms, peak GiB, last output)."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    fn = build()
    ms, out = timed(fn)
    peak = torch.cuda.max_memory_allocated() / 2**30
    out = None if out is None else out.clone()
    return ms, peak, out


def build_distill():
    st = TrainStep(student(), distill_loss(), B, S, S, in_dtype=torch.uint8, max_gt=64, teacher=teacher(), temperature=T,
                   max_epoch=MAX_EPOCH)
    st.load(x, targets)
    return lambda: st.run(epoch_num=EPOCH)


def build_plain():
    crit = ComputeLoss(**dict(kw_dfl, use_dfl=False, reg_max=0)) if ns else ComputeLoss(**kw_dfl)   # the lrtb head has 4 channels
    st = TrainStep(student(), crit, B, S, S, in_dtype=torch.uint8, max_gt=64)
    st.load(x, targets)
    return lambda: st.run(epoch_num=EPOCH)


def build_teacher():
    eng = teacher().teacher_engine()
    eng._plan(B, S, S, torch.uint8)
    eng.x_static.copy_(x)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):           # module loads and plans before capture
        eng.begin_step()
        eng.run_forward(_lib.stream_ptr())
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    gph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gph):
        eng.begin_step()
        eng.run_forward(_lib.stream_ptr())
    return gph.replay


def build_fuseab():
    st = TrainStep(teacher(), ComputeLoss(**kw_dfl), B, S, S, in_dtype=torch.uint8, max_gt=64,
                   compute_loss_ab=ComputeLossAB(**dict(kw_dfl, use_dfl=False, reg_max=0)))
    st.load(x, targets)
    return lambda: st.run(epoch_num=EPOCH)


def build_compatible():
    s, t, crit = student(), teacher(), distill_loss()

    def step():
        for p in s.parameters():
            p.grad = None
        preds, s_feats = s(x)
        with torch.no_grad():
            t_preds, t_feats = t(x)
        loss, _ = crit(preds, t_preds, s_feats, t_feats, targets, EPOCH, MAX_EPOCH, T, 0, S, S)
        loss.backward()
        return loss.detach()
    return step


res = {}
for key, build in (("distill_step", build_distill), ("plain_step", build_plain), ("teacher_fwd", build_teacher),
                   ("fuseab_step", build_fuseab), ("compatible", build_compatible)):
    ms, peak, out = phase(build)
    res[key] = dict(ms=round(ms, 3), peak_mem_gib=round(peak, 3))
    if out is not None:
        res[key]["loss"] = float(out[0] if out.dim() else out)
hidden = res["plain_step"]["ms"] + res["teacher_fwd"]["ms"] - res["distill_step"]["ms"]
print(json.dumps({"metric": f"self-distillation TrainStep ms/step {name} {S} bs{B} uint8 TAL ({'distill_ns student, ComputeLossNS' if ns else 'ComputeLoss'}, "
                            "fuse_ab teacher)", "value": res["distill_step"]["ms"], "unit": "ms/step",
                  "gpu": smi[0], "power_limit_w": float(smi[1]), "max_sm_clock_mhz": float(smi[2]), "steps": args.steps, "warmup": args.warmup,
                  "teacher_hidden_ms": round(hidden, 3), "teacher_hidden_frac": round(hidden / res["teacher_fwd"]["ms"], 3), **res}))
