"""CPU replay of the detection losses' host code (loss.py, loss_fuseab.py, loss_distill.py): every library call of
`forward_backward`, `distill_forward_backward` and `__call__` -- target padding, box decode, label assignment, the loss
descriptor and the KL terms -- recorded against the stand-ins of tests/launch_log.py and compared with a fixture
(tests/golden/loss_plan.json.gz, written by tests/golden/make_golden_loss_plan.py).

The losses allocate their buffers (padded targets, assignment, workspaces, outputs) inside the call, so pointers are kept
as they are seen and resolved to (storage ordinal, offset) after it, against the inputs, the loss object and every tensor a
torch function made during the call (kept alive until then)."""
import contextlib
import ctypes as C
import json
import math
import os

import pytest
import torch
from torch.overrides import TorchFunctionMode

from launch_log import FakeLib, Recorder, dump, first_difference, load  # noqa: F401  (dump: make_golden_loss_plan.py)
from yolov6_b200 import _lib, loss, loss_distill, loss_fuseab

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_plan.json.gz")
B, NC, S = 2, 3, 64
SIZES = [(S // s, S // s) for s in (8, 16, 32)]
A = sum(h * w for h, w in SIZES)
DFL = dict(use_dfl=True, reg_max=16)


class _Ptr:
    """A pointer argument or descriptor field, resolved once the call has returned."""

    def __init__(self, p, where):
        self.p, self.where = p, where


class LossRecorder(Recorder):
    def __init__(self):
        super().__init__(None)

    def ptr(self, p, where):
        if isinstance(p, C.c_void_p):
            p = p.value
        return _Ptr(p, where) if p else 0

    def lib_call(self, fn, args):
        if fn.endswith("_workspace_bytes"):          # no handle, no stream: a size at least as large as the library asks for
            self.log.append({"fn": fn, "args": list(args)})
            return 1024 + 64 * math.prod(args)
        return super().lib_call(fn, args)

    def resolve(self, *roots):
        self.collect_storages(*roots)

        def fix(v):
            if isinstance(v, _Ptr):
                return Recorder.ptr(self, v.p, v.where)
            return [fix(x) for x in v] if isinstance(v, list) else v

        for e in self.log:
            e["args"] = fix(e["args"])
            if "desc" in e:
                e["desc"] = {k: fix(v) for k, v in e["desc"].items()}


class KeepAlive(TorchFunctionMode):
    """Holds every tensor a torch function returns, so that the pointers of the call's temporaries stay valid."""

    def __init__(self):
        super().__init__()
        self.made = []

    def __torch_function__(self, func, types_, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        self.made += [t for t in (out if isinstance(out, (tuple, list)) else [out]) if isinstance(t, torch.Tensor)]
        return out


@contextlib.contextmanager
def stand_ins(rec):
    """The library, its handle and stream replaced by the recorder's stand-ins; the CUDA-only checks switched off."""
    saved = (_lib.lib, _lib.handle, _lib.stream_ptr, _lib.require_cuda)
    fake = FakeLib(rec)
    _lib.lib = lambda: fake
    _lib.handle = lambda device_index=0: rec.handle
    _lib.stream_ptr = lambda stream=None: C.c_void_p(rec.main.cuda_stream)
    _lib.require_cuda = lambda t, what: None
    try:
        yield
    finally:
        _lib.lib, _lib.handle, _lib.stream_ptr, _lib.require_cuda = saved


def inputs(seed=0):
    """Seeded CPU tensors: student and teacher head outputs, box branches of 4 and 68 channels, targets of three boxes in
    image 0, two in image 1 and one padding row (image -1), neck feature maps."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, generator=g)          # noqa: E731
    t = torch.rand(6, 6, generator=g)
    t[:, 0] = torch.tensor([0, 1, 0, 1, -1, 0], dtype=torch.float32)
    t[:, 1] = torch.tensor([0, 2, 1, 1, 0, 2], dtype=torch.float32)
    feats = [torch.zeros(B, 1, h, w) for h, w in SIZES]
    return dict(ps=r(B, A, NC), pd4=r(B, A, 4), pd68=r(B, A, 68), tps=r(B, A, NC), tpd68=r(B, A, 68),
                ps_ab=r(B, 3 * A, NC), pd_ab=r(B, 3 * A, 4), targets=t, none=torch.zeros(0, 6), feats=feats,
                s_feat=[r(B, 8, h, w) for h, w in SIZES], t_feat=[r(B, 8, h, w) for h, w in SIZES])


def _af(x, crit):
    crit.forward_backward(x["ps"], x["pd4"], SIZES, x["targets"], 10, S, S)


def _af_warmup(x, crit):
    crit.forward_backward(x["ps"], x["pd68"], SIZES, x["targets"], 1, S, S)


def _af_max_gt(x, crit):
    crit.forward_backward(x["ps"], x["pd68"], SIZES, x["targets"], 10, S, S, max_gt=8, grad_scores=torch.empty(B, A, NC),
                          grad_distri=torch.empty(B, A, 68), grad_scale=0.5)


def _af_no_targets(x, crit):
    crit.forward_backward(x["ps"], x["pd4"], SIZES, x["none"], 10, S, S)
    crit.forward_backward(x["ps"], x["pd4"], SIZES, x["none"], 0, S, S)


def _af_reuse(x, crit):
    st = crit.forward_backward(x["ps"], x["pd68"], SIZES, x["targets"], 10, S, S, max_gt=8)
    crit.forward_backward(x["ps"], x["pd4"], SIZES, None, 10, S, S, reuse=st, weights=(0.0, 2.5, 0.0),
                          grad_distri=torch.empty(B, A, 4))


def _ab(x, crit):
    crit.forward_backward(x["ps_ab"], x["pd_ab"], SIZES, x["targets"], 0, S, S)


def _ab_max_gt(x, crit):
    crit.forward_backward(x["ps_ab"], x["pd_ab"], SIZES, x["targets"], 3, S, S, max_gt=8,
                          grad_scores=torch.empty(B, 3 * A, NC), grad_distri=torch.empty(B, 3 * A, 4), grad_scale=2.0)


def _distill(x, crit):
    crit.distill_forward_backward(x["ps"], x["pd68"], x["tps"], x["tpd68"], SIZES, x["targets"], 3, 10, 20.0, S, S,
                                  x["s_feat"], x["t_feat"], max_gt=8, grad_scores=torch.empty(B, A, NC),
                                  grad_distri=torch.empty(B, A, 68))


def _distill_ns(x, crit):
    crit.distill_forward_backward(x["ps"], x["pd68"], x["tps"], x["tpd68"], SIZES, x["targets"], 3, 10, 20.0, S, S,
                                  max_gt=8, pred_lrtb=x["pd4"], grad_lrtb=torch.empty(B, A, 4))


def _call(x, crit):
    """__call__ with differentiable inputs; backward hands every input a gradient of its own shape and dtype."""
    ins = {k: (v.clone().requires_grad_() if k in ("ps", "pd4", "pd68", "ps_ab", "pd_ab") else v) for k, v in x.items()}
    if isinstance(crit, loss_distill.ComputeLossNS):
        leaves = [ins["ps"], ins["pd68"], ins["pd4"]]
        out = crit((x["feats"], *leaves), (x["feats"], x["tps"], x["tpd68"]), (), (), x["targets"], 3, 10, 20.0, 0, S, S)
    elif isinstance(crit, loss_distill.ComputeLoss):
        leaves = [ins["ps"], ins["pd68"]]
        out = crit((x["feats"], *leaves), (x["feats"], x["tps"], x["tpd68"]), (), (), x["targets"], 3, 10, 20.0, 0, S, S)
    elif isinstance(crit, loss_fuseab.ComputeLoss):
        leaves = [ins["ps_ab"], ins["pd_ab"]]
        out = crit((x["feats"], *leaves), x["targets"], 3, 0, S, S)
    else:
        leaves = [ins["ps"], ins["pd4"]]
        out = crit((x["feats"], *leaves), x["targets"], 10, 0, S, S)
    out[0].backward()
    for t in leaves:
        assert t.grad is not None and t.grad.shape == t.shape and t.grad.dtype == t.dtype


def af_loss(**kw):
    return loss.ComputeLoss(num_classes=NC, ori_img_size=S, **kw)


# name -> (loss constructor, what the case calls)
CASES = {
    "af_tal": (lambda: af_loss(iou_type="siou"), _af),
    "af_atss_warmup": (lambda: af_loss(warmup_epoch=4, **DFL), _af_warmup),
    "af_max_gt": (lambda: af_loss(loss_weight={"class": 0.5, "iou": 3.0, "dfl": 0.25}, **DFL), _af_max_gt),
    "af_no_targets": (lambda: af_loss(), _af_no_targets),
    "af_reuse_weights": (lambda: af_loss(**DFL), _af_reuse),
    "af_call": (lambda: af_loss(), _call),
    "ab": (lambda: loss_fuseab.ComputeLoss(num_classes=NC, ori_img_size=S), _ab),
    "ab_max_gt": (lambda: loss_fuseab.ComputeLoss(num_classes=NC, ori_img_size=S, iou_type="CIoU"), _ab_max_gt),
    "ab_call": (lambda: loss_fuseab.ComputeLoss(num_classes=NC, ori_img_size=S), _call),
    "distill": (lambda: loss_distill.ComputeLoss(num_classes=NC, ori_img_size=S, **DFL), _distill),
    "distill_feat": (lambda: loss_distill.ComputeLoss(num_classes=NC, ori_img_size=S, distill_feat=True,
                                                      distill_weight={"class": 2.0, "dfl": 0.5}, **DFL), _distill),
    "distill_call": (lambda: loss_distill.ComputeLoss(num_classes=NC, ori_img_size=S, **DFL), _call),
    "distill_ns": (lambda: loss_distill.ComputeLossNS(num_classes=NC, ori_img_size=S, **DFL), _distill_ns),
    "distill_ns_call": (lambda: loss_distill.ComputeLossNS(num_classes=NC, ori_img_size=S, **DFL), _call),
}


def replay(case):
    make, run = CASES[case]
    x, crit, rec, keep = inputs(), make(), LossRecorder(), KeepAlive()
    with stand_ins(rec), keep:
        run(x, crit)
    rec.resolve(x, crit, keep.made)
    return rec.log


@pytest.fixture(scope="module")
def fixture():
    return load(FIXTURE)


@pytest.mark.parametrize("case", list(CASES))
def test_loss_host_replays_the_pinned_calls(case, fixture):
    first_difference(case, fixture[case], json.loads(json.dumps(replay(case))))


def test_loss_path_refuses_cpu_tensors():
    from yolov6_b200 import assigners
    x = inputs()
    for call, what in [
        (lambda: af_loss().forward_backward(x["ps"], x["pd4"], SIZES, x["targets"], 10, S, S), "yolov6_b200.ComputeLoss runs"),
        (lambda: loss_fuseab.ComputeLoss().forward_backward(x["ps_ab"], x["pd_ab"], SIZES, x["targets"], 10, S, S),
         "yolov6_b200.loss_fuseab.ComputeLoss runs"),
        (lambda: assigners.tal_compact(x["ps"], x["pd4"], x["pd4"][0, :, :2], None, None), "yolov6_b200 assigners run"),
        (lambda: assigners.atss_compact(x["pd4"][0], [A], None, None, None, NC), "yolov6_b200 assigners run"),
    ]:
        with pytest.raises(RuntimeError, match=f"^{what} on CUDA tensors only"):
            call()
