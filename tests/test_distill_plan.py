"""CPU replay of the self-distillation teacher's forward-only plan (train.py, `TrainEngine(teacher=True)`) and of segment 0 of a
distillation TrainStep (step.py), recorded with the stand-ins of tests/launch_log.py on dry engines built as in
tests/test_train_plan.py.

The teacher plan must be the training forward of the same model, launch for launch, minus the anchor-aided pred convs and
their pack, with the same descriptors except that the BatchNorm finalize launches get null running statistics (batch
statistics only, track_running_stats = False) and the BN apply descriptors carry no backward fields.  The step must fork the
teacher onto a stream of its own and join it before the loss."""
import bisect
import contextlib
import ctypes as C
import types

import pytest
import torch

from launch_log import FakeLib, FakeStream, Recorder
from test_train_plan import dry_engine_of
from yolov6_b200 import _lib, configs
from yolov6_b200.model import build_model
from yolov6_b200.step import TrainStep
from yolov6_b200.train import TrainEngine

BATCH = 2
# name -> config, model options, image size
CASES = {
    "yolov6n_fuse_ab": dict(cfg="yolov6n", fuse_ab=True, size=64),
    "yolov6n6": dict(cfg="yolov6n6", size=128),
    "yolov6n_qa": dict(cfg="yolov6n_qa", size=64),
}
# descriptor fields only the backward pass reads (yv6_bn_bwd shares the BN apply descriptor), and the running statistics a
# teacher leaves alone
BACKWARD_FIELDS = {"s1", "s2", "dx", "dx_pitch", "accumulate", "dy", "dy_pitch", "work", "counter", "coef", "zeroed", "dres",
                   "dres_pitch", "dalpha", "dres_assign"}
RUNNING_STATS = {"running_mean", "running_var"}


def teacher_cfg(name, dfl=False):
    cfg = configs.get_config(name)
    if dfl:                       # the N / S recipe: teacher and student with the DFL head
        cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
    return cfg


def dry_teacher(cfg, fuse_ab=False, rec=None):
    """A teacher TrainEngine over a CPU model, with the recorder's library stand-in (a new recorder unless one is given)."""
    m = build_model(cfg, 80, torch.device("cpu"), fuse_ab=fuse_ab).train()
    eng = TrainEngine.__new__(TrainEngine)
    eng.model, eng.g, eng.dev, eng.teacher = m, m.graph, torch.device("cpu"), True
    eng.n_buckets = 1
    eng.debug, eng.dbg, eng._shape, eng.bucket_hook = False, {}, None, None
    eng.overlap_wgrad, eng._wg_stream = True, None
    eng.external_feat_grads, eng._feat_grads = False, None
    eng._build_state()
    rec = rec or Recorder(eng)
    eng.lib, eng.h = FakeLib(rec), rec.handle
    return eng, rec


class NamedRecorder(Recorder):
    """Records pointers by where they lie in the engine -- (attribute path, byte offset) -- so that two engines' logs compare.
    Zero-arena pointers are recorded without their offset: a teacher's arena holds the forward slots only.  `strict`: every
    pointer must lie in one of the forward's tensors; otherwise the others (gradients, scratch) are recorded as "other"."""
    strict = True

    ATTRS = ("x_static", "bufs", "cls", "reg", "stat_out", "wts", "ctx", "_ab", "zero_arena")

    def name_storages(self, eng):
        found = {}

        def visit(o, path):
            if isinstance(o, torch.Tensor):
                s = o.untyped_storage()
                if s.nbytes() and s.data_ptr() not in found:
                    found[s.data_ptr()] = (s.nbytes(), path)
            elif isinstance(o, dict):
                for k in sorted(o, key=repr):
                    visit(o[k], f"{path}[{k!r}]")
            elif isinstance(o, (list, tuple)):
                for j, v in enumerate(o):
                    visit(v, f"{path}[{j}]")

        for a in self.ATTRS:
            visit(getattr(eng, a, None), a)
        visit(eng.flat.pflat, "flat.pflat")
        self.lo = sorted(found)
        self.hi = [lo + found[lo][0] for lo in self.lo]
        self.path = [found[lo][1] for lo in self.lo]

    def ptr(self, p, where):
        if isinstance(p, C.c_void_p):
            p = p.value
        if not p:
            return 0
        j = bisect.bisect_right(self.lo, p) - 1
        if not (j >= 0 and p < self.hi[j]):
            assert not self.strict, f"{where}: pointer {p:#x} lies outside the engine's forward tensors"
            return "other"
        return "zero_arena" if self.path[j] == "zero_arena" else [self.path[j], p - self.lo[j]]


def forward_log(eng):
    rec = NamedRecorder(eng)
    rec.strict = eng.teacher
    rec.name_storages(eng)
    eng.lib, eng.h = FakeLib(rec), rec.handle
    with rec.fakes():
        eng.run_forward(_lib.stream_ptr())
    return rec.log


def student_and_teacher(case):
    c = CASES[case]
    s_eng, _ = dry_engine_of(c["cfg"], 1, fuse_ab=c.get("fuse_ab", False))
    t_eng, _ = dry_teacher(teacher_cfg(c["cfg"]), fuse_ab=c.get("fuse_ab", False))
    s_eng._plan(BATCH, c["size"], c["size"], torch.float32)
    t_eng._plan(BATCH, c["size"], c["size"], torch.float32, x_static=s_eng.x_static)
    return s_eng, t_eng


@pytest.mark.parametrize("case", list(CASES))
def test_teacher_plan_is_the_training_forward_without_running_statistics(case):
    s_eng, t_eng = student_and_teacher(case)
    want, got = forward_log(s_eng), forward_log(t_eng)
    # the anchor-aided pred convs (they write the `_ab` outputs) and their pack are the student's alone
    want = [e for e in want if e["fn"] != "yv6_head_ab_pack" and not (e.get("desc", {}).get("y", [""])[0].startswith("_ab"))]
    if s_eng.g.fuse_ab:
        assert len(want) == len(forward_log(s_eng)) - 3 * len(s_eng.g.strides)   # two convs and a pack per level
    assert [e["fn"] for e in got] == [e["fn"] for e in want], f"{case}: launch sequence"
    finalize = 0
    for j, (w, g) in enumerate(zip(want, got)):
        assert g["stream"] == w["stream"] and g["args"] == w["args"], f"{case}: call {j} ({w['fn']})"
        if "desc" not in w:
            continue
        wd = dict(w["desc"])
        if w["fn"] == "yv6_bn_apply_fwd":
            wd = {k: v for k, v in wd.items() if k not in BACKWARD_FIELDS}
        if w["fn"] in ("yv6_bn_stats_finalize", "yv6_qa_fwd"):
            finalize += any(k in wd for k in RUNNING_STATS)
            wd = {k: v for k, v in wd.items() if k not in RUNNING_STATS}
        assert not RUNNING_STATS & set(g["desc"]), f"{case}: call {j} ({w['fn']}) updates running statistics"
        assert g["desc"] == wd, f"{case}: call {j} ({w['fn']}): " + ", ".join(
            f"{k}: want {wd.get(k)}, got {g['desc'].get(k)}" for k in sorted(set(wd) | set(g["desc"])) if wd.get(k) != g["desc"].get(k))
    assert finalize > 0


@pytest.mark.parametrize("case", list(CASES))
def test_teacher_plan_has_no_backward(case):
    s_eng, t_eng = student_and_teacher(case)
    assert t_eng.bwd_calls == [] and t_eng.zero_gbufs == [] and t_eng.grad_tables == []
    assert all(g is None for g in t_eng.gbufs)
    for name in ("grad_cls", "grad_reg", "grad_cls_ab", "grad_reg_ab", "scratch", "cls_ab", "reg_ab"):
        assert not hasattr(t_eng, name), name
    assert t_eng.launch_counts() == (len(t_eng.fwd_calls), 0)
    assert t_eng.coef_out == {} and all("wt" not in w and all("wt" not in e for e in w.get("br", [])) for w in t_eng.wts.values())
    assert t_eng.zero_arena.numel() < s_eng.zero_arena.numel() // 4       # the forward's statistics sums only


@pytest.mark.parametrize("case", list(CASES))
def test_teacher_stem_reads_the_students_input(case):
    s_eng, t_eng = student_and_teacher(case)
    assert t_eng.x_static is s_eng.x_static
    stems = [c for c in t_eng.fwd_calls if c.fn == "yv6_stem_fwd"]
    assert stems and all(c.desc.x == s_eng.x_static.data_ptr() for c in stems)


@contextlib.contextmanager
def stream_context(rec):
    """torch.cuda.stream(s) for the recorder's stand-in streams: current_stream() is `s` inside."""
    saved = torch.cuda.stream

    @contextlib.contextmanager
    def stream(s):
        torch.cuda.current_stream = lambda device=None: s
        try:
            yield
        finally:
            torch.cuda.current_stream = lambda device=None: rec.main

    torch.cuda.stream = stream
    try:
        yield
    finally:
        torch.cuda.stream = saved


def test_segment_zero_forks_the_teacher_onto_its_own_stream():
    """N / S recipe: distill_ns student, fuse_ab teacher.  Every teacher launch (its arena clear, weight pack and forward) is
    enqueued on one stream other than the main one, after that stream waited for a fork event recorded on the main stream
    and before a join event the main stream waits for; the loss comes after the join."""
    s_eng, rec = dry_engine_of("yolov6n", 1, distill_ns=True)
    t_eng, _ = dry_teacher(teacher_cfg("yolov6n", dfl=True), fuse_ab=True, rec=rec)
    S = 64
    s_eng._plan(BATCH, S, S, torch.float32)
    t_eng._plan(BATCH, S, S, torch.float32, x_static=s_eng.x_static)
    rec.collect_storages(t_eng)

    def loss(*a, **kw):
        rec.log.append({"fn": "loss"})
        return {"feat_grads": []}

    step = TrainStep.__new__(TrainStep)
    with rec.fakes(), stream_context(rec):
        step.__dict__.update(eng=s_eng, teng=t_eng, t_stream=FakeStream(rec), dev=torch.device("cpu"), sizes=s_eng.sizes, targets=None,
                             max_gt=8, H=S, W=S, max_epoch=300, temperature=20.0, fuse_ab=False, distill=True, accumulate=False,
                             loss=types.SimpleNamespace(distill_feat=False, distill_forward_backward=loss))
        step._segment(0, 0)
    log = rec.log
    t_arena = rec.ptr(t_eng.zero_arena.data_ptr(), "teacher arena")
    t_stream = step.t_stream.ordinal
    assert t_stream != rec.main.ordinal
    fork = next(j for j, e in enumerate(log) if e["fn"] == "wait_event" and e["stream"] == t_stream)
    ev_fork = log[fork]["event"]
    assert any(e["fn"] == "record_event" and e["event"] == ev_fork and e["stream"] == rec.main.ordinal for e in log[:fork])
    join = next(j for j, e in enumerate(log) if e["fn"] == "record_event" and e["stream"] == t_stream)
    ev_join = log[join]["event"]
    wait = next(j for j, e in enumerate(log) if e["fn"] == "wait_event" and e["event"] == ev_join)
    assert log[wait]["stream"] == rec.main.ordinal
    teacher = [j for j, e in enumerate(log) if e.get("stream") == t_stream and "args" in e]
    assert len(teacher) == 1 + len(t_eng.fwd_calls)                          # pack + forward
    assert log[teacher[0]]["fn"] == "yv6_xform" and all(fork < j < join for j in teacher)
    clear = [j for j, e in enumerate(log) if e["fn"] == "torch.zero_" and e["args"][0][0] == t_arena]
    assert len(clear) == 1 and fork < clear[0] < teacher[0]
    # the student's forward runs on the main stream meanwhile; the loss waits for the join
    student_fwd = [j for j, e in enumerate(log) if e.get("stream") == rec.main.ordinal and e["fn"] == "yv6_stem_fwd"]
    assert student_fwd and all(join < j < wait for j in student_fwd)
    assert next(j for j, e in enumerate(log) if e["fn"] == "loss") > wait


def test_distillation_misuse_is_rejected_before_planning():
    """Each combination core/engine.py does not allow raises ValueError in the constructor, before any engine is built (these
    CPU models could not be planned)."""
    from yolov6_b200 import loss as det_loss
    from yolov6_b200 import loss_distill
    cpu = torch.device("cpu")
    dfl = teacher_cfg("yolov6n", dfl=True)
    ns_student = build_model(dfl, 80, cpu, distill_ns=True)
    teacher = build_model(dfl, 80, cpu, fuse_ab=True)
    kw = dict(num_classes=80, ori_img_size=64, warmup_epoch=0, use_dfl=True, reg_max=16)
    ns_loss, ml_loss = loss_distill.ComputeLossNS(**kw), loss_distill.ComputeLoss(**kw)
    cases = {
        "distillation loss without a teacher": (ns_student, ns_loss, dict(max_epoch=300)),
        "teacher without a distillation loss": (build_model("yolov6n", 80, cpu), det_loss.ComputeLoss(), dict(teacher=teacher, max_epoch=300)),
        "teacher class count": (ns_student, ns_loss, dict(teacher=build_model(dfl, 20, cpu, fuse_ab=True), max_epoch=300)),
        "teacher box channels": (ns_student, ns_loss, dict(teacher=build_model("yolov6n", 80, cpu, fuse_ab=True), max_epoch=300)),
        "teacher levels": (build_model("yolov6m", 80, cpu), ml_loss, dict(teacher=build_model("yolov6m6", 80, cpu), max_epoch=300)),
        "distill_ns student without ComputeLossNS": (ns_student, ml_loss, dict(teacher=teacher, max_epoch=300)),
        "ComputeLossNS without a distill_ns student": (build_model(dfl, 80, cpu), ns_loss, dict(teacher=teacher, max_epoch=300)),
        "fuse_ab student": (build_model("yolov6m", 80, cpu, fuse_ab=True), ml_loss,
                            dict(teacher=build_model("yolov6m", 80, cpu, fuse_ab=True), max_epoch=300, compute_loss_ab=object())),
        "no max_epoch": (ns_student, ns_loss, dict(teacher=teacher)),
    }
    for what, (student, crit, extra) in cases.items():
        with pytest.raises(ValueError):
            TrainStep(student, crit, BATCH, 64, 64, **extra)
            pytest.fail(what)
