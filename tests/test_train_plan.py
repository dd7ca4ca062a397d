"""CPU replay of the training engine's step (train.py): every library call, tensor copy / clear, stream and event of
`begin_step`, `run_forward` and a `backward` cut into the segments TrainStep captures, recorded against stand-ins for the
library and for torch's CUDA streams and events, and compared with a fixture (tests/golden/train_plan.json.gz, written by
tests/golden/make_golden_train_plan.py).

Pointers are recorded as (ordinal of the storage they point into, by first use; byte offset), so the log does not depend on
where the allocator put the tensors, and every pointer must lie inside a tensor reachable from the engine.  Descriptor fields
and scalar arguments are recorded by value (fields that are zero are left out)."""
import bisect
import contextlib
import ctypes as C
import gzip
import json
import os
import types

import pytest
import torch
from torch.overrides import TorchFunctionMode

from yolov6_b200 import _lib, configs
from yolov6_b200.model import build_model
from yolov6_b200.step import TrainStep
from yolov6_b200.train import TrainEngine

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_plan.json.gz")
BATCH, N_BUCKETS = 2, 3
# name -> config, model options, image size, input dtype, neck outputs as differentiable outputs, second step with accumulate=True
CASES = {
    "yolov6n": dict(cfg="yolov6n", accumulate_step=True),
    "yolov6n_u8": dict(cfg="yolov6n", dtype=torch.uint8),
    "yolov6m": dict(cfg="yolov6m"),
    "yolov6l6_128": dict(cfg="yolov6l6", size=128),
    "yolov6s_mbla": dict(cfg="yolov6s_mbla"),
    "yolov6n_qa": dict(cfg="yolov6n_qa"),
    "yolov6m_qa": dict(cfg="yolov6m_qa"),
    "yolov6n_fuse_ab": dict(cfg="yolov6n", fuse_ab=True),
    "yolov6n_distill_ns": dict(cfg="yolov6n", distill_ns=True, external_feat_grads=True),
}
TENSOR_OPS = ("copy_", "zero_", "clone")
STREAM_BASE = 0x5000


class Recorder:
    """The call log, the engine's storages and the stand-ins that write into the log."""

    def __init__(self, eng):
        self.log, self.streams, self.events, self.ordinal = [], [], [], {}
        self.handle = C.c_void_p(0x1000)
        self.main = FakeStream(self)
        self.eng = eng
        self.lo, self.hi = [], []

    def collect_storages(self):
        """Every storage reachable from the engine through attributes, lists, tuples, dicts and yolov6_b200 objects."""
        found, seen, stack = {}, set(), [self.eng]
        while stack:
            o = stack.pop()
            if id(o) in seen:
                continue
            seen.add(id(o))
            if isinstance(o, torch.Tensor):
                s = o.untyped_storage()
                if s.nbytes():
                    found[s.data_ptr()] = s.nbytes()
            elif isinstance(o, dict):
                stack += list(o.values())
            elif isinstance(o, (list, tuple)):
                stack += list(o)
            elif type(o).__module__.startswith("yolov6_b200") and hasattr(o, "__dict__"):
                stack += list(vars(o).values())
        self.lo = sorted(found)
        self.hi = [lo + found[lo] for lo in self.lo]

    def ptr(self, p, where):
        if isinstance(p, C.c_void_p):
            p = p.value
        if not p:
            return 0
        j = bisect.bisect_right(self.lo, p) - 1
        assert j >= 0 and p < self.hi[j], f"{where}: pointer {p:#x} lies outside every tensor reachable from the engine"
        base = self.lo[j]
        if base not in self.ordinal:
            self.ordinal[base] = len(self.ordinal)
        return [self.ordinal[base], p - base]

    def stream(self, sp):
        k = (sp.value if isinstance(sp, C.c_void_p) else sp) - STREAM_BASE
        assert 0 <= k < len(self.streams), f"unknown stream {sp}"
        return k

    def struct(self, d, where):
        out = {}
        for name, typ in d._fields_:
            v = getattr(d, name)
            if typ is C.c_void_p:
                v = self.ptr(v, f"{where}.{name}")
            elif issubclass(typ, C.Array):
                v = [self.ptr(x, f"{where}.{name}[{b}]") for b, x in enumerate(v)] if typ._type_ is C.c_void_p else list(v)
            if v != 0 and not (isinstance(v, list) and all(x == 0 for x in v)):
                out[name] = v
        return out

    def lib_call(self, fn, args):
        argtypes = _lib._SIGNATURES[fn][1]
        assert len(args) == len(argtypes) and args[0] is self.handle, fn
        entry = {"fn": fn, "stream": self.stream(args[-1]), "args": []}
        for j, (typ, a) in enumerate(zip(argtypes[1:-1], args[1:-1]), 1):
            where = f"{fn} argument {j}"
            if hasattr(a, "_obj"):                        # C.byref(descriptor)
                entry["desc"] = self.struct(a._obj, where)
                a = "desc"
            elif typ is C.c_void_p:
                a = self.ptr(a, where)
            elif isinstance(a, C.Array):
                a = list(a)
            else:
                assert isinstance(a, (int, float)), (where, a)
            entry["args"].append(a)
        self.log.append(entry)
        return 0

    def tensor_op(self, name, args):
        ts = [a for a in args if isinstance(a, torch.Tensor)]
        self.log.append({"fn": "torch." + name, "args": [[self.ptr(t.data_ptr(), f"torch.{name}"), list(t.shape), list(t.stride())]
                                                         for t in ts]})

    @contextlib.contextmanager
    def fakes(self):
        rec = self
        saved = (torch.cuda.current_stream, torch.cuda.Stream, torch.cuda.Event)
        torch.cuda.current_stream = lambda device=None: rec.main
        torch.cuda.Stream = lambda device=None, **kw: FakeStream(rec)
        torch.cuda.Event = lambda **kw: FakeEvent(rec)
        try:
            with TensorOps(self):
                yield
        finally:
            torch.cuda.current_stream, torch.cuda.Stream, torch.cuda.Event = saved


class FakeStream:
    def __init__(self, rec):
        self.rec, self.ordinal = rec, len(rec.streams)
        self.cuda_stream = STREAM_BASE + self.ordinal
        rec.streams.append(self)

    def wait_event(self, ev):
        self.rec.log.append({"fn": "wait_event", "stream": self.ordinal, "event": ev.ordinal})


class FakeEvent:
    def __init__(self, rec):
        self.rec, self.ordinal = rec, len(rec.events)
        rec.events.append(self)

    def record(self, stream=None):
        self.rec.log.append({"fn": "record_event", "stream": (stream or self.rec.main).ordinal, "event": self.ordinal})


class FakeLib:
    def __init__(self, rec):
        self.rec = rec

    def __getattr__(self, fn):
        return lambda *args: self.rec.lib_call(fn, args)


class TensorOps(TorchFunctionMode):
    """Logs the copies, clears and clones the engine issues while it runs."""

    def __init__(self, rec):
        super().__init__()
        self.rec = rec

    def __torch_function__(self, func, types_, args=(), kwargs=None):
        name = getattr(func, "__name__", "")
        if name in TENSOR_OPS:
            self.rec.tensor_op(name, args)
        return func(*args, **(kwargs or {}))


def dry_engine(case):
    """A TrainEngine over a CPU model whose library, handle and streams are the recorder's stand-ins."""
    c = CASES[case]
    cfg = configs.get_config(c["cfg"])
    if c.get("distill_ns"):       # the N / S distillation student needs the DFL head
        cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
    m = build_model(cfg, 80, torch.device("cpu"), fuse_ab=c.get("fuse_ab", False), distill_ns=c.get("distill_ns", False)).train()
    eng = TrainEngine.__new__(TrainEngine)
    eng.model, eng.g, eng.dev = m, m.graph, torch.device("cpu")
    eng.n_buckets = N_BUCKETS
    eng.debug, eng.dbg, eng._shape, eng.bucket_hook = False, {}, None, None
    eng.overlap_wgrad, eng._wg_stream = True, None
    eng.external_feat_grads, eng._feat_grads = bool(c.get("external_feat_grads")), None
    eng._build_state()
    rec = Recorder(eng)
    eng.lib, eng.h = FakeLib(rec), rec.handle
    return eng, rec


def replay(case):
    c = CASES[case]
    eng, rec = dry_engine(case)
    size = c.get("size", 64)
    eng._plan(BATCH, size, size, c.get("dtype", torch.float32))
    rec.collect_storages()
    firsts, lasts = TrainStep._segments(types.SimpleNamespace(eng=eng))
    steps = [False, True] if c.get("accumulate_step") else [False]
    with rec.fakes():
        for accumulate in steps:
            eng.debug = accumulate            # the second step also snapshots every op's incoming gradient
            sp = _lib.stream_ptr()
            rec.log.append({"fn": "step", "accumulate": accumulate})
            eng.begin_step(sp)
            eng.run_forward(sp)
            for first, last in zip(firsts, lasts):
                rec.log.append({"fn": "segment"})
                eng.backward(None, None, accumulate=accumulate, first=first, last=last)
    zero = [rec.ptr(t.data_ptr(), "zero_gbufs") for t in eng.zero_gbufs]
    return {"log": rec.log, "launch_counts": list(eng.launch_counts()), "zero_gbufs": zero, "streams": len(rec.streams),
            "events": len(rec.events), "debug_ops": sorted(eng.dbg)}


def dump(obj, path):
    raw = json.dumps(obj, sort_keys=True, separators=(",", ":")).encode()
    with open(path, "wb") as f, gzip.GzipFile(filename="", mode="wb", fileobj=f, mtime=0) as gz:
        gz.write(raw)


def load(path):
    with gzip.open(path, "rb") as f:
        return json.loads(f.read())


@pytest.fixture(scope="module")
def fixture():
    return load(FIXTURE)


@pytest.mark.parametrize("case", list(CASES))
def test_training_step_replays_the_pinned_launches(case, fixture):
    want, got = fixture[case], json.loads(json.dumps(replay(case)))
    for key in ("launch_counts", "zero_gbufs", "streams", "events", "debug_ops"):
        assert got[key] == want[key], f"{case}: {key}: want {want[key]}, got {got[key]}"
    for j, (w, g) in enumerate(zip(want["log"], got["log"])):
        if w == g:
            continue
        for k in sorted(set(w) | set(g)):
            if w.get(k) == g.get(k):
                continue
            if k == "desc" and isinstance(w.get(k), dict) and isinstance(g.get(k), dict):
                f = next(f for f in sorted(set(w[k]) | set(g[k])) if w[k].get(f) != g[k].get(f))
                pytest.fail(f"{case}: call {j} ({w['fn']}): desc.{f}: want {w[k].get(f, 0)}, got {g[k].get(f, 0)}")
            if k == "args" and isinstance(w.get(k), list) and isinstance(g.get(k), list) and len(w[k]) == len(g[k]):
                a = next(a for a in range(len(w[k])) if w[k][a] != g[k][a])
                pytest.fail(f"{case}: call {j} ({w['fn']}): argument {a + 1}: want {w[k][a]}, got {g[k][a]}")
            pytest.fail(f"{case}: call {j} ({w.get('fn')} / {g.get('fn')}): {k}: want {w.get(k)}, got {g.get(k)}")
    assert len(got["log"]) == len(want["log"]), f"{case}: {len(got['log'])} calls, want {len(want['log'])}"
