"""Stand-ins for the library and for torch's CUDA streams and events, which record what an engine enqueues instead of running
it: the CPU replays of tests/test_train_plan.py and tests/test_infer_plan.py compare that log with a fixture.

Pointers are recorded as (ordinal of the storage they point into, by first use; byte offset), so the log does not depend on
where the allocator put the tensors, and every pointer must lie inside a tensor reachable from the engine.  Descriptor fields
and scalar arguments are recorded by value (fields that are zero are left out)."""
import bisect
import contextlib
import ctypes as C
import gzip
import json

import torch
from torch.overrides import TorchFunctionMode

from yolov6_b200 import _lib

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

    def collect_storages(self, *extra):
        """Every storage reachable from the engine (and from `extra`) through attributes, lists, tuples, dicts and yolov6_b200
        objects."""
        found, seen, stack = {}, set(), [self.eng, *extra]
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
        """torch.cuda's streams, events and synchronize replaced by the recorder's stand-ins, tensor ops logged."""
        rec = self
        saved = (torch.cuda.current_stream, torch.cuda.Stream, torch.cuda.Event, torch.cuda.synchronize)
        torch.cuda.current_stream = lambda device=None: rec.main
        torch.cuda.Stream = lambda device=None, **kw: FakeStream(rec)
        torch.cuda.Event = lambda **kw: FakeEvent(rec)
        torch.cuda.synchronize = lambda device=None: None
        try:
            with TensorOps(self):
                yield
        finally:
            torch.cuda.current_stream, torch.cuda.Stream, torch.cuda.Event, torch.cuda.synchronize = saved


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

    def elapsed_time(self, other):
        return 0.0


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


def dump(obj, path):
    raw = json.dumps(obj, sort_keys=True, separators=(",", ":")).encode()
    with open(path, "wb") as f, gzip.GzipFile(filename="", mode="wb", fileobj=f, mtime=0) as gz:
        gz.write(raw)


def load(path):
    with gzip.open(path, "rb") as f:
        return json.loads(f.read())


def first_difference(case, want, got):
    """pytest.fail with the first call where two logs differ, naming the descriptor field or argument."""
    import pytest
    for j, (w, g) in enumerate(zip(want, got)):
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
    assert len(got) == len(want), f"{case}: {len(got)} calls, want {len(want)}"
