"""CPU replay of the serving pipelines (pipeline.py): every library call, tensor copy / clear / clone / read, stream, event,
synchronize, graph capture and graph replay that `DetectPipeline`, `DetectRing`, `DetectStream` and `DetectFarm` make, and
what each of their calls returns, recorded against stand-ins and compared with a fixture (tests/golden/serving_plan.json.gz,
written by tests/golden/make_golden_serving_plan.py).

The stand-ins, on top of tests/launch_log.py and the dry engine of tests/test_infer_plan.py:
- device tensors are CPU tensors that answer `.device` with cuda:0 (factory calls and `.to` with a CUDA device, and tensors
  computed from device tensors); `pin_memory()` is the identity;
- `torch.cuda.stream` switches the stand-in current stream, so each call is logged on the stream it is enqueued on;
- a graph capture runs on a capture stream and logs its calls once; their effects (copies, clears, the NMS and rescale
  stand-ins) are kept in the graph and run at each `replay()`;
- the NMS stand-in writes a per-call count and distinguishable rows (overflow set on the calls a case names), the rescale
  stand-in shifts the rows by the source size in the geometry table, so the returned rows show which batch and which
  geometry they came from.
Streams, events, graphs and storages are numbered by first appearance in the log."""
import contextlib
import ctypes as C
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch.overrides import TorchFunctionMode

import test_infer_plan as tip
from launch_log import FakeEvent, FakeLib, FakeStream, Recorder, dump, first_difference, load  # noqa: F401  (dump: make_golden)
from yolov6_b200 import _lib, engine, pipeline

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "serving_plan.json.gz")
CUDA0 = torch.device("cuda", 0)
B, S = 2, 64
HOST_CALLS = ("yv6_nms_workspace_bytes", "yv6_conv_plan_host", "yv6_last_error")     # size and plan queries: the real library
LOGGED_OPS = ("copy_", "zero_", "clone", "tolist", "item")


def _is_cuda(d):
    return isinstance(d, (str, torch.device)) and torch.device(d).type == "cuda"


def _array(p, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(p.value if isinstance(p, C.c_void_p) else p))


class Stream(FakeStream):
    def synchronize(self):
        self.rec.log.append({"fn": "stream_synchronize", "stream": self.ordinal})

    def wait_stream(self, other):
        self.rec.log.append({"fn": "wait_stream", "stream": self.ordinal, "other": other.ordinal})


class Event(FakeEvent):
    def record(self, stream=None):
        self.rec.log.append({"fn": "record_event", "stream": (stream or self.rec.current).ordinal, "event": self.ordinal})

    def synchronize(self):
        self.rec.log.append({"fn": "event_synchronize", "event": self.ordinal})


class Graph:
    """torch.cuda.CUDAGraph: `work` holds the effects of the captured calls, run again at each replay."""

    def __init__(self, rec):
        self.rec, self.ordinal, self.work = rec, len(rec.graphs), []
        rec.graphs.append(self)

    def replay(self):
        self.rec.log.append({"fn": "replay", "graph": self.ordinal, "stream": self.rec.current.ordinal})
        for fn in self.work:
            fn()


def nms_effect(rec, h, cls, reg, Bn, nc, R, nl, lh, lw, ls, conf, iou, agnostic, ml, mask, max_det, out, count, src, overflow,
               ws, ws_bytes, stream):
    n = rec.nms_calls
    rec.nms_calls += 1
    o = _array(out, C.c_float, Bn * max_det * 6).reshape(Bn, max_det, 6)
    c = _array(count, C.c_int32, Bn)
    o[:] = 0
    for b in range(Bn):
        c[b] = 1 + (n + b) % 3
        for j in range(c[b]):
            o[b, j] = (n, b, j, 100 + n, 0.5, j % nc)
    _array(overflow, C.c_int32, 1)[0] = int(n in rec.overflow_at)


def rescale_effect(rec, h, out, count, geo, Bn, max_det, H, W, res, stream):
    o = _array(out, C.c_float, Bn * max_det * 6).reshape(Bn, max_det, 6)
    r = _array(res, C.c_float, Bn * max_det * 6).reshape(Bn, max_det, 6)
    c = _array(count, C.c_int32, Bn)
    g = _array(geo, C.c_int32, Bn * 8).reshape(Bn, 8)
    r[:] = 0
    for b in range(Bn):
        r[b, :c[b]] = o[b, :c[b]]
        r[b, :c[b], 0] += g[b, 2]           # w0
        r[b, :c[b], 1] += g[b, 1]           # h0


EFFECTS = {"yv6_nms_batched_head": nms_effect, "yv6_rescale_boxes": rescale_effect}


class ServingRecorder(Recorder):
    def __init__(self, overflow_at=()):
        super().__init__(None)
        self.streams, self.graphs = [], []
        self.main = Stream(self)
        self.stack, self.capturing, self.capture_stream = [self.main], None, None
        self.spans, self.cuda, self.keep, self.dirty = {}, set(), [], False
        self.real = _lib.lib()
        self.nms_calls, self.overflow_at = 0, set(overflow_at)

    @property
    def current(self):
        return self.stack[-1]

    def run(self, effect):
        """Now, or at each replay of the graph being captured."""
        if self.capturing is not None:
            self.capturing.work.append(effect)
        else:
            effect()

    def add(self, t, cuda=False):
        s = t.untyped_storage()
        base, n = s.data_ptr(), s.nbytes()
        if n and base not in self.spans:
            self.spans[base], self.dirty = n, True
            self.keep.append(t)           # the storage is never freed, so its address never comes back as another tensor
            if cuda:
                self.cuda.add(base)

    def add_tree(self, obj):
        """The storages reachable from `obj` (an engine's weights), as device storages."""
        self.collect_storages(obj)
        for lo, hi in zip(self.lo, self.hi):
            self.spans.setdefault(lo, hi - lo)
            self.cuda.add(lo)
        self.dirty = True

    def on_cuda(self, t):
        return t.untyped_storage().data_ptr() in self.cuda

    def ptr(self, p, where):
        if self.dirty:
            self.lo = sorted(self.spans)
            self.hi = [lo + self.spans[lo] for lo in self.lo]
            self.dirty = False
        return super().ptr(p, where)

    def lib_call(self, fn, args):
        if fn in HOST_CALLS:
            return getattr(self.real, fn)(*args)
        super().lib_call(fn, args)
        if fn in EFFECTS:
            self.run(lambda: EFFECTS[fn](self, *args))
        return 0

    def tensor_op(self, name, args):
        super().tensor_op(name, args)
        if any(isinstance(a, torch.Tensor) and self.on_cuda(a) for a in args):
            self.log[-1]["stream"] = self.current.ordinal


class Devices(TorchFunctionMode):
    """Device tensors on the CPU (see the module docstring); logs the tensor ops of LOGGED_OPS, defers copies and clears made
    during a capture to the graph's replays."""

    def __init__(self, rec):
        super().__init__()
        self.rec = rec

    def __torch_function__(self, func, types_, args=(), kwargs=None):
        rec, kwargs = self.rec, dict(kwargs or {})
        if getattr(func, "__self__", None) is torch.Tensor.device:         # the Tensor.device getter
            return CUDA0 if rec.on_cuda(args[0]) else func(*args)
        name = getattr(func, "__name__", "")
        if name == "pin_memory":
            return args[0]
        to_cuda = _is_cuda(kwargs.get("device")) or (name == "to" and any(_is_cuda(a) for a in args[1:]))
        if to_cuda:
            args = ["cpu" if j and _is_cuda(a) else a for j, a in enumerate(args)]
            kwargs = {k: "cpu" if _is_cuda(v) else v for k, v in kwargs.items()}
            if name == "to":
                kwargs["copy"] = True
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        for t in tensors:
            rec.add(t)
        if name in LOGGED_OPS:
            rec.tensor_op(name, tensors)
            if name in ("copy_", "zero_") and rec.capturing is not None:
                rec.capturing.work.append(lambda: func(*args, **kwargs))
                return args[0]
        out = func(*args, **kwargs)
        if isinstance(out, torch.Tensor):
            rec.add(out, to_cuda or any(rec.on_cuda(t) for t in tensors))
        return out


@contextlib.contextmanager
def stand_ins(rec, lane_engine):
    """torch.cuda's streams, events, synchronize and graphs, the library and its handle, and the engines of DetectFarm's extra
    lanes replaced by the recorder's stand-ins; device tensors on the CPU."""
    cuda = torch.cuda
    names = ("current_stream", "Stream", "Event", "synchronize", "stream", "graph", "CUDAGraph", "is_current_stream_capturing")
    saved = [getattr(cuda, n) for n in names] + [_lib.lib, _lib.handle, engine.InferEngine]

    @contextlib.contextmanager
    def stream(s):
        rec.stack.append(s or rec.current)
        try:
            yield
        finally:
            rec.stack.pop()

    @contextlib.contextmanager
    def graph(g, **kw):
        if rec.capture_stream is None:
            rec.capture_stream = Stream(rec)
        rec.log.append({"fn": "capture_begin", "graph": g.ordinal, "stream": rec.capture_stream.ordinal})
        rec.stack.append(rec.capture_stream)
        rec.capturing = g
        try:
            yield
        finally:
            rec.capturing = None
            rec.stack.pop()
            rec.log.append({"fn": "capture_end", "graph": g.ordinal})

    fake = FakeLib(rec)
    cuda.current_stream = lambda device=None: rec.current
    cuda.Stream = lambda device=None, **kw: Stream(rec)
    cuda.Event = lambda **kw: Event(rec)
    cuda.synchronize = lambda device=None: rec.log.append({"fn": "synchronize"})
    cuda.stream, cuda.graph, cuda.CUDAGraph = stream, graph, lambda: Graph(rec)
    cuda.is_current_stream_capturing = lambda: rec.capturing is not None
    _lib.lib, _lib.handle = lambda: fake, lambda device_index=0: rec.handle
    engine.InferEngine = lambda graph, state_dict, device, precision="bf16": lane_engine()
    try:
        with tip.host_planner(), Devices(rec):
            yield
    finally:
        for n, v in zip(names, saved):
            setattr(cuda, n, v)
        _lib.lib, _lib.handle, engine.InferEngine = saved[len(names):]


class Model:
    """What the pipelines use of a Model: eval(), parameters()' device, graph, state_dict(), precision and engine()."""

    def __init__(self, eng):
        self.eng, self.graph, self.precision = eng, eng.g, eng.precision

    def eval(self):
        return self

    def parameters(self):
        return iter([SimpleNamespace(device=CUDA0)])

    def state_dict(self):
        return {}

    def engine(self):
        return self.eng


def dry(rec, cfg):
    """The dry engine of tests/test_infer_plan.py on cuda:0, calling the recorder's library."""
    with torch._C.DisableTorchFunction():
        eng, _ = tip.dry_engine(dict(cfg=cfg))
        rec.add_tree(eng)
    eng.device, eng.lib, eng.handle = CUDA0, FakeLib(rec), rec.handle
    return eng


def rows(v):
    if isinstance(v, torch.Tensor):
        return {"device": str(v.device), "shape": list(v.shape), "values": v.numpy().tolist()}
    return None if v is None else [rows(x) for x in v]


def nms_rows(out, count, *rest):
    """Device NMS results (out [B, max_det, 6], count [B], then overflow [1] when given): the rows count says are valid."""
    return rows([out[j, :int(k)] for j, k in enumerate(count.numpy())] + [count, *rest])


def got(rec, call):
    """What `call()` returns, or the RuntimeError / AssertionError it raises, into the log."""
    try:
        v = call()
    except (RuntimeError, AssertionError) as e:
        rec.log.append({"fn": "raised", "error": f"{type(e).__name__}: {e}"})
        return
    rec.log.append({"fn": "returned", "value": rows(v)})


def images(i):
    return torch.full((B, 3, S, S), i, dtype=torch.uint8)


def host_frames(layout="bgr_hwc"):
    shapes = [(40, 52), (64, 30)]
    return [np.full((h, w, 3), 9, np.uint8) if layout == "bgr_hwc" else torch.full((3, h, w), 9, dtype=torch.uint8)
            for h, w in shapes]


def dev_frames(layout="bgr_hwc"):
    shapes = [(48, 36), (20, 70)]
    return [torch.zeros((h, w, 3) if layout == "bgr_hwc" else (3, h, w), dtype=torch.uint8, device="cuda") for h, w in shapes]


def stream_loop(rec, ds, n, submit):
    for i in range(n):
        submit(i)
        got(rec, ds.collect)
    ds.drain()
    got(rec, ds.collect)
    got(rec, ds.collect)


def _pipeline_u8(rec, m):
    p = pipeline.DetectPipeline(m, B, S, S)
    for i in range(2):
        got(rec, lambda: p(images(i)))


def _pipeline_device_input(rec, m):
    p = pipeline.DetectPipeline(m, B, S, S, host_input=False)
    got(rec, lambda: p(torch.zeros(B, 3, S, S, device="cuda")))
    got(rec, p)
    rec.log.append({"fn": "outputs", "value": nms_rows(p.out_dev, p.count_dev)})


def _pipeline_overlap(rec, m):
    p = pipeline.DetectPipeline(m, B, S, S, overlap_h2d=True)
    for i in range(2):
        got(rec, lambda: p(images(i)))
    p.x_host.copy_(images(5))
    p.launch()
    got(rec, p)


def _pipeline_raw(rec, m):
    p = pipeline.DetectPipeline(m, B, S, S, raw_input=True)
    got(rec, lambda: p(host_frames()))
    got(rec, lambda: p(dev_frames()))
    got(rec, lambda: p([host_frames("rgb_chw")[0], dev_frames("rgb_chw")[1]], layout="rgb_chw"))
    got(rec, lambda: p(host_frames()[:1]))
    got(rec, lambda: p(host_frames(), layout="rgb_chw"))


def _ring(rec, m):
    r = pipeline.DetectRing(m, B, S, S)
    r.submit(images(0))
    got(rec, lambda: r.submit(images(1)) or r.submit(images(9)))
    for i in range(2, 5):
        got(rec, r.collect)
        r.submit(images(i))
    got(rec, r.collect)
    got(rec, r.collect)
    got(rec, r.collect)


def _stream_host(rec, m):
    ds = pipeline.DetectStream(m, B, S, S)
    stream_loop(rec, ds, 4, lambda i: ds.submit(images(i)))


def _stream_device_input(rec, m):
    ds = pipeline.DetectStream(m, B, S, S, host_input=False)
    stream_loop(rec, ds, 4, lambda i: ds.submit(torch.zeros(B, 3, S, S, device="cuda")))
    rec.log.append({"fn": "outputs", "value": [nms_rows(*d[k]) for d in (ds.dev_step, ds.dev_drain) for k in (0, 1)]})


def _stream_raw_ready(rec, m):
    ds = pipeline.DetectStream(m, B, S, S, raw_input=True, max_src_bytes=1 << 16)
    producer, ready = torch.cuda.Stream(), torch.cuda.Event()

    def submit(i):
        ready.record(producer)
        ds.submit(dev_frames()[: 1 + i % 2], ready=ready)
    stream_loop(rec, ds, 3, submit)
    ds.submit(host_frames("rgb_chw"), layout="rgb_chw")
    got(rec, lambda: ds.submit(host_frames()))
    got(rec, lambda: ds.submit(host_frames()))
    ds.drain()
    got(rec, ds.collect)


def _stream_fork_start(rec, m):
    saved = os.environ.get("YV6_NMS_FORK")
    os.environ["YV6_NMS_FORK"] = "start"
    try:
        ds = pipeline.DetectStream(m, B, S, S)
    finally:
        if saved is None:
            del os.environ["YV6_NMS_FORK"]
        else:
            os.environ["YV6_NMS_FORK"] = saved
    stream_loop(rec, ds, 3, lambda i: ds.submit(images(i)))


def _stream_four_levels(rec, m):
    ds = pipeline.DetectStream(m, B, 128, 128)
    stream_loop(rec, ds, 3, lambda i: ds.submit(torch.full((B, 3, 128, 128), i, dtype=torch.uint8)))


def _farm_bench(rec, m):
    """As bench.py's bench_infer drives the device-input farm."""
    farm = pipeline.DetectFarm(m, B, S, S, lanes=2, host_input=False)
    x = [torch.zeros(B, 3, S, S, device="cuda") for _ in range(2)]
    for ln in farm.lanes:
        for i in range(2):
            ln.x_dev[i].copy_(x[i])
    farm.release()
    for _ in range(5):
        farm.launch()
    farm.fence()
    ln = farm.lanes[(farm.n - 1) % len(farm.lanes)]
    o, c, overflow = ln.dev_step[1 - ((ln.steps - 1) & 1)]
    rec.log.append({"fn": "outputs", "value": nms_rows(o, c, overflow)})


def _farm_raw(rec, m):
    farm = pipeline.DetectFarm(m, B, S, S, lanes=2, raw_input=True, max_src_bytes=1 << 16)
    L = len(farm.lanes)
    for j in range(5):
        farm.submit(dev_frames() if j % 2 else host_frames())
        got(rec, farm.lanes[j % L].collect)
        rec.log.append({"fn": "lane_of_next", "lane": farm.lanes.index(farm.lane_of_next())})
    for ln, lane in enumerate(farm.lanes):
        with torch.cuda.stream(farm.streams[ln]):
            lane.drain()
        torch.cuda.synchronize()
        got(rec, lane.collect)


def _errors(rec, m):
    class Cpu(Model):
        def parameters(self):
            return iter([SimpleNamespace(device=torch.device("cpu"))])
    for cls in (pipeline.DetectPipeline, pipeline.DetectStream):
        got(rec, lambda: cls(Cpu(m.eng), B, S, S))
        got(rec, lambda: cls(m, B, S, S, raw_input=True, host_input=False))
    ds = pipeline.DetectStream(m, B, S, S, host_input=False)
    x = torch.zeros(B, 3, S, S, device="cuda")
    got(rec, lambda: [ds.submit(x) for _ in range(4)])
    ring = pipeline.DetectRing(m, B, S, S)
    got(rec, ring.collect)


# name -> (what the case runs, model config, NMS calls that report an overflow)
CASES = {
    "pipeline_u8": (_pipeline_u8, "yolov6n", {3}),
    "pipeline_device_input": (_pipeline_device_input, "yolov6n", ()),
    "pipeline_overlap_h2d": (_pipeline_overlap, "yolov6n", ()),
    "pipeline_raw": (_pipeline_raw, "yolov6n", ()),
    "ring": (_ring, "yolov6n", {7}),
    "stream_host": (_stream_host, "yolov6n", {6}),
    "stream_device_input": (_stream_device_input, "yolov6n", {6}),
    "stream_raw_ready": (_stream_raw_ready, "yolov6n", ()),
    "stream_fork_start": (_stream_fork_start, "yolov6n", ()),
    "stream_yolov6n6_128": (_stream_four_levels, "yolov6n6", ()),
    "farm_bench": (_farm_bench, "yolov6n", ()),
    "farm_raw": (_farm_raw, "yolov6n", ()),
    "errors": (_errors, "yolov6n", ()),
}


def renumber(log):
    """Streams, events and graphs numbered by first appearance in the log."""
    kinds = {"stream": "stream", "other": "stream", "event": "event", "graph": "graph"}
    seen = {k: {} for k in set(kinds.values())}
    for e in log:
        for key, kind in kinds.items():
            if key in e:
                e[key] = seen[kind].setdefault(e[key], len(seen[kind]))
    return log


def replay(case):
    run, cfg, overflow_at = CASES[case]
    rec = ServingRecorder(overflow_at)
    m = Model(dry(rec, cfg))
    with stand_ins(rec, lambda: dry(rec, cfg)), torch.no_grad():
        run(rec, m)
    return renumber(json.loads(json.dumps(rec.log)))


@pytest.fixture(scope="module")
def fixture():
    return load(FIXTURE)


@pytest.mark.parametrize("case", list(CASES))
def test_serving_replays_the_pinned_calls(case, fixture):
    first_difference(case, fixture[case], replay(case))
