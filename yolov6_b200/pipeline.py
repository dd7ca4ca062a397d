"""Steady-state detection pipeline: host images -> detections, replayed as ONE CUDA graph.

The reference's `Inferer.infer` / `Evaler.predict_model` (core/inferer.py:70-82, core/evaler.py:118-134)
run H2D copy, `.float()/255`, the model and NMS as separate eager calls per batch.  `DetectPipeline`
captures the same sequence -- pinned-host uint8 batch -> device (stem kernel scales by 1/255 on the
fly) -> network kernels -> decode -> batched NMS -> detections back to pinned host memory -- into a
CUDA graph once per (batch, size); `__call__` is then a single graph launch, so the ~80 kernel
launches and all Python/ctypes work disappear from the steady state (SURVEY.md 8f N1).

`overlap_h2d=True` keeps the host->device copy of the images out of the graph and issues it on a copy
stream instead: with two pipelines used alternately (see `DetectRing`) the copy of batch i+1 runs on the
copy engine while the kernels of batch i run on the SMs, so a serving loop is bound by max(copy, compute)
instead of their sum.

`raw_input=True` serves decoded frames (any size, sizes mixed freely within a batch) instead of letterboxed batches, in OpenCV's
`imread` layout (uint8 HWC BGR, `layout="bgr_hwc"`, the default) or torchvision's decoders' (uint8 RGB CHW, `layout="rgb_chw"`).
A host frame (numpy array or CPU tensor) goes through a fixed-capacity pinned staging buffer (`max_src_bytes`, host frames
only) that is copied to the device on the copy stream; a CUDA tensor on the pipeline's device is read in place.  Per-image
source records and geometry go up on the copy stream too, and the graph runs letterbox -> network -> NMS -> rescale -> D2H
(`yolov6_b200.preprocess`).  Results are per-image [k, 6] rows in source pixels, what `Inferer.infer` holds in `det` after
core/inferer.py:103.  Records and geometry are data, so one captured graph serves any mix of image sizes, layouts and
locations.

Device frames are read in stream order: the copy stream waits for the work enqueued on the caller's current stream before
the call, so frames a kernel wrote there are complete when the graph reads them.  They are read in place, so the caller
must not write to them until `collect()` has returned their batch (`DetectPipeline.__call__` returns after the batch is
done); the pipeline keeps a reference to them at least until then, so dropping them early is safe.

`auto=True` (with raw_input) serves the way `tools/infer.py` letterboxes: `Inferer.process_image` pads a frame only up to the
next multiple of the stride (letterbox auto=True), so a 1920 x 1080 frame at img_size 640 runs on a 384 x 640 canvas, 0.6
of the square one's conv work.  `height, width` are then Inferer's img_size and `source_shape=(h0, w0)` names the frames
served: the pipeline is built, pinned and captured at `rect_canvas(h0, w0, (height, width), stride)`, exposed as `.canvas`
(one fixed shape, so slots, graphs and lanes are those of the full canvas).  A frame of any size is accepted when its own
rect canvas is that one (1080p and 720p both give 384 x 640 at 640); any other frame raises RuntimeError before anything is
written.  `stride` defaults to Inferer's `max(model stride, 32)`.

Each batch in flight lives in a `BatchSlot` (its input and staging buffers, pinned results and events): `DetectPipeline`
holds one, `DetectStream` two, used by alternate steps.
"""
import functools
import os

import torch

from .nms import nms_batched_head, workspace_bytes
from .preprocess import (REC, check_frames, inferer_size, inferer_stride, letterbox_frames_launch, pack_sources, rect_canvas,
                         rescale_launch)

RAW_DEFAULT_BYTES = 1920 * 1080 * 3        # staging bytes per batch slot when max_src_bytes is not given: one 1080p frame each
OVERFLOW = "non_max_suppression: more than 65536 near-identical candidate scores in one image; raise conf_thres"


class BatchSlot:
    """The buffers and events of one batch in flight: the device input with its pinned host input or, for raw frames, the
    staging buffer, record and geometry tables; the pinned results; `ev_copied` (its H2D is complete) and `ev_done` (the
    step that read it is complete).  `hold_geo`: the letterbox keeps a copy of the geometry (`res_geo`) for a rescale that
    runs after the copy stream may already have refilled `geo_dev` with the next batch's.  The input is `height x width`;
    with `auto`, raw frames are letterboxed at img_size `size` with padding to a multiple of `stride` and must land on it."""

    def __init__(self, batch, height, width, max_det, host_input, raw_input, max_src_bytes, dev, hold_geo=False, auto=False,
                 stride=32, size=None):
        self.dev, self.host_input, self.raw, self.hold_geo = dev, host_input, raw_input, hold_geo
        self.auto, self.stride, self.size = auto, stride, tuple(size or (height, width))
        self.x_dev = torch.zeros(batch, 3, height, width, dtype=torch.uint8 if host_input else torch.float32, device=dev)
        self.x_host = torch.zeros(batch, 3, height, width, dtype=torch.uint8).pin_memory() if host_input and not raw_input else None
        if raw_input:
            cap = int(max_src_bytes) if max_src_bytes else batch * RAW_DEFAULT_BYTES
            geo = torch.tensor([[0, height, width, 0, 0, 0, 0, 0]] * batch, dtype=torch.int32)    # all border until frames arrive
            rec = torch.zeros(batch * REC, dtype=torch.uint8)          # null records: an all-border slot reads no source
            self.src_host = torch.empty(cap, dtype=torch.uint8).pin_memory()
            self.geo_host, self.rec_host = geo.pin_memory(), rec.pin_memory()
            self.src_dev, self.geo_dev, self.rec_dev = torch.zeros(cap, dtype=torch.uint8, device=dev), geo.to(dev), rec.to(dev)
            self.res_geo = geo.to(dev) if hold_geo else self.geo_dev
            self.res = torch.zeros(batch, max_det, 6, device=dev)
            self.nbytes, self.frames = 0, []          # staged host bytes; device frames, read in place by the next launch
        self.out_host = torch.zeros(batch, max_det, 6).pin_memory()
        self.count_host = torch.zeros(batch + 1, dtype=torch.int32).pin_memory()      # per-image counts, then the overflow flag
        self.ev_copied, self.ev_done, self.ev_ready = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        self.ready = None          # event the next H2D waits for: the producer of the staged device frames
        self.used = False          # ev_done has been recorded

    def stage(self, images, layout="bgr_hwc", ready=None):
        """Put the next batch into the slot: an image batch into x_host (host input) or x_dev, or 1..B raw frames into the
        staging tables (RuntimeError before anything is written when a frame is unusable).  The H2D of device frames waits
        for `ready`, by default an event recorded now on the current stream."""
        if not self.raw:
            (self.x_host if self.host_input else self.x_dev).copy_(images)
            return
        srcs = check_frames(images, self.geo_host.shape[0], layout, self.dev)
        self.nbytes, _, self.frames = pack_sources(srcs, self.geo_host.shape[0], *self.size, True, layout, self.src_host,
                                                   self.geo_host, self.rec_host, self.src_dev.data_ptr(), self.auto, self.stride,
                                                   tuple(self.x_dev.shape[2:]))
        # only device frames need it: the caller's stream usually holds the previous step, and a copy that waited for it
        # would no longer overlap that step
        if self.frames:
            if ready is None:
                ready = self.ev_ready
                ready.record(torch.cuda.current_stream(self.dev))
            self.ready = ready

    def h2d(self, copy_stream, cur):
        """Copy the staged input to the device on `copy_stream`, after the slot's previous step and the producer of its
        device frames; `cur` waits for the copy."""
        if self.used:
            copy_stream.wait_event(self.ev_done)           # the previous step of this slot is done with x_dev
        if self.ready is not None:
            copy_stream.wait_event(self.ready)
            self.ready = None
        with torch.cuda.stream(copy_stream):
            if not self.raw:
                self.x_dev.copy_(self.x_host, non_blocking=True)
            else:
                if self.nbytes:
                    self.src_dev[:self.nbytes].copy_(self.src_host[:self.nbytes], non_blocking=True)
                self.rec_dev.copy_(self.rec_host, non_blocking=True)
                self.geo_dev.copy_(self.geo_host, non_blocking=True)
            self.ev_copied.record(copy_stream)
        cur.wait_event(self.ev_copied)

    def done(self, stream):
        self.ev_done.record(stream)
        self.used = True

    def letterbox(self):
        """Raw frames -> x_dev (nothing to do for letterboxed input)."""
        if self.raw:
            letterbox_frames_launch(self.rec_dev, self.geo_dev, self.x_dev)
            if self.hold_geo:
                self.res_geo.copy_(self.geo_dev)

    def detect(self, nms, cls, reg):
        """NMS over the head tensors, rescaled to source pixels (raw frames) and copied to the pinned results (host input).
        Returns the device results (out, count, overflow)."""
        out, count, _, overflow = nms(cls, reg)
        if self.raw:
            out = rescale_launch(out, count, self.res_geo, self.x_dev.shape[2], self.x_dev.shape[3], res=self.res)
        if self.host_input:
            self.out_host.copy_(out, non_blocking=True)
            self.count_host[:-1].copy_(count, non_blocking=True)
            self.count_host[-1:].copy_(overflow, non_blocking=True)
        return out, count, overflow

    def rows(self, n, dev=None):
        """The per-image [k, 6] detections of the first n images of the slot's finished batch, from the pinned results or,
        when given, from the device results `dev` = (out, count, overflow)."""
        if dev is None:
            out, counts = self.out_host, self.count_host.tolist()
            if counts[-1]:
                raise RuntimeError(OVERFLOW)
        else:
            out, count, overflow = dev
            if overflow.item():
                raise RuntimeError(OVERFLOW)
            counts = count.tolist()
        return [out[j, :counts[j]].clone() for j in range(n)]


class _Served:
    """What DetectPipeline and DetectStream share: the checks, NMS settings, pinned engine shape, NMS workspace and batch
    slots, and the warm-up-then-capture of their graphs.  `canvas` is the (H, W) everything is built at: (height, width),
    or with auto=True the rect canvas of `source_shape` at img_size (height, width)."""

    def __init__(self, model, batch, height, width, nms_kw, host_input, raw_input, max_src_bytes, slots, engine=None, auto=False,
                 source_shape=None, stride=None):
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} needs a CUDA model")
        if raw_input and not host_input:
            raise RuntimeError(f"{type(self).__name__}: raw_input returns detections in host memory (host_input=True)")
        size = (height, width)
        if auto:
            if not raw_input or source_shape is None:
                raise RuntimeError(f"{type(self).__name__}: auto=True letterboxes decoded frames: it needs raw_input=True and "
                                   f"source_shape=(h0, w0)")
            stride = int(stride or inferer_stride(model.graph.strides))
            size = inferer_size(size, stride)
            height, width = rect_canvas(*source_shape, size, stride)
        self.canvas = (height, width)
        self.host_input = bool(host_input)
        self.slots = [BatchSlot(batch, height, width, nms_kw["max_det"], self.host_input, raw_input, max_src_bytes, self.dev,
                                hold_geo=slots > 1, auto=bool(auto), stride=stride or 32, size=size) for _ in range(slots)]
        self.shape = (batch, height, width, self.slots[0].x_dev.dtype)
        self.eng = engine if engine is not None else model.engine()
        self.eng.pin(*self.shape)          # the graphs point at this shape's buffers
        self.eng.attach(self)              # a refold of the engine waits for this pipeline's batches in flight
        self.sizes = [(height // int(s), width // int(s)) for s in model.graph.strides]
        A = sum(h * w for h, w in self.sizes)
        # scratch owned by this pipeline: a shared cache could be replaced (freed) while a graph still references it
        self.nms_ws = torch.empty(workspace_bytes(batch, A, model.graph.num_classes, nms_kw["multi_label"]), dtype=torch.uint8,
                                  device=self.dev)
        self.nms = functools.partial(nms_batched_head, sizes=self.sizes, strides=model.graph.strides, workspace=self.nms_ws, **nms_kw)

    def in_flight(self):
        """What a refold of the engine must follow: the done events of the slots' last steps and, for a pipeline that does not
        record them (DetectPipeline without overlap_h2d), the stream of its last launch."""
        out = [sl.ev_done for sl in self.slots if sl.used]
        if getattr(self, "launch_stream", None) is not None:
            out.append(self.launch_stream)
        return out

    def _capture(self, warm, bodies):
        """Run `warm` on a side stream (plans, tensor maps, cudaFuncSetAttribute, allocator warm-up), then capture one graph
        per body."""
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            warm()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        graphs = []
        for body in bodies:
            graphs.append(torch.cuda.CUDAGraph())
            with torch.cuda.graph(graphs[-1]), torch.no_grad():
                body()
        return graphs


class DetectPipeline(_Served):
    def __init__(self, model, batch, height, width, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
                 multi_label=False, max_det=300, host_input=True, overlap_h2d=False, copy_stream=None, raw_input=False,
                 max_src_bytes=None, auto=False, source_shape=None, stride=None):
        super().__init__(model, batch, height, width, dict(conf_thres=conf_thres, iou_thres=iou_thres, classes=classes,
                         agnostic=agnostic, multi_label=multi_label, max_det=max_det), host_input, raw_input, max_src_bytes, 1,
                         auto=auto, source_shape=source_shape, stride=stride)
        self.slot = self.slots[0]
        self.x_dev, self.x_host = self.slot.x_dev, self.slot.x_host
        self.n_frames = batch
        self.overlap_h2d = bool((overlap_h2d or raw_input) and host_input)
        if self.overlap_h2d:
            self.copy_stream = copy_stream or torch.cuda.Stream(device=self.dev)
        self.graph, = self._capture(lambda: (self._body(), self._body()), [self._body])

    def _body(self):
        self.slot.letterbox()
        if self.host_input and not self.overlap_h2d:
            self.x_dev.copy_(self.x_host, non_blocking=True)
        # the [B, A, 5+nc] prediction tensor of Detect.forward (effidehead.py:131-139) is never materialised here: the NMS
        # kernels scan the class scores where the cls_pred convs wrote them and decode boxes for the candidates only
        cls, reg, _ = self.eng.forward(self.x_dev, decode=False)
        self.out_dev, self.count_dev, _ = self.slot.detect(self.nms, cls, reg)

    def launch(self):
        """Enqueue one batch (input already in `x_host` / `x_dev`); asynchronous.  It runs after the last refold of the
        engine (InferEngine.refold)."""
        cur = torch.cuda.current_stream(self.dev)
        self.eng.after_fold(cur)
        if not self.overlap_h2d:
            self.graph.replay()
            self.launch_stream = cur      # a refold orders itself after this stream's work (in_flight)
            return
        self.slot.h2d(self.copy_stream, cur)
        self.graph.replay()
        self.slot.done(cur)

    def __call__(self, images=None, layout="bgr_hwc"):
        """images: uint8 [B,3,H,W] host tensor (host_input) or fp32 device tensor; with raw_input, a list of 1..B uint8 frames
        in `layout` (see the module docstring), each a numpy array, a CPU tensor or a CUDA tensor on the pipeline's device.
        Returns the list of per-image [k,6] detections (host tensors when host_input) like `non_max_suppression`; with
        raw_input in source pixels, rounded (Inferer.rescale(...).round())."""
        if images is not None:
            self.slot.stage(images, layout)
            if self.slot.raw:
                self.n_frames = len(images)
        self.launch()
        torch.cuda.current_stream(self.dev).synchronize()
        if self.host_input:
            return self.slot.rows(self.n_frames)
        counts = self.count_dev.tolist()
        return [self.out_dev[i, :counts[i]] for i in range(self.out_dev.shape[0])]


class DetectRing:
    """Two `DetectPipeline`s used alternately with one shared copy stream: `submit(images)` enqueues a batch and
    returns immediately, `collect()` returns the detections of the oldest batch in flight.  The H2D copy of a
    batch overlaps the kernels of the batch before it (the reference's Inferer is strictly serial,
    core/inferer.py:70-82)."""

    def __init__(self, model, batch, height, width, depth=2, **kw):
        dev = next(model.parameters()).device
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.pipes = [DetectPipeline(model, batch, height, width, host_input=True, overlap_h2d=True,
                                     copy_stream=self.copy_stream, **kw) for _ in range(depth)]
        self.done = [torch.cuda.Event() for _ in range(depth)]
        self.head = self.tail = 0          # submitted / collected counters

    def submit(self, images):
        assert self.head - self.tail < len(self.pipes), "collect() a batch before submitting another"
        p = self.pipes[self.head % len(self.pipes)]
        p.x_host.copy_(images)
        p.launch()
        self.done[self.head % len(self.pipes)].record(torch.cuda.current_stream(p.dev))
        self.head += 1

    def collect(self):
        assert self.tail < self.head, "nothing in flight"
        i = self.tail % len(self.pipes)
        self.done[i].synchronize()
        self.tail += 1
        return self.pipes[i].slot.rows(self.pipes[i].n_frames)


class DetectStream(_Served):
    """Software-pipelined serving loop: ONE graph launch per batch in which the network of batch i and the NMS of batch
    i - 1 are parallel branches.

    The NMS tail of a batch (candidate scan, top-K sort, greedy suppression: ~150 us for YOLOv6-S bs32, most of it on
    one CTA per image) leaves the tensor cores and most SMs idle, and the first network kernels of the next batch (stem,
    64-channel layers) are HBM-bound.  The head convs alternate between two (cls, reg) output sets (engine head_set 0 / 1);
    the graph of step i = { network(x_i) -> head set i & 1 }  ||  { NMS(head set 1 - (i & 1)) -> detections of batch i - 1 },
    joined at the end, so every dependency is a graph edge and the results are those of the serial pipeline, one step
    later.  `submit(images)` enqueues a step; `collect()` returns the detections of the oldest finished batch (None while
    the pipeline is still filling); `drain()` runs the NMS of the last submitted batch.  The reference's Inferer is
    strictly serial per batch (core/inferer.py:70-82).

    host_input=True: uint8 images come from pinned host memory (H2D of batch i + 1 on a copy stream under the kernels of
    batch i, as in DetectRing) and detections go back to pinned host memory inside the NMS branch.

    raw_input=True: `submit(frames, layout=...)` takes 1..B decoded uint8 frames of any sizes, host or CUDA (see the module
    docstring); the step graph letterboxes them before the network and the NMS branch rescales the previous batch's rows to
    its source pixels.
    """

    def __init__(self, model, batch, height, width, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
                 multi_label=False, max_det=300, host_input=True, engine=None, raw_input=False, max_src_bytes=None, auto=False,
                 source_shape=None, stride=None):
        super().__init__(model, batch, height, width, dict(conf_thres=conf_thres, iou_thres=iou_thres, classes=classes,
                         agnostic=agnostic, multi_label=multi_label, max_det=max_det), host_input, raw_input, max_src_bytes, 2,
                         engine, auto, source_shape, stride)
        self.B = batch
        self.x_dev = [s.x_dev for s in self.slots]
        self.x_host = [s.x_host for s in self.slots] if self.slots[0].x_host is not None else None
        self.n_frames = {}        # batch number -> frames in it (raw_input)
        self.dev_step, self.dev_drain = {}, {}      # head set -> (out, count, overflow) device tensors of the step / drain graphs
        self.fork_at_neck = os.environ.get("YV6_NMS_FORK", "neck") == "neck"
        self._drained = False
        self.side = torch.cuda.Stream(device=self.dev)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.ev_fork, self.ev_join = torch.cuda.Event(), torch.cuda.Event()
        self.steps = 0            # submitted batches
        self.collected = 0

        def warm():
            for k in (0, 1, 0, 1):     # both head sets exist and hold valid scores before anything is captured
                self.slots[k].letterbox()
                self.eng.forward(self.x_dev[k], decode=False, head_set=k)
                self._nms(k, {})
        g = self._capture(warm, [f for k in (0, 1) for f in (lambda k=k: self._body(k), lambda k=k: self._nms(k, self.dev_drain))])
        self.graphs, self.drain_graphs = g[0::2], g[1::2]

    def _nms(self, k, store):
        """NMS over head set k -> result slot k (pinned host when host_input; the device tensors go to `store[k]`)."""
        store[k] = self.slots[k].detect(self.nms, *self.eng.head_outputs(*self.shape, head_set=k))

    def _body(self, k):
        cur = torch.cuda.current_stream(self.dev)

        def fork():
            self.ev_fork.record(cur)
            self.side.wait_event(self.ev_fork)
            with torch.cuda.stream(self.side):
                self._nms(1 - k, self.dev_step)                # previous batch
                self.ev_join.record(self.side)

        # The branch starts where the backbone ends: the neck / head launches are single waves of <= 128 CTAs that leave SMs
        # idle, whereas next to the backbone's persistent one-CTA-per-SM kernels the one-CTA-per-image NMS kernels just take SMs away
        # (forking at the start of the step gains 2 %, measured).
        at = self.eng.neck_start(*self.shape) if self.fork_at_neck else 0
        self.slots[k].letterbox()
        self.eng.forward(self.x_dev[k], decode=False, head_set=k, hook=(at, fork))
        cur.wait_event(self.ev_join)

    def launch(self):
        """Enqueue one step on the current stream (input of slot steps & 1 already in x_host / x_dev); asynchronous.  It runs
        after the last refold of the engine (InferEngine.refold)."""
        slot = self.slots[self.steps & 1]
        cur = torch.cuda.current_stream(self.dev)
        if self.host_input:
            slot.h2d(self.copy_stream, cur)
        self.eng.after_fold(cur)
        self.graphs[self.steps & 1].replay()
        slot.done(cur)
        self.steps += 1

    def submit(self, images, layout="bgr_hwc", ready=None):
        """Enqueue batch number `steps`.  Its graph also post-processes batch steps - 1 into the result slot that batch
        steps - 3 used, so at most two batches may be waiting for `collect()`.  With raw_input, device frames are read after
        the work enqueued before this call on the current stream, or after the event `ready` when one is given."""
        if self.steps - self.collected > 2:
            raise RuntimeError("DetectStream: collect() the oldest batch before submitting another (result slots would be overwritten)")
        slot = self.slots[self.steps & 1]
        if self.host_input and slot.used:
            slot.ev_done.synchronize()          # the step two submissions ago has copied x_host and read the frames
        slot.stage(images, layout, ready)
        if slot.raw:
            self.n_frames[self.steps] = len(images)
        self._drained = False
        self.launch()

    def collect(self):
        """Detections of the oldest uncollected batch: batch t is post-processed by step t + 1 (or by `drain()` when it is
        the last one).  Returns None while that has not been enqueued yet."""
        t = self.collected
        if t >= self.steps:
            return None
        if t + 1 < self.steps:
            self.slots[(t + 1) & 1].ev_done.synchronize()
            store = self.dev_step
        elif self._drained:
            torch.cuda.current_stream(self.dev).synchronize()
            store = self.dev_drain
        else:
            return None
        self.collected += 1
        return self.slots[t & 1].rows(self.n_frames.pop(t, self.B), None if self.host_input else store[t & 1])

    def drain(self):
        """NMS of the last submitted batch (nothing follows it in the pipeline)."""
        if self.steps == 0 or self._drained or self.collected >= self.steps:
            return
        self.drain_graphs[(self.steps - 1) & 1].replay()
        self._drained = True


class DetectFarm:
    """`lanes` independent DetectStreams -- each with its own inference engine (own activation buffers) and its own CUDA
    stream -- fed round-robin.  Batches of different lanes have no dependency on each other, so the GPU runs the tail of
    one lane's kernel (the CTAs still working on their last tile of a 3.24-wave layer, an exposed epilogue, the launch gap
    before the next dependent kernel) next to the head of the other lane's kernel: the persistent conv kernels hold one CTA
    per SM, so the lanes interleave kernel by kernel rather than share SMs, and what one lane leaves idle the other fills.
    Costs `lanes` x the activation memory (YOLOv6-S bs32: ~2.3 GB per lane).  Per-lane results are those of DetectStream
    (bit-identical to the serial path); batch order across lanes is the submission order.  `.canvas` is the lanes' input
    shape (with auto=True, the rect canvas of `source_shape`)."""

    def __init__(self, model, batch, height, width, lanes=2, **kw):
        from .engine import InferEngine
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        self.streams = [torch.cuda.Stream(device=self.dev) for _ in range(lanes)]
        self.lanes = []
        for i in range(lanes):
            eng = model.engine() if i == 0 else InferEngine(model.graph, model.state_dict(), self.dev, model.precision)
            self.lanes.append(DetectStream(model, batch, height, width, engine=eng, **kw))
        self.canvas = self.lanes[0].canvas
        self.n = 0
        self._ev = [torch.cuda.Event() for _ in range(lanes)]
        self._go = torch.cuda.Event()
        self._ready = torch.cuda.Event()

    def lane_of_next(self):
        return self.lanes[self.n % len(self.lanes)]

    def launch(self):
        i = self.n % len(self.lanes)
        with torch.cuda.stream(self.streams[i]):
            self.lanes[i].launch()
        self.n += 1

    def submit(self, images, layout="bgr_hwc"):
        i = self.n % len(self.lanes)
        # recorded on the caller's stream, where device frames were produced, before the lane's stream becomes current
        self._ready.record(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.streams[i]):
            self.lanes[i].submit(images, layout=layout, ready=self._ready)
        self.n += 1

    def fence(self):
        """The current stream waits for everything enqueued on the lanes."""
        cur = torch.cuda.current_stream(self.dev)
        for ev, st in zip(self._ev, self.streams):
            ev.record(st)
            cur.wait_event(ev)

    def load_weights_(self, src):
        """Load new weights into the model and every lane, in place: Model.load_weights_ for the model (and its engine), then
        InferEngine.refold of each lane's engine.  No graph is recaptured; each lane's next step runs after the fold of its
        engine, and each fold after the lane's batches in flight (InferEngine.refold).  A source whose BottleRep alpha differs
        raises refold.AlphaChanged before any lane is written."""
        from .refold import weight_source
        flat, slots, ints = weight_source(src, self.dev)      # staged once for the model and every lane
        self.model._load_flat_(flat, slots, ints)
        for lane in self.lanes:
            if lane.eng is not self.model.__dict__.get("_engine"):
                lane.eng.refold(flat, slots)
        return self

    def release(self):
        """The lanes wait for everything enqueued on the current stream (e.g. a timing event)."""
        self._go.record(torch.cuda.current_stream(self.dev))
        for st in self.streams:
            st.wait_event(self._go)
