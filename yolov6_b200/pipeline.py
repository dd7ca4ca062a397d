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
done); the pipeline keeps a reference to them until then, so dropping them early is safe.
"""
import torch

from .nms import nms_batched_head, workspace_bytes
from .preprocess import GEO, REC, check_frames, letterbox_frames_launch, pack_sources, rescale_launch

RAW_DEFAULT_BYTES = 1920 * 1080 * 3        # staging bytes per batch slot when max_src_bytes is not given: one 1080p frame each


def raw_buffers(batch, height, width, max_det, max_src_bytes, dev):
    """Pinned staging + device buffers of one raw-frame slot."""
    cap = int(max_src_bytes) if max_src_bytes else batch * RAW_DEFAULT_BYTES
    geo = torch.tensor([[0, height, width, 0, 0, 0, 0, 0]] * batch, dtype=torch.int32)     # all border until frames arrive
    rec = torch.zeros(batch * REC, dtype=torch.uint8)          # null records: an all-border slot reads no source
    return dict(src_host=torch.empty(cap, dtype=torch.uint8).pin_memory(), geo_host=geo.pin_memory(), rec_host=rec.pin_memory(),
                src_dev=torch.zeros(cap, dtype=torch.uint8, device=dev), geo_dev=geo.to(dev), rec_dev=rec.to(dev), res_geo=geo.to(dev),
                res=torch.zeros(batch, max_det, 6, device=dev), nbytes=0, frames=[])


def raw_pack(slot, frames, height, width, layout, dev):
    """Validate 1..B frames and lay them out in one raw-frame slot's host tables; RuntimeError before anything is written
    when a frame is unusable.  Returns the device frames (read in place by the slot's next launch)."""
    srcs = check_frames(frames, slot["geo_host"].shape[0], layout, dev)
    slot["nbytes"], _, devs = pack_sources(srcs, slot["geo_host"].shape[0], height, width, True, layout, slot["src_host"],
                                           slot["geo_host"], slot["rec_host"], slot["src_dev"].data_ptr())
    return devs


def raw_h2d(slot):
    """Copy the used staging bytes, the source records and the geometry of one raw-frame slot to the device (current stream)."""
    n = slot["nbytes"]
    if n:
        slot["src_dev"][:n].copy_(slot["src_host"][:n], non_blocking=True)
    slot["rec_dev"].copy_(slot["rec_host"], non_blocking=True)
    slot["geo_dev"].copy_(slot["geo_host"], non_blocking=True)


class DetectPipeline:
    def __init__(self, model, batch, height, width, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
                 multi_label=False, max_det=300, host_input=True, overlap_h2d=False, copy_stream=None, raw_input=False,
                 max_src_bytes=None):
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError("DetectPipeline needs a CUDA model")
        if raw_input and not host_input:
            raise RuntimeError("DetectPipeline: raw_input returns detections in host memory (host_input=True)")
        self.kw = dict(conf_thres=conf_thres, iou_thres=iou_thres, classes=classes, agnostic=agnostic,
                       multi_label=multi_label, max_det=max_det)
        self.host_input = host_input
        self.raw = raw_input and raw_buffers(batch, height, width, max_det, max_src_bytes, self.dev)
        self.n_frames = batch
        self.overlap_h2d = bool((overlap_h2d or raw_input) and host_input)
        if self.overlap_h2d:
            self.copy_stream = copy_stream or torch.cuda.Stream(device=self.dev)
            self.ev_copied = torch.cuda.Event()
            self.ev_done = torch.cuda.Event()
            self.ev_ready = torch.cuda.Event()
            self._ready = None       # event the next copy waits for: the caller's stream when device frames were given
            self._used = False
        dt = torch.uint8 if host_input else torch.float32
        self.x_dev = torch.zeros(batch, 3, height, width, dtype=dt, device=self.dev)
        self.x_host = torch.zeros(batch, 3, height, width, dtype=torch.uint8).pin_memory() if host_input and not self.raw else None
        self.out_host = torch.zeros(batch, max_det, 6).pin_memory()
        self.count_host = torch.zeros(batch + 1, dtype=torch.int32).pin_memory()
        self.eng = model.engine()
        self.eng.pin(batch, height, width, dt)          # the graph points at this shape's buffers
        A = sum((height // int(s)) * (width // int(s)) for s in model.graph.strides)
        nc = model.graph.num_classes
        # scratch owned by this pipeline: a shared cache could be replaced (freed) while the graph still references it
        self.nms_ws = torch.empty(workspace_bytes(batch, A, nc, multi_label), dtype=torch.uint8, device=self.dev)
        self.graph = None
        self._warm()

    def _body(self):
        if self.raw:
            letterbox_frames_launch(self.raw["rec_dev"], self.raw["geo_dev"], self.x_dev)
        elif self.host_input and not self.overlap_h2d:
            self.x_dev.copy_(self.x_host, non_blocking=True)
        # the [B, A, 5+nc] prediction tensor of Detect.forward (effidehead.py:131-139) is never materialised here: the NMS
        # kernels scan the class scores where the cls_pred convs wrote them and decode boxes for the candidates only
        cls, reg, sizes = self.eng.forward(self.x_dev, decode=False)
        out, count, src, overflow = nms_batched_head(cls, reg, sizes, self.model.graph.strides, workspace=self.nms_ws, **self.kw)
        if self.raw:
            out = rescale_launch(out, count, self.raw["geo_dev"], self.x_dev.shape[2], self.x_dev.shape[3], res=self.raw["res"])
        self.out_dev, self.count_dev = out, count
        if self.host_input:
            self.out_host.copy_(out, non_blocking=True)
            self.count_host[:-1].copy_(count, non_blocking=True)
            self.count_host[-1:].copy_(overflow, non_blocking=True)

    def _warm(self):
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(2):     # plans, tensor maps, cudaFuncSetAttribute, allocator warm-up
                self._body()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self._body()

    def launch(self):
        """Enqueue one batch (input already in `x_host` / `x_dev`); asynchronous."""
        if self.overlap_h2d:
            cur = torch.cuda.current_stream(self.dev)
            if self._used:
                self.copy_stream.wait_event(self.ev_done)      # the previous batch of THIS pipeline is done with x_dev
            if self._ready is not None:
                self.copy_stream.wait_event(self._ready)       # the producer of the device frames
                self._ready = None
            with torch.cuda.stream(self.copy_stream):
                if self.raw:
                    raw_h2d(self.raw)
                else:
                    self.x_dev.copy_(self.x_host, non_blocking=True)
                self.ev_copied.record(self.copy_stream)
            cur.wait_event(self.ev_copied)
            self.graph.replay()
            self.ev_done.record(cur)
            self._used = True
            return
        self.graph.replay()

    def __call__(self, images=None, layout="bgr_hwc"):
        """images: uint8 [B,3,H,W] host tensor (host_input) or fp32 device tensor; with raw_input, a list of 1..B uint8 frames
        in `layout` (see the module docstring), each a numpy array, a CPU tensor or a CUDA tensor on the pipeline's device.
        Returns the list of per-image [k,6] detections (host tensors when host_input) like `non_max_suppression`; with
        raw_input in source pixels, rounded (Inferer.rescale(...).round())."""
        devs = None          # device frames of this batch, referenced until the batch is done
        if images is not None:
            if self.raw:
                devs = raw_pack(self.raw, images, self.x_dev.shape[2], self.x_dev.shape[3], layout, self.dev)
                if devs:
                    self.ev_ready.record(torch.cuda.current_stream(self.dev))
                    self._ready = self.ev_ready
                self.n_frames = len(images)
            else:
                (self.x_host if self.host_input else self.x_dev).copy_(images)
        self.launch()
        torch.cuda.current_stream(self.dev).synchronize()
        if self.host_input:
            counts = self.count_host.tolist()
            if counts[-1]:
                raise RuntimeError("non_max_suppression: more than 65536 near-identical candidate scores in one image; raise conf_thres")
            return [self.out_host[i, :counts[i]].clone() for i in range(self.n_frames)]
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
        p = self.pipes[i]
        counts = p.count_host.tolist()
        self.tail += 1
        if counts[-1]:
            raise RuntimeError("non_max_suppression: more than 65536 near-identical candidate scores in one image; raise conf_thres")
        return [p.out_host[j, :counts[j]].clone() for j in range(p.out_host.shape[0])]


class DetectStream:
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
                 multi_label=False, max_det=300, host_input=True, engine=None, raw_input=False, max_src_bytes=None):
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError("DetectStream needs a CUDA model")
        if raw_input and not host_input:
            raise RuntimeError("DetectStream: raw_input returns detections in host memory (host_input=True)")
        self.kw = dict(conf_thres=conf_thres, iou_thres=iou_thres, classes=classes, agnostic=agnostic,
                       multi_label=multi_label, max_det=max_det)
        self.host_input = bool(host_input)
        self.B = batch
        dt = torch.uint8 if host_input else torch.float32
        self.x_dev = [torch.zeros(batch, 3, height, width, dtype=dt, device=self.dev) for _ in range(2)]
        self.raw = [raw_buffers(batch, height, width, max_det, max_src_bytes, self.dev) for _ in range(2)] if raw_input else None
        self.n_frames = {}        # batch number -> frames in it (raw_input)
        self.x_host = ([torch.zeros(batch, 3, height, width, dtype=torch.uint8).pin_memory() for _ in range(2)]
                       if host_input and not raw_input else None)
        self.out_host = [torch.zeros(batch, max_det, 6).pin_memory() for _ in range(2)]
        self.count_host = [torch.zeros(batch + 1, dtype=torch.int32).pin_memory() for _ in range(2)]
        self.dev_step, self.dev_drain = {}, {}      # head set -> (out, count, overflow) device tensors of the step / drain graphs
        import os
        self.fork_at_neck = os.environ.get("YV6_NMS_FORK", "neck") == "neck"
        self._drained = False
        self.eng = engine if engine is not None else model.engine()
        self.eng.pin(batch, height, width, dt)
        self.shape = (batch, height, width, dt)
        self.sizes = [(height // int(s), width // int(s)) for s in model.graph.strides]
        A = sum(h * w for h, w in self.sizes)
        self.nms_ws = torch.empty(workspace_bytes(batch, A, model.graph.num_classes, multi_label), dtype=torch.uint8, device=self.dev)
        self.side = torch.cuda.Stream(device=self.dev)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.ev_fork, self.ev_join = torch.cuda.Event(), torch.cuda.Event()
        self.ev_copied = [torch.cuda.Event(), torch.cuda.Event()]
        self.ev_done = [torch.cuda.Event(), torch.cuda.Event()]
        self.ev_ready = torch.cuda.Event()
        self._ready = None        # event the next copy waits for: the producer of the submitted device frames
        self.steps = 0            # submitted batches
        self.collected = 0
        self.graphs = [None, None]
        self.drain_graphs = [None, None]
        self._build()

    def _nms(self, k, store):
        """NMS over head set k -> result slot k (pinned host when host_input; the device tensors go to `store[k]`)."""
        cls, reg = self.eng.head_outputs(*self.shape, head_set=k)
        out, count, src, overflow = nms_batched_head(cls, reg, self.sizes, self.model.graph.strides, workspace=self.nms_ws, **self.kw)
        if self.raw:
            # res_geo[k] is the geometry of the batch whose network wrote head set k: the copy stream may already be refilling
            # geo_dev[k] with the batch after next
            out = rescale_launch(out, count, self.raw[k]["res_geo"], self.x_dev[k].shape[2], self.x_dev[k].shape[3], res=self.raw[k]["res"])
        store[k] = (out, count, overflow)
        if self.host_input:
            self.out_host[k].copy_(out, non_blocking=True)
            self.count_host[k][:-1].copy_(count, non_blocking=True)
            self.count_host[k][-1:].copy_(overflow, non_blocking=True)

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
        self._letterbox(k)
        self.eng.forward(self.x_dev[k], decode=False, head_set=k, hook=(at, fork))
        cur.wait_event(self.ev_join)

    def _letterbox(self, k):
        if self.raw:
            letterbox_frames_launch(self.raw[k]["rec_dev"], self.raw[k]["geo_dev"], self.x_dev[k])
            self.raw[k]["res_geo"].copy_(self.raw[k]["geo_dev"])

    def _build(self):
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            for k in (0, 1, 0, 1):     # both head sets exist and hold valid scores before anything is captured
                self._letterbox(k)
                self.eng.forward(self.x_dev[k], decode=False, head_set=k)
                self._nms(k, {})
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        for k in (0, 1):
            self.graphs[k] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graphs[k]), torch.no_grad():
                self._body(k)
            self.drain_graphs[k] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.drain_graphs[k]), torch.no_grad():
                self._nms(k, self.dev_drain)

    def launch(self):
        """Enqueue one step on the current stream (input of slot steps & 1 already in x_host / x_dev); asynchronous."""
        k = self.steps & 1
        cur = torch.cuda.current_stream(self.dev)
        if self.host_input:
            if self.steps >= 2:
                self.copy_stream.wait_event(self.ev_done[k])   # the step that last read x_dev[k] has finished
            if self._ready is not None:
                self.copy_stream.wait_event(self._ready)
                self._ready = None
            with torch.cuda.stream(self.copy_stream):
                if self.raw:
                    raw_h2d(self.raw[k])
                else:
                    self.x_dev[k].copy_(self.x_host[k], non_blocking=True)
                self.ev_copied[k].record(self.copy_stream)
            cur.wait_event(self.ev_copied[k])
        self.graphs[k].replay()
        self.ev_done[k].record(cur)
        self.steps += 1

    def submit(self, images, layout="bgr_hwc", ready=None):
        """Enqueue batch number `steps`.  Its graph also post-processes batch steps - 1 into the result slot that batch
        steps - 3 used, so at most two batches may be waiting for `collect()`.  With raw_input, device frames are read after
        the work enqueued before this call on the current stream, or after the event `ready` when one is given."""
        if self.steps - self.collected > 2:
            raise RuntimeError("DetectStream: collect() the oldest batch before submitting another (result slots would be overwritten)")
        k = self.steps & 1
        if self.host_input:
            if self.steps >= 2:
                self.ev_done[k].synchronize()                  # x_host[k] was copied by the step two submissions ago
            if self.raw:
                devs = raw_pack(self.raw[k], images, self.x_dev[k].shape[2], self.x_dev[k].shape[3], layout, self.dev)
                # the step that read the slot's previous device frames is complete (ev_done[k] above): release them now
                self.raw[k]["frames"] = devs
                # only device frames need it: the caller's stream usually holds the previous step, and a copy that waited for
                # it would no longer overlap that step
                if devs:
                    if ready is None:
                        ready = self.ev_ready
                        ready.record(torch.cuda.current_stream(self.dev))
                    self._ready = ready
                self.n_frames[self.steps] = len(images)
            else:
                self.x_host[k].copy_(images)
        else:
            self.x_dev[k].copy_(images)
        self._drained = False
        self.launch()

    def _results(self, k, store, n):
        if self.host_input:
            counts = self.count_host[k].tolist()
            if counts[-1]:
                raise RuntimeError("non_max_suppression: more than 65536 near-identical candidate scores in one image; raise conf_thres")
            return [self.out_host[k][j, :counts[j]].clone() for j in range(n)]
        out, count, overflow = store[k]
        if int(overflow.item()):
            raise RuntimeError("non_max_suppression: more than 65536 near-identical candidate scores in one image; raise conf_thres")
        counts = count.tolist()
        return [out[j, :counts[j]].clone() for j in range(self.B)]

    def collect(self):
        """Detections of the oldest uncollected batch: batch t is post-processed by step t + 1 (or by `drain()` when it is
        the last one).  Returns None while that has not been enqueued yet."""
        t = self.collected
        if t >= self.steps:
            return None
        if t + 1 < self.steps:
            self.ev_done[(t + 1) & 1].synchronize()
            store = self.dev_step
        elif self._drained:
            torch.cuda.current_stream(self.dev).synchronize()
            store = self.dev_drain
        else:
            return None
        self.collected += 1
        return self._results(t & 1, store, self.n_frames.pop(t, self.B))

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
    (bit-identical to the serial path); batch order across lanes is the submission order."""

    def __init__(self, model, batch, height, width, lanes=2, **kw):
        from .engine import InferEngine
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        self.streams = [torch.cuda.Stream(device=self.dev) for _ in range(lanes)]
        self.lanes = []
        for i in range(lanes):
            eng = model.engine() if i == 0 else InferEngine(model.graph, model.state_dict(), self.dev, model.precision)
            self.lanes.append(DetectStream(model, batch, height, width, engine=eng, **kw))
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

    def release(self):
        """The lanes wait for everything enqueued on the current stream (e.g. a timing event)."""
        self._go.record(torch.cuda.current_stream(self.dev))
        for st in self.streams:
            st.wait_event(self._go)
