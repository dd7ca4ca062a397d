"""Inference engine: walks the layer graph (arch.py) and issues one sm_90a kernel per op.

What the reference does with nested nn.Module.forward calls, cuDNN and ~15 eager ops for the head
decode (Model.forward yolo.py:33-41, Detect.forward effidehead.py:93-139), this does with:
  * folded deploy-form weights (fold.py's float64 fold, run on the device by yv6_fold: refold.py) packed to KRSC bf16 (or
    three bf16 planes), refoldable in place from new train-form weights (InferEngine.refold),
  * pre-allocated NHWC activation buffers (concats are channel slices),
  * a prepared list of C-ABI descriptors per input shape, replayed per batch -- optionally as one
    captured CUDA graph (no Python / launch overhead in steady state).
Precision modes: "bf16" (bf16 operands, fp32 accumulate), "fp16" (fp16 operands and activations, fp32 accumulate: the same
launches and tile plans as bf16, 3 more mantissa bits, activations beyond 65504 become inf as under the reference's --half) and
"fp32" (bf16x3 split operands: fp32-equivalent products, used for the 1e-4 parity bar of BASELINE.json).
"""
import ctypes as C
import itertools
import os
from dataclasses import dataclass

import torch

from . import _lib, ops, refold
from ._lib import ConvDesc


def siblings(g):
    """Pairs of convs that read the same tensor with the same geometry and can run as ONE launch over the
    concatenated output channels: the cls / reg branches of the decoupled head (effidehead.py:79-84).  {first: second}"""
    pairs = {}
    for i, a in enumerate(g.ops):
        if a.kind != "conv" or not a.name.startswith("detect.cls_convs."):
            continue
        for j in range(i + 1, min(i + 3, len(g.ops))):
            b = g.ops[j]
            if (b.kind == "conv" and b.name == a.name.replace("cls_convs", "reg_convs") and b.src == a.src and
                    (b.k, b.s, b.act, b.cout, b.cin) == (a.k, a.s, a.act, a.cout, a.cin) and a.res is None and b.res is None and
                    a.dst.c_off == 0 and b.dst.c_off == 0 and a.cout % 64 == 0):
                pairs[i] = j
    return pairs


def sibling_slices(g, sibling):
    """Sibling convs write one [.., 2 x Cout] buffer and their consumers read its two channel halves:
    graph buffer index -> (first conv of the pair, channel offset, channel pitch) in that buffer."""
    out = {}
    for i, j in sibling.items():
        c = g.ops[i].cout
        out[g.ops[i].dst.buf] = (i, 0, 2 * c)
        out[g.ops[j].dst.buf] = (i, c, 2 * c)
    return out


def pair_view_candidate(op):
    """3x3 stride-2 convs over <= 32 channels, or over 64 | 128 (the view's zero blocks are skipped there): the convs that get
    column-pair-view weights and may run on the view (pair_view)."""
    return op.kind == "conv" and op.k == 3 and op.s == 2 and (op.cin <= 32 or op.cin in (64, 128))


def pair_view(d, w_pair, plan_fn):
    """Descriptor d of a 3x3 stride-2 conv, moved onto the column-pair view of the same memory where that pays; d otherwise.

    On the view, [N, H, W/2, 2*Cin] with the weights w_pair (ops.pair_view_weights), it is a 3x2 conv with stride (2, 1) over
    contiguous 2*Cin-channel rows.  <= 32 channels: 64-byte pixels fetched with an element stride of 2 keep the TMA unit, not the
    tensor pipe, busy (ERBlock_2.0 of YOLOv6-S: 170 -> 135 us).  More channels: kept only where the library's halo-reuse
    mainloop takes the view (plan_fn(view)["halo"] == 2; one 9 x 33 input box per 8 x 16 output tile instead of one box per tap,
    include/yv6.h `pair_view`), so the input operand crosses L2 -> shared memory 2.6x less often, which is what bounds these
    small-K layers; on the generic mainloop the plain stride-2 conv moves fewer bytes.  Needs an unsliced input of even width."""
    if d.x_c_total != d.Cin or d.W % 2:
        return d
    v = ConvDesc.from_buffer_copy(d)
    v.W, v.Cin, v.x_c_total = d.W // 2, 2 * d.Cin, 2 * d.Cin
    v.w, v.w_plane_stride = w_pair, d.w_plane_stride // 9 * 12          # planes of [Cout][3][2][2*Cin] instead of [Cout][3][3][Cin]
    v.kw, v.stride_w, v.pad_w, v.out_w, v.pair_view = 2, 1, 1, d.W // 2, 1
    return v if d.Cin <= 32 or plan_fn(v)["halo"] == 2 else d


def conv_window(g, op):
    """Input channels [lo, hi) a conv / pred launch reads.  On the Lite graphs (arch.LiteGraph: 16-aligned pitches, zero pad
    channels) that is the 16-aligned window around the op's slice, so that the conv kernel's Cin % 16 == 0 and 16-byte
    alignment hold for any slice; window_weights gives the columns outside the slice zero weight.  Elsewhere it is the slice."""
    a, c = op.src.c_off, op.src.c
    if not g.lite:
        return a, a + c
    return a // 16 * 16, (a + c + 15) // 16 * 16


def window_weights(g, op, w):
    """KRSC weights [Cout, k, k, Cin] of a conv / pred op -> [Cout, k, k, hi - lo] over its conv_window, zero outside the slice."""
    lo, hi = conv_window(g, op)
    if (lo, hi) == (op.src.c_off, op.src.c_off + op.src.c):
        return w
    out = w.new_zeros(w.shape[:3] + (hi - lo,))
    out[..., op.src.c_off - lo:op.src.c_off - lo + op.src.c] = w
    return out


def stem_channels(g, op):
    """Channels the stem writes: its buffer's pitch (the Lite stem: 24 real + 8 zero-weight channels, Hardswish(0) = 0)."""
    return g.bufs[op.dst.buf].c_total


@dataclass(eq=False)
class InferLaunch(ops.Launch):
    """One launch of the inference forward (ops.Launch) with what the scheduler and the profilers need: the op `name`, the
    (buffer, first channel, end channel) spans it `reads` and `writes` -- buffers are ("buf", graph buffer index), ("fused",
    first conv of a sibling pair) or ("head", "cls" | "reg", level) --, `head` "cls" | "reg" for a head conv (its output moves
    with the head set), and for a conv launch `conv`: its geometry (cin, cout, k, s, input h, w, output ho, wo), algorithmic
    `flops` (the column-pair view's zero taps do not count) and `y_f32`.

    `writes` covers every element the launch stores.  `reads` covers every element whose value reaches the output; a conv of
    a Lite graph also loads the rest of its 16-aligned channel window (conv_window), through weights that are zero in every
    plane, and those channels are not declared: any finite value there contributes exactly 0, so the schedule need not order
    the launch after their writers."""
    name: str = ""
    reads: tuple = ()
    writes: tuple = ()
    head: str = None
    conv: dict = None


def _viewer(g, N, H, W, sibling, addr):
    """view(t) -> (buffer key, address, channel offset, (N, h, w, channel pitch)) of graph tensor slice t: buffers are ("buf",
    graph buffer index) or, for the outputs of a sibling pair, ("fused", first conv of the pair)."""
    slices = sibling_slices(g, sibling)

    def view(t):
        b = g.bufs[t.buf]
        nhw = (N, H >> b.level, W >> b.level)
        if t.buf in slices:
            i, c0, pitch = slices[t.buf]
            return ("fused", i), addr("fused", i), c0 + t.c_off, nhw + (pitch,)
        return ("buf", t.buf), addr("buf", t.buf), t.c_off, nhw + (b.c_total,)
    return view


def conv_launches(g, N, H, W, nsplit, sibling, addr, plan_fn, f16=False):
    """Descriptors of the conv launches of one inference forward of graph g over an [N, 3, H, W] input, in launch order:
    {op index: [ConvDesc, ...]} -- four 1x1 quadrant launches for a transposed conv, one otherwise; the first conv of a sibling pair
    computes both.  Descriptors only: no allocation and no CUDA call, so the planner can be checked on these launches without a GPU.

    nsplit: 1 (bf16, or fp16 if f16) or 3 (bf16x3 planes); sibling: siblings(g) or {}.  addr(kind, key, q=0) resolves device addresses:
    ("buf", buffer index) activation buffers, ("fused", first conv of the pair) the [.., 2 x Cout] sibling outputs,
    ("head", "cls" | "reg") the [N, A, ch] fp32 head tensors, ("w", op index, quadrant q of a transposed conv) packed weights,
    ("w_pair" | "w_fused" | "bias" | "bias_fused", op index) the other packed weights and padded biases; ("alpha", op index) is
    the residual scale.
    plan_fn(desc) -> plan dict (ops.PLAN_KEYS) decides where the column-pair view is kept."""
    offs = list(itertools.accumulate(((H // s) * (W // s) for s in g.strides), initial=0))    # first anchor of each level
    A = offs[-1]
    view = _viewer(g, N, H, W, sibling, addr)
    second = set(sibling.values())
    out = {}
    for i, op in enumerate(g.ops):
        if op.kind not in ("conv", "pred", "convT") or i in second:
            continue                      # the second conv of a sibling pair is computed by the first one's launch
        if op.kind == "pred" and op.head[0] not in ("cls", "reg"):
            continue                      # eval forward: anchor-free (cls, reg) branches only (effidehead_fuseab.py:141-199, _distill_ns.py:105-150)
        fused = i in sibling
        _, x, x_off, xs = view(op.src)
        k, s = (1, 1) if op.kind == "convT" else (op.k, op.s)
        cin = op.cin
        if op.kind != "convT":
            lo, hi = conv_window(g, op)
            x_off, cin = x_off - op.src.c_off + lo, hi - lo
        ws = (2 * op.cout if fused else op.cout, k, k, cin)
        kw = dict(x_c_off=x_off, bias=addr("bias_fused" if fused else "bias", i), stride=s, act=op.act, nsplit=nsplit, f16=f16)
        if op.res is not None:
            _, r, r_off, (_, rh, rw, rct) = view(op.res)
            kw.update(res=r, res_c_off=r_off, res_strides=(rh * rw * rct, rw * rct, rct), alpha=addr("alpha", i))
        if op.kind == "pred":
            which, lvl = op.head
            ch, lw = op.cout, W // g.strides[lvl]
            out[i] = [ops.conv_desc(x, xs, addr("w", i), ws, addr("head", which), (A * ch, lw * ch, ch), y_elem_off=offs[lvl] * ch,
                                    y_f32=True, **kw)]
            continue
        _, y, y_off, (_, dh, dw, dct) = view(op.dst)
        if op.kind == "convT":           # scatter quadrant (dy, dx) of the 2x upsample
            out[i] = [ops.conv_desc(x, xs, addr("w", i, q), ws, y, (dh * dw * dct, 2 * dw * dct, 2 * dct), y_c_off=y_off,
                                    y_elem_off=(q // 2 * dw + q % 2) * dct, **kw) for q in range(4)]
            continue
        d = ops.conv_desc(x, xs, addr("w_fused" if fused else "w", i), ws, y, (dh * dw * dct, dw * dct, dct), y_c_off=y_off, **kw)
        if pair_view_candidate(op):
            d = pair_view(d, addr("w_pair", i), plan_fn)
        out[i] = [d]
    return out


def forward_launches(g, N, H, W, nsplit, addr, plan_fn, u8=False, f16=False):
    """Every launch of one inference forward of graph g over an [N, 3, H, W] input (uint8 if u8), in launch order, as InferLaunch
    records: stem, the conv launches of conv_launches (the fused head siblings of siblings(g) included), SPPF pool, depthwise
    conv, SE, channel shuffle, upsample (the head decode is not included).  Records only: no allocation and no CUDA call, so the
    launches can be checked without a GPU.  The stem's input address is 0 (set per forward).

    nsplit, addr, plan_fn and f16 (fp16 activations: the _f16 entry points, fp16 descriptors) as for conv_launches; addr also
    resolves ("w_dev" | "b_dev" | "w1" | "b1" | "w2" | "b2", op index):
    the stem, depthwise and SE weights and biases."""
    sibling = siblings(g)
    convs = conv_launches(g, N, H, W, nsplit, sibling, addr, plan_fn, f16)
    sfx = "_f16" if f16 else ""
    view = _viewer(g, N, H, W, sibling, addr)

    def span(t):
        key, _, c0, _ = view(t)
        return (key, c0, c0 + t.c)

    def at(t):
        """(address of the slice's first channel, channel pitch, plane stride) of graph tensor slice t."""
        _, a, c0, (n, h, w, pitch) = view(t)
        return a + 2 * c0, pitch, n * h * w * pitch if nsplit == 3 else 0

    out = []
    for i, op in enumerate(g.ops):
        rec = dict(name=op.name)
        if op.kind == "stem":         # writes its buffer's whole pitch (the Lite stem's zero pad channels included)
            key, y, c0, (_, h, w, pitch) = view(op.dst)
            assert c0 == 0
            d = ops.stem_desc(0, N, H, W, u8, addr("w_dev", i), addr("b_dev", i), stem_channels(g, op), op.act, y, nsplit,
                              N * h * w * pitch if nsplit == 3 else 0)
            out.append(InferLaunch("stem", "yv6_stem_fwd" + sfx, (C.byref(d),), d, writes=[(key, 0, stem_channels(g, op))], **rec))
        elif op.kind in ("pool", "dw", "se", "shuffle", "up"):
            (x, xp, xpl), (_, _, _, (_, h, w, _)) = at(op.src), view(op.src)
            if op.kind == "pool":      # in place: channels [0, C) -> [C, 4C) of one buffer
                key, y, _, (_, h, w, ct) = view(op.dst)
                out.append(InferLaunch("pool", "yv6_sppf_pool" + sfx, (y, N, h, w, op.cin, ct, nsplit, N * h * w * ct if nsplit == 3 else 0),
                                       reads=[(key, 0, op.cin)], writes=[(key, op.cin, 4 * op.cin)], **rec))
            elif op.kind == "dw":
                y, yp, ypl = at(op.dst)
                d = ops.dw_desc(x, (N, h, w, xp), xpl, addr("w_dev", i), addr("b_dev", i), op.cin, op.k, op.s, op.act, y, yp, ypl, nsplit)
                out.append(InferLaunch("dw", "yv6_dwconv_fwd" + sfx, (C.byref(d),), d, reads=[span(op.src)], writes=[span(op.dst)], **rec))
            elif op.kind == "se":      # in place
                d = ops.se_desc(x, N, h * w, op.cin, op.cout, xp, xpl, *(addr(k, i) for k in ("w1", "b1", "w2", "b2")), nsplit=nsplit, f16=f16)
                out.append(InferLaunch("se", "yv6_se_fwd", (C.byref(d),), d, reads=[span(op.src)], writes=[span(op.src)], **rec))
            elif op.kind == "shuffle":
                out.append(InferLaunch("shuffle", "yv6_channel_shuffle", (x, xp, xpl, *at(op.src2), N * h * w, op.cin, *at(op.dst), nsplit),
                                       reads=[span(op.src), span(op.src2)], writes=[span(op.dst)], **rec))
            else:
                out.append(InferLaunch("up", "yv6_upsample2x", (x, xp, xpl, N, h, w, op.cin, *at(op.dst), nsplit),
                                       reads=[span(op.src)], writes=[span(op.dst)], **rec))
        elif i in convs:
            rec["reads"] = [span(op.src)] + ([span(op.res)] if op.res is not None else [])
            if op.kind == "pred":
                rec.update(head=op.head[0], writes=[(("head",) + tuple(op.head), 0, 1)])
            else:
                rec["writes"] = [(("fused", i), 0, 2 * op.cout) if i in sibling else span(op.dst)]
            _, _, _, (_, sh, sw, _) = view(op.src)
            for q, d in enumerate(convs[i]):
                k, s = d.kh, d.stride      # (of the 3x3 stride-2 conv, also on the column-pair view)
                oh, ow = (sh + 2 * (k // 2) - k) // s + 1, (sw + 2 * (k // 2) - k) // s + 1
                geom = dict(name=op.name if op.kind != "convT" else f"{op.name}[{q}]", cin=op.cin, cout=d.Cout, k=k, s=s, ho=oh, wo=ow,
                            h=sh, w=sw, flops=2.0 * N * oh * ow * d.Cout * op.cin * k * k, y_f32=op.kind == "pred")
                out.append(InferLaunch("conv", "yv6_conv_fwd", (C.byref(d),), d, conv=geom, **rec))
    return out


class _Plan:
    """Buffers, launch records and stream schedule of one input shape.  bufs: the graph's activation buffers; fused: first conv
    of a sibling pair -> the pair's [.., 2 x Cout] output; heads[k]: (cls [N,A,nc], reg [N,A,R]) fp32 of head set k (set 1 is
    allocated on first use); pred [N,A,5+nc]: the decoded output; launches: forward_launches' records; decode: the head decode
    launch; lane / waits / tails / events / fork: the stream schedule (InferEngine._schedule); neck_start: index of the first
    launch after the backbone; image: the input of the last forward (kept alive while its kernels run)."""


class InferEngine:
    def __init__(self, graph, state_dict, device, precision="bf16"):
        if device.type != "cuda":
            raise RuntimeError("yolov6_b200 runs its networks on sm_90a CUDA kernels only (no CPU fallback); "
                               f"got device {device}")
        assert precision in ("bf16", "fp16", "fp32")
        self.g = graph
        self.device = device
        self.precision = precision
        self.nsplit = 3 if precision == "fp32" else 1
        self.handle = _lib.handle(device.index or 0)
        self.lib = _lib.lib()
        self.n_lanes = int(os.environ.get("YV6_LANES", "4"))   # streams the launches of one forward are spread over (1 = serial)
        self._side = None
        self.weights = {}     # op index -> dict(w=..., bias=..., alpha=...)
        self._plans = {}      # (N, H, W, dtype) -> plan, least recently used first; bounded (rect-shaped evaluation
        self.max_plans = 4    # would otherwise keep one full activation set per distinct shape)
        self._pinned = set()  # shapes captured into CUDA graphs (their buffers must outlive the graph)
        self._pack(state_dict)

    @property
    def f16(self):
        """fp16 operands and activations (precision "fp16")."""
        return self.precision == "fp16"

    @property
    def act_dtype(self):
        """dtype of the activation buffers (bf16 planes in the fp32 mode)."""
        return torch.float16 if self.f16 else torch.bfloat16

    # ------------------------------------------------------------------ weight packing
    def _pack(self, sd):
        """Allocate the weight tensors (zeroed) and fold the state_dict sd into them: staged into one flat buffer on the
        engine's device and folded by yv6_fold (refold.py), then synchronized, as an upload would be."""
        self.sibling = siblings(self.g)
        for i, ent in refold.allocate(self.g, self.precision, self.device).items():
            op = self.g.ops[i]
            if op.kind != "se":
                ent["alpha"] = float(sd[op.alpha]) if (op.alpha and op.res is not None) else 1.0
            self.weights[i] = ent
        flat, slots = refold.stage(sd, self.device)
        self._fold(flat, slots)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()
            self._fold_ev = None

    def _resolve(self, dst):
        t = self.weights[dst[1]][dst[0]]
        return t[dst[2]] if dst[0] == "w" else t

    def _fold_plan(self, slots):
        plans = self.__dict__.setdefault("_fold_plans", {})
        key = refold.layout_key(self.g, slots)
        plan = plans.get(key)
        if plan is None:
            plan = plans[key] = refold.build_plan(self.g, self.precision, slots)
        return plan

    def _fold(self, flat, slots, stream=None):
        """Fold the state in flat (laid out as slots) into the weight tensors.  On the CUDA device the fold is enqueued on
        `stream` (default: the current stream) after the work already enqueued on the current stream, the batches in flight on
        the pipelines attached to this engine and the previous fold; fp16 runs the range check first (one host sync)."""
        plan = self._fold_plan(slots)
        if self.device.type != "cuda":          # a CPU-device engine (planner tests): the same records, executed on the host
            refold.replay_host(plan, flat, self._resolve)
            return
        if flat.device != self.device or flat.dtype != torch.float32 or not flat.is_contiguous():
            raise ValueError(f"refold: the source must be a contiguous fp32 tensor on {self.device}")
        tables = plan.dev.get(id(self))
        if tables is None:
            tables = plan.dev[id(self)] = refold.device_tables(plan, self._resolve, self.device)
        cur = torch.cuda.current_stream(self.device)
        s = stream if stream is not None else cur
        if s != cur:
            s.wait_stream(cur)
        for x in self._in_flight():
            if isinstance(x, torch.cuda.Event):
                s.wait_event(x)
            else:
                s.wait_stream(x)
        if self.__dict__.get("_fold_ev") is not None:
            s.wait_event(self._fold_ev)
        if self.f16:
            refold.device_check(self.lib, self.handle, plan, tables, flat, s)
        refold.launch(self.lib, self.handle, tables, flat, False, s)
        self._fold_ev = torch.cuda.Event()
        self._fold_ev.record(s)
        if s != cur:                      # the caching allocator must not recycle the source before the fold has read it
            flat.record_stream(s)
        self._fold_src = flat

    def _in_flight(self):
        """Events (or streams) of the batches in flight on the pipelines attached to this engine (pipeline.in_flight)."""
        out = []
        for p in list(self.__dict__.get("_users", ())):
            out += p.in_flight()
        return out

    def attach(self, pipeline):
        """Register a pipeline whose captured graphs run this engine: refold orders itself after its batches in flight, and
        the pipeline calls after_fold before each launch."""
        import weakref
        self.__dict__.setdefault("_users", weakref.WeakSet()).add(pipeline)

    def after_fold(self, stream):
        """Make `stream` wait for the last refold (nothing to do if the engine was never refolded)."""
        ev = self.__dict__.get("_fold_ev")
        if ev is not None:
            stream.wait_event(ev)

    def refold(self, src, slots, stream=None):
        """Rewrite the weights of this engine in place from the train-form state in the flat fp32 CUDA tensor `src`, laid out
        as `slots` ({name: (offset, numel, shape)}: FlatState.slots, or refold.stage of a state_dict).  Every plan, launch
        record and captured CUDA graph of the engine stays valid and runs the new weights.

        Stream order: the fold runs on `stream` (default: the current stream) after the work already enqueued on the current
        stream -- so after the last FusedSGDEMA step there when src is its `ema` -- and after the batches in flight on the
        pipelines built on this engine (the done events of their batch slots, or the stream a DetectPipeline without
        overlap_h2d last launched on); their next launch(), and the next eager forward, wait for it.  The source must not be
        overwritten until then (the engine keeps a reference).

        Raises refold.AlphaChanged (a ValueError) before anything is written when a BottleRep alpha of src differs from the one
        the engine was built with (it is baked into the conv descriptors), and in the fp16 mode fold.to_f16's ValueError, also
        before anything is written, when a folded weight is outside fp16's range."""
        if self.device.type != "cuda" or src.device != self.device:
            raise ValueError(f"refold: the source must be a CUDA tensor on {self.device}")
        alphas = [(i, op.alpha) for i, op in enumerate(self.g.ops) if op.alpha and op.res is not None and i in self.weights]
        if alphas:
            idx = torch.tensor([slots[a][0] for _, a in alphas], dtype=torch.int64, device=self.device)
            for (i, a), v in zip(alphas, src.index_select(0, idx).tolist()):
                if v != self.weights[i]["alpha"]:
                    raise refold.AlphaChanged(f"refold: {a} is {v!r}, the engine was built with {self.weights[i]['alpha']!r}; "
                                              "rebuild the engine (alpha is baked into its conv descriptors)")
        self._fold(src, slots, stream)

    # ------------------------------------------------------------------ per-shape plan
    def _plan(self, N, H, W, in_dtype):
        key = (N, H, W, in_dtype)
        if key in self._plans:
            plan = self._plans.pop(key)
            self._plans[key] = plan          # most recently used last
            return plan
        while len(self._plans) >= self.max_plans:
            victim = next((k for k in self._plans if k not in self._pinned), None)
            if victim is None:
                break
            del self._plans[victim]
        g, dev, P = self.g, self.device, self.nsplit
        maxs = max(g.strides)
        if H % maxs or W % maxs:
            raise RuntimeError(f"input {H}x{W} must be a multiple of the largest stride {maxs}")

        def zeros(level, c):
            shape = (N, H >> level, W >> level, c)
            return torch.zeros((P,) + shape if P == 3 else shape, dtype=self.act_dtype, device=dev)

        plan = _Plan()
        plan.bufs = [zeros(b.level, b.c_total) for b in g.bufs]
        plan.fused = {i: zeros(g.bufs[g.ops[i].dst.buf].level, 2 * g.ops[i].cout) for i in self.sibling}
        sizes = [(H // s, W // s) for s in g.strides]
        A, nc, R = sum(h * w for h, w in sizes), g.num_classes, 4 * (g.reg_max + 1)
        plan.heads = [(torch.empty(N, A, nc, dtype=torch.float32, device=dev), torch.empty(N, A, R, dtype=torch.float32, device=dev))]
        plan.pred = torch.empty(N, A, 5 + nc, dtype=torch.float32, device=dev)
        plan.sizes, plan.head_set, plan.image = sizes, 0, None

        def addr(kind, key, q=0):
            """Device addresses of this plan's tensors and the packed weights (see forward_launches)."""
            if kind in ("buf", "fused"):
                return (plan.bufs if kind == "buf" else plan.fused)[key].data_ptr()
            if kind == "head":
                return plan.heads[0][("cls", "reg").index(key)].data_ptr()
            if kind == "alpha":
                return self.weights[key]["alpha"]
            t = self.weights[key][kind]
            return (t[q] if kind == "w" else t).data_ptr()

        plan.launches = forward_launches(g, N, H, W, P, addr, lambda d: ops.plan_of(d, dev.index or 0), in_dtype == torch.uint8,
                                         self.f16)
        plan.stem = next(r.desc for r in plan.launches if r.kind == "stem")
        plan.neck_start = next((j for j, r in enumerate(plan.launches) if r.kind == "conv" and r.name.startswith("neck.")), 0)
        lvl = [(C.c_int32 * len(sizes))(*[h for h, _ in sizes]), (C.c_int32 * len(sizes))(*[w for _, w in sizes]),
               (C.c_float * len(sizes))(*[float(s) for s in g.strides])]
        plan.decode = ops.Launch("decode", "yv6_head_decode", (*(t.data_ptr() for t in plan.heads[0] + (plan.pred,)), N, nc, R,
                                                               len(sizes), *lvl))
        self._schedule(plan)
        self._plans[key] = plan
        return plan

    def _schedule(self, plan):
        """Assigns every launch to one of a few streams from its data dependencies (channel slices of the activation buffers):
        a chain keeps its stream, an op whose producers' streams have moved on takes the least recently used one and waits on
        events.  The backbone stays one chain; the branches of BiFusion (transpose-conv quadrants, cv1, cv2 + downsample), of
        CSPSPPF and the three head levels run side by side -- these launches are tens of CTAs and a few microseconds each, and
        their launch-to-first-MMA latency and drain overlap instead of adding up.  Inside a captured CUDA graph the events
        become plain graph edges."""
        K = self.n_lanes
        n = len(plan.launches)
        writers = {}
        lane, waits = [0] * n, [[] for _ in range(n)]
        last_on = [-1] * K
        for i, r in enumerate(plan.launches):
            prod = set()
            for key, lo, hi in r.reads:
                for wlo, whi, j in writers.get(key, ()):
                    if wlo < hi and lo < whi:
                        prod.add(j)
            chain = [lane[j] for j in prod if last_on[lane[j]] == j]
            if chain:
                s = min(chain)
            elif not prod:
                s = 0
            else:
                s = min(range(K), key=lambda t: last_on[t])
            lane[i] = s
            waits[i] = sorted(j for j in prod if lane[j] != s)
            last_on[s] = i
            for key, lo, hi in r.writes:
                writers.setdefault(key, []).append((lo, hi, i))
        need = set(j for w in waits for j in w)
        tails = [last_on[t] for t in range(1, K) if last_on[t] >= 0]
        need.update(tails)
        plan.lane, plan.waits, plan.tails = lane, waits, tails
        plan.events = {j: torch.cuda.Event() for j in need}
        plan.fork = torch.cuda.Event()

    def pin(self, N, H, W, in_dtype=torch.float32):
        """Keep the buffers of this shape for the engine's lifetime (they are referenced by a captured CUDA graph)."""
        self._plan(N, H, W, in_dtype)
        self._pinned.add((N, H, W, in_dtype))

    def launches(self, N, H, W, in_dtype=torch.float32):
        """The launch records (InferLaunch) of one forward of this shape, in launch order; the head decode is not among them."""
        return self._plan(N, H, W, in_dtype).launches

    def neck_start(self, N, H, W, in_dtype=torch.float32):
        """Index of the first launch after the backbone (the serving pipeline forks its NMS branch there)."""
        return self._plan(N, H, W, in_dtype).neck_start

    # ------------------------------------------------------------------ execution
    def launch_count(self, N, H, W, in_dtype=torch.float32):
        """Kernels launched per forward for this shape (convs + stem + pools + decode)."""
        return len(self.launches(N, H, W, in_dtype)) + 1

    def _heads(self, plan, k):
        """(cls, reg) of head set k of a plan, allocating set 1 on first use."""
        if k == 1 and len(plan.heads) == 1:
            plan.heads.append(tuple(torch.empty_like(t) for t in plan.heads[0]))
        return plan.heads[k]

    def _select_head_set(self, plan, k):
        """Point the pred convs at head-output set k (0 = the default tensors; 1 = a second pair, allocated on first use).
        The software-pipelined serving loop (pipeline.DetectStream) alternates between the two so that the NMS of batch
        i - 1 can read one set while the network of batch i writes the other."""
        if k == plan.head_set:
            return
        old, new = self._heads(plan, plan.head_set), self._heads(plan, k)
        for r in plan.launches:
            if r.head is not None:
                j = ("cls", "reg").index(r.head)
                r.desc.y += new[j].data_ptr() - old[j].data_ptr()
        plan.head_set = k

    def forward(self, x, stream=None, decode=True, head_set=0, hook=None):
        """x: [N,3,H,W] CUDA tensor, fp32 in [0,1] or uint8.  Returns pred [N,A,5+nc] fp32 (a buffer owned
        by the engine, overwritten by the next call with the same shape).  decode=False stops after the head convs and
        returns (cls [N,A,nc], reg [N,A,R], level sizes): the serving pipeline feeds them to the NMS kernels directly;
        head_set = 1 makes the head convs write the alternate (cls, reg) pair (decode=False only).  hook = (i, fn): fn() is
        called just before launch number i is enqueued, with the main stream current (used to fork a side branch there)."""
        if x.device != self.device:
            raise RuntimeError(f"input on {x.device}, engine on {self.device}")
        if x.dtype not in (torch.float32, torch.uint8):
            x = x.float()
        x = x.contiguous()
        N, Cin, H, W = x.shape
        assert Cin == 3
        plan = self._plan(N, H, W, x.dtype)
        plan.image = x  # keep alive while kernels are in flight
        assert head_set == 0 or not decode, "the alternate head set is for decode=False callers"
        self._select_head_set(plan, head_set)
        main = stream if stream is not None else torch.cuda.current_stream(self.device)
        if self.__dict__.get("_fold_ev") is not None and not torch.cuda.is_current_stream_capturing():
            main.wait_event(self._fold_ev)        # eager forward after a refold (captured pipelines wait in launch())
        sp = _lib.stream_ptr(main)
        lib, h = self.lib, self.handle
        plan.stem.x = x.data_ptr()
        lane, waits, events = plan.lane, plan.waits, plan.events
        multi = self.n_lanes > 1 and max(lane) > 0
        if multi:
            if self._side is None:
                self._side = [torch.cuda.Stream(device=self.device) for _ in range(self.n_lanes - 1)]
            streams = [main] + self._side
            sps = [_lib.stream_ptr(t) for t in streams]
            plan.fork.record(main)
            forked = set()
        for i, r in enumerate(plan.launches):
            if hook is not None and i == hook[0]:
                hook[1]()
            if multi:
                t = lane[i]
                if t and t not in forked:        # a side stream starts after everything the caller queued before this forward
                    streams[t].wait_event(plan.fork)
                    forked.add(t)
                for j in waits[i]:
                    streams[t].wait_event(events[j])
                sp = sps[t]
            r.run(lib, h, sp)
            if multi and i in events:
                events[i].record(streams[lane[i]])
        if multi:                                  # join: the caller's stream continues after every lane
            for j in plan.tails:
                main.wait_event(events[j])
            sp = sps[0]
        if not decode:
            return (*plan.heads[head_set], plan.sizes)
        plan.decode.run(lib, h, sp)
        return plan.pred

    def head_outputs(self, N, H, W, in_dtype=torch.float32, head_set=0):
        """(cls [N,A,nc] post-sigmoid, reg [N,A,R] raw) of head set `head_set` (see forward) of the last forward with this shape."""
        return self._heads(self._plan(N, H, W, in_dtype), head_set)

    def feature_maps(self, N, H, W, in_dtype=torch.float32):
        """Neck outputs as NCHW views (reference `featmaps`, yolo.py:37-39); bf16 (hi plane in fp32 mode), fp16 in fp16 mode."""
        plan = self._plan(N, H, W, in_dtype)
        out = []
        for t in self.g.feat:
            buf = plan.bufs[t.buf]
            buf = buf[0] if self.nsplit == 3 else buf
            out.append(buf[..., t.c_off:t.c_off + t.c].permute(0, 3, 1, 2))
        return out

    # ------------------------------------------------------------------ profiling
    def _profiled(self, x, stream):
        """(launch records, stream pointer) of x's shape after one forward of x, synchronized."""
        x = x.contiguous()
        N, _, H, W = x.shape
        launches = self.launches(N, H, W, x.dtype if x.dtype == torch.uint8 else torch.float32)
        self.forward(x, stream)
        torch.cuda.synchronize()
        return launches, _lib.stream_ptr(stream)

    def _timed(self, launches, sp, steps, before=None):
        """Device times (ms) of `steps` runs of the launches back to back between one pair of CUDA events, each run
        synchronized; before() runs ahead of each."""
        ts = []
        for _ in range(steps):
            if before is not None:
                before()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for r in launches:
                r.run(self.lib, self.handle, sp)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return ts

    def profile_calls(self, x, steps=20, stream=None):
        """Device time of every launch of one forward, each launched alone between CUDA events (serial, one stream):
        [(kind, op name, ms)], the median over `steps` runs."""
        launches, sp = self._profiled(x, stream)
        return [(r.kind, r.name, sorted(self._timed([r], sp, steps))[steps // 2]) for r in launches]

    def profile_convs(self, x, steps=5, stream=None):
        """Roofline instrumentation for bench.py: CUDA events around every conv_igemm launch.
        Returns (conv-kernel ms per forward, algorithmic conv FLOPs per forward, launches per forward)."""
        launches, sp = self._profiled(x, stream)
        convs = [r for r in launches if r.kind == "conv"]
        # one event pair around the back-to-back conv launches of a forward (launch gaps between the
        # kernels are part of the step, so they stay in the denominator)
        return sum(self._timed(convs, sp, steps)) / steps, sum(r.conv["flops"] for r in convs), len(convs)

    def conv_bytes_per_launch(self, N, H, W):
        """Algorithmic HBM bytes of an average conv launch: each conv reads its input slice and writes its output
        slice once (bf16), weights once."""
        tot, n = 0.0, 0
        for r in self.launches(N, H, W):
            if r.kind == "conv":
                ci = r.conv
                ysz = 4 if ci["y_f32"] else 2
                tot += N * (ci["h"] * ci["w"] * ci["cin"] * 2 + ci["ho"] * ci["wo"] * ci["cout"] * ysz) + ci["cout"] * ci["k"] ** 2 * ci["cin"] * 2
                n += 1
        return tot / max(n, 1)

    def profile_layers(self, x, iters=10, stream=None):
        """Per-launch timing table (name, shape, ms, TFLOP/s) with an L2 flush before every launch."""
        launches, sp = self._profiled(x, stream)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=self.device)
        rows = []
        for r in launches:
            if r.kind != "conv":
                continue
            ci, d = r.conv, r.desc
            ms = sorted(self._timed([r], sp, iters, flush.zero_))[iters // 2]
            ho, wo = ci["ho"], ci["wo"]
            by = 2.0 * d.N * (ci["h"] * ci["w"] * ci["cin"] + ho * wo * ci["cout"])
            rows.append(dict(name=ci["name"], cin=ci["cin"], cout=ci["cout"], k=ci["k"], s=ci["s"], hw=f"{ho}x{wo}", ms=ms,
                             tflops=ci["flops"] / ms / 1e9, gbs=by / ms / 1e6, plan=ops.plan_of(d, self.device.index or 0)))
        return rows
