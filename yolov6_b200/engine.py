"""Inference engine: walks the layer graph (arch.py) and issues one sm_90a kernel per op.

What the reference does with nested nn.Module.forward calls, cuDNN and ~15 eager ops for the head
decode (Model.forward yolo.py:33-41, Detect.forward effidehead.py:93-139), this does with:
  * folded deploy-form weights (fold.py) packed once to KRSC bf16 (or three bf16 planes),
  * pre-allocated NHWC activation buffers (concats are channel slices),
  * a prepared list of C-ABI descriptors per input shape, replayed per batch -- optionally as one
    captured CUDA graph (no Python / launch overhead in steady state).
Precision modes: "bf16" (bf16 operands, fp32 accumulate) and "fp32" (bf16x3 split operands: fp32-
equivalent products, used for the 1e-4 parity bar of BASELINE.json).
"""
import ctypes as C
import itertools
import os

import torch

from . import _lib, ops
from ._lib import ConvDesc
from .fold import fold_op, se_weights


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


def conv_launches(g, N, H, W, nsplit, sibling, addr, plan_fn):
    """Descriptors of the conv launches of one inference forward of graph g over an [N, 3, H, W] input, in launch order:
    {op index: [ConvDesc, ...]} -- four 1x1 quadrant launches for a transposed conv, one otherwise; the first conv of a sibling pair
    computes both.  Descriptors only: no allocation and no CUDA call, so the planner can be checked on these launches without a GPU.

    nsplit: 1 (bf16) or 3 (bf16x3 planes); sibling: siblings(g) or {}.  addr(kind, key, q=0) resolves device addresses:
    ("buf", buffer index) activation buffers, ("fused", first conv of the pair) the [.., 2 x Cout] sibling outputs,
    ("head", "cls" | "reg") the [N, A, ch] fp32 head tensors, ("w", op index, quadrant q of a transposed conv) packed weights,
    ("w_pair" | "w_fused" | "bias" | "bias_fused", op index) the other packed weights and padded biases; ("alpha", op index) is
    the residual scale.
    plan_fn(desc) -> plan dict (ops.PLAN_KEYS) decides where the column-pair view is kept."""
    offs = list(itertools.accumulate(((H // s) * (W // s) for s in g.strides), initial=0))    # first anchor of each level
    A = offs[-1]
    slices = sibling_slices(g, sibling)
    second = set(sibling.values())

    def view(t):
        """(address, channel offset, (N, h, w, channel pitch)) of graph tensor slice t."""
        b = g.bufs[t.buf]
        nhw = (N, H >> b.level, W >> b.level)
        if t.buf in slices:
            i, c0, pitch = slices[t.buf]
            return addr("fused", i), c0 + t.c_off, nhw + (pitch,)
        return addr("buf", t.buf), t.c_off, nhw + (b.c_total,)

    out = {}
    for i, op in enumerate(g.ops):
        if op.kind not in ("conv", "pred", "convT") or i in second:
            continue                      # the second conv of a sibling pair is computed by the first one's launch
        if op.kind == "pred" and op.head[0] not in ("cls", "reg"):
            continue                      # eval forward: anchor-free (cls, reg) branches only (effidehead_fuseab.py:141-199, _distill_ns.py:105-150)
        fused = i in sibling
        x, x_off, xs = view(op.src)
        k, s = (1, 1) if op.kind == "convT" else (op.k, op.s)
        cin = op.cin
        if op.kind != "convT":
            lo, hi = conv_window(g, op)
            x_off, cin = x_off - op.src.c_off + lo, hi - lo
        ws = (2 * op.cout if fused else op.cout, k, k, cin)
        kw = dict(x_c_off=x_off, bias=addr("bias_fused" if fused else "bias", i), stride=s, act=op.act, nsplit=nsplit)
        if op.res is not None:
            r, r_off, (_, rh, rw, rct) = view(op.res)
            kw.update(res=r, res_c_off=r_off, res_strides=(rh * rw * rct, rw * rct, rct), alpha=addr("alpha", i))
        if op.kind == "pred":
            which, lvl = op.head
            ch, lw = op.cout, W // g.strides[lvl]
            out[i] = [ops.conv_desc(x, xs, addr("w", i), ws, addr("head", which), (A * ch, lw * ch, ch), y_elem_off=offs[lvl] * ch,
                                    y_f32=True, **kw)]
            continue
        y, y_off, (_, dh, dw, dct) = view(op.dst)
        if op.kind == "convT":           # scatter quadrant (dy, dx) of the 2x upsample
            out[i] = [ops.conv_desc(x, xs, addr("w", i, q), ws, y, (dh * dw * dct, 2 * dw * dct, 2 * dct), y_c_off=y_off,
                                    y_elem_off=(q // 2 * dw + q % 2) * dct, **kw) for q in range(4)]
            continue
        d = ops.conv_desc(x, xs, addr("w_fused" if fused else "w", i), ws, y, (dh * dw * dct, dw * dct, dct), y_c_off=y_off, **kw)
        if pair_view_candidate(op):
            d = pair_view(d, addr("w_pair", i), plan_fn)
        out[i] = [d]
    return out


class InferEngine:
    def __init__(self, graph, state_dict, device, precision="bf16"):
        if device.type != "cuda":
            raise RuntimeError("yolov6_b200 runs its networks on sm_90a CUDA kernels only (no CPU fallback); "
                               f"got device {device}")
        assert precision in ("bf16", "fp32")
        self.g = graph
        self.device = device
        self.precision = precision
        self.nsplit = 3 if precision == "fp32" else 1
        self.handle = _lib.handle(device.index or 0)
        self.lib = _lib.lib()
        self.fuse_siblings = True
        self.n_lanes = int(os.environ.get("YV6_LANES", "4"))   # streams the launches of one forward are spread over (1 = serial)
        self._side = None
        self.weights = {}     # op index -> dict(w=..., bias=..., alpha=...)
        self._plans = {}      # (N, H, W, dtype) -> plan, least recently used first; bounded (rect-shaped evaluation
        self.max_plans = 4    # would otherwise keep one full activation set per distinct shape)
        self._pinned = set()  # shapes captured into CUDA graphs (their buffers must outlive the graph)
        self._pack(state_dict)

    # ------------------------------------------------------------------ weight packing
    def _pack(self, sd):
        sd = {k: v.detach().cpu() for k, v in sd.items()}
        dev = self.device

        def planes(w):       # KRSC weights in the precision's operand layout
            w = w.float().to(dev)
            return ops.split3(w).contiguous() if self.nsplit == 3 else w.to(torch.bfloat16).contiguous()

        self.sibling = siblings(self.g) if self.fuse_siblings else {}
        for i, op in enumerate(self.g.ops):
            if op.kind in ("pool", "shuffle", "up") or (op.kind == "pred" and op.head[0] not in ("cls", "reg")):   # fuse_ab / distillation preds: training only
                continue
            if op.kind == "se":
                self.weights[i] = dict(zip(("w1", "b1", "w2", "b2"), (t.float().contiguous().to(dev) for t in se_weights(sd, op))))
                continue
            w, b = fold_op(sd, op)
            ent = {}
            if op.kind == "stem":
                cp = stem_channels(self.g, op)
                w, b = torch.cat([w, w.new_zeros((cp - op.cout,) + w.shape[1:])]), torch.cat([b, b.new_zeros(cp - op.cout)])
                ent["w_dev"] = w.float().permute(1, 2, 3, 0).contiguous().to(dev)       # [3][3][3][Cout]
                ent["b_dev"] = b.float().contiguous().to(dev)
            elif op.kind == "dw":
                # fp32 [k*k][C]: the exact folded weights serve both precision modes and cost k*k*C*4 bytes per launch
                ent["w_dev"] = w[..., 0].permute(1, 2, 0).reshape(op.k * op.k, op.cin).float().contiguous().to(dev)
                ent["b_dev"] = b.float().contiguous().to(dev)
            else:
                w = w if op.kind == "convT" else window_weights(self.g, op, w)
                ws = w if isinstance(w, list) else [w]
                ent["w"] = [planes(wi) for wi in ws]
                if pair_view_candidate(op):      # [Cout][3][2][2*Cin] weights of the column-pair view (see pair_view)
                    ent["w_pair"] = planes(ops.pair_view_weights(ws[0].float()))
                ent["bias"] = ops.pad_bias(b.to(dev), op.cout)
            ent["alpha"] = float(sd[op.alpha]) if (op.alpha and op.res is not None) else 1.0
            self.weights[i] = ent
        for i, j in self.sibling.items():      # one conv with 2 x Cout output channels: [cls branch | reg branch]
            (wa, ba), (wb, bb) = fold_op(sd, self.g.ops[i]), fold_op(sd, self.g.ops[j])
            self.weights[i]["w_fused"] = planes(torch.cat([wa, wb], 0))
            self.weights[i]["bias_fused"] = ops.pad_bias(torch.cat([ba, bb]).to(dev), 2 * self.g.ops[i].cout)

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
        plan = {"bufs": [], "calls": [], "conv_info": [], "deps": [], "pred_descs": [], "head_set": 0}
        for b in g.bufs:
            h, w = H >> b.level, W >> b.level
            shape = (P, N, h, w, b.c_total) if P == 3 else (N, h, w, b.c_total)
            plan["bufs"].append(torch.zeros(shape, dtype=torch.bfloat16, device=dev))
        sizes = [(H // s, W // s) for s in g.strides]
        A = sum(h * w for h, w in sizes)
        nc, R = g.num_classes, 4 * (g.reg_max + 1)
        plan["cls"] = torch.empty(N, A, nc, dtype=torch.float32, device=dev)
        plan["reg"] = torch.empty(N, A, R, dtype=torch.float32, device=dev)
        plan["pred"] = torch.empty(N, A, 5 + nc, dtype=torch.float32, device=dev)
        plan["sizes"], plan["A"] = sizes, A
        plan["lvl_h"] = (C.c_int32 * len(sizes))(*[h for h, _ in sizes])
        plan["lvl_w"] = (C.c_int32 * len(sizes))(*[w for _, w in sizes])
        plan["lvl_s"] = (C.c_float * len(sizes))(*[float(s) for s in g.strides])
        plan["image"] = None

        slices = sibling_slices(g, self.sibling)
        fused = {}          # first conv of a sibling pair -> the pair's [.., 2 x Cout] output
        for i in self.sibling:
            lvl = g.bufs[g.ops[i].dst.buf].level
            shape = (N, H >> lvl, W >> lvl, 2 * g.ops[i].cout)
            fused[i] = torch.zeros((P,) + shape if P == 3 else shape, dtype=torch.bfloat16, device=dev)
        plan["fused_bufs"] = list(fused.values())

        def view(t):
            """(tensor, first channel) of a graph tensor slice."""
            if t.buf in slices:
                i, c0, _ = slices[t.buf]
                return fused[i], c0 + t.c_off
            return plan["bufs"][t.buf], t.c_off

        def span(t):
            """(tensor identity, first channel, end channel) of a graph tensor slice: the unit of the dependency analysis."""
            buf, c0 = view(t)
            return (id(buf), c0, c0 + t.c)

        def addr(kind, key, q=0):
            """Device addresses of this plan's tensors and the packed weights (see conv_launches)."""
            if kind == "buf":
                return plan["bufs"][key].data_ptr()
            if kind == "fused":
                return fused[key].data_ptr()
            if kind == "head":
                return plan[key].data_ptr()
            if kind == "alpha":
                return self.weights[key]["alpha"]
            t = self.weights[key][kind]
            return (t[q] if kind == "w" else t).data_ptr()

        launches = conv_launches(g, N, H, W, P, self.sibling, addr, lambda d: ops.plan_of(d, dev.index or 0))

        def slice_args(t):
            """(address of the slice's first channel, channel pitch, plane stride) of a graph tensor slice."""
            buf, c0 = view(t)
            return buf.data_ptr() + 2 * c0, buf.shape[-1], buf.stride(0) if P == 3 else 0

        plan["call_names"] = []
        for i, op in enumerate(g.ops):
            lvl = g.bufs[op.src.buf].level if op.src is not None else 0
            if op.kind == "stem":
                buf, _ = view(op.dst)
                ent = self.weights[i]
                d = ops.stem_desc(0, N, H, W, in_dtype == torch.uint8, ent["w_dev"].data_ptr(), ent["b_dev"].data_ptr(), stem_channels(g, op),
                                  op.act, buf.data_ptr(), P, buf.stride(0) if P == 3 else 0)
                plan["stem"] = d
                plan["calls"].append(("stem", d))
                plan["deps"].append(dict(reads=[], writes=[span(op.dst)]))
            elif op.kind == "pool":
                buf, _ = view(op.dst)
                h, w, ct = buf.shape[-3:]
                plan["calls"].append(("pool", (buf.data_ptr(), N, h, w, op.cin, ct, P, buf.stride(0) if P == 3 else 0)))
                plan["deps"].append(dict(reads=[(id(buf), 0, op.cin)], writes=[(id(buf), op.cin, 4 * op.cin)]))
            elif op.kind == "dw":
                ent = self.weights[i]
                (x, xp, xpl), (y, yp, ypl) = slice_args(op.src), slice_args(op.dst)
                d = ops.dw_desc(x, (N, H >> lvl, W >> lvl, xp), xpl, ent["w_dev"].data_ptr(), ent["b_dev"].data_ptr(), op.cin, op.k, op.s,
                                op.act, y, yp, ypl, P)
                plan["calls"].append(("dw", d))
                plan["deps"].append(dict(reads=[span(op.src)], writes=[span(op.dst)]))
            elif op.kind == "se":
                ent = self.weights[i]
                x, xp, xpl = slice_args(op.src)
                d = ops.se_desc(x, N, (H >> lvl) * (W >> lvl), op.cin, op.cout, xp, xpl, *(ent[k].data_ptr() for k in ("w1", "b1", "w2", "b2")),
                                nsplit=P)
                plan["calls"].append(("se", d))
                plan["deps"].append(dict(reads=[span(op.src)], writes=[span(op.src)]))
            elif op.kind == "shuffle":
                (a, ap, apl), (b, bp, bpl), (y, yp, ypl) = slice_args(op.src), slice_args(op.src2), slice_args(op.dst)
                plan["calls"].append(("shuffle", (a, ap, apl, b, bp, bpl, N * (H >> lvl) * (W >> lvl), op.cin, y, yp, ypl, P)))
                plan["deps"].append(dict(reads=[span(op.src), span(op.src2)], writes=[span(op.dst)]))
            elif op.kind == "up":
                (x, xp, xpl), (y, yp, ypl) = slice_args(op.src), slice_args(op.dst)
                plan["calls"].append(("up", (x, xp, xpl, N, H >> lvl, W >> lvl, op.cin, y, yp, ypl, P)))
                plan["deps"].append(dict(reads=[span(op.src)], writes=[span(op.dst)]))
            plan["call_names"] += [op.name] * (len(plan["calls"]) - len(plan["call_names"]))
            for q, d in enumerate(launches.get(i, ())):
                lvl = g.bufs[op.src.buf].level
                sh, sw, k, s = H >> lvl, W >> lvl, d.kh, d.stride      # (of the 3x3 stride-2 conv, also on the column-pair view)
                oh, ow = (sh + 2 * (k // 2) - k) // s + 1, (sw + 2 * (k // 2) - k) // s + 1
                plan["conv_info"].append(dict(name=op.name if op.kind != "convT" else f"{op.name}[{q}]", cin=op.cin, cout=d.Cout,
                                              k=k, s=s, ho=oh, wo=ow, h=sh, w=sw, flops=2.0 * N * oh * ow * d.Cout * op.cin * k * k,
                                              y_f32=op.kind == "pred"))
                reads = [span(op.src)] + ([span(op.res)] if op.res is not None else [])
                if op.kind == "pred":
                    plan["pred_descs"].append((d, op.head[0], d.y - plan[op.head[0]].data_ptr()))
                    writes = [(("head",) + tuple(op.head), 0, 1)]
                elif i in fused:
                    writes = [(id(fused[i]), 0, 2 * op.cout)]
                else:
                    writes = [span(op.dst)]
                if "neck_start" not in plan and op.name.startswith("neck."):
                    plan["neck_start"] = len(plan["calls"])     # first launch after the backbone (pipeline.DetectStream forks here)
                plan["calls"].append(("conv", d))
                plan["deps"].append(dict(reads=reads, writes=writes))
                plan["call_names"].append(op.name)
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
        deps = plan["deps"]
        n = len(deps)
        writers = {}
        lane, waits = [0] * n, [[] for _ in range(n)]
        last_on = [-1] * K
        for i, dp in enumerate(deps):
            prod = set()
            for key, lo, hi in dp["reads"]:
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
            for key, lo, hi in dp["writes"]:
                writers.setdefault(key, []).append((lo, hi, i))
        need = set(j for w in waits for j in w)
        tails = [last_on[t] for t in range(1, K) if last_on[t] >= 0]
        need.update(tails)
        plan["lane"], plan["waits"], plan["tails"] = lane, waits, tails
        plan["events"] = {j: torch.cuda.Event() for j in need}
        plan["fork"] = torch.cuda.Event()

    def pin(self, N, H, W, in_dtype=torch.float32):
        """Keep the buffers of this shape for the engine's lifetime (they are referenced by a captured CUDA graph)."""
        self._plan(N, H, W, in_dtype)
        self._pinned.add((N, H, W, in_dtype))

    # ------------------------------------------------------------------ execution
    def launch_count(self, N, H, W, in_dtype=torch.float32):
        """Kernels launched per forward for this shape (convs + stem + pools + decode)."""
        return len(self._plan(N, H, W, in_dtype)["calls"]) + 1

    def _select_head_set(self, plan, k):
        """Point the pred convs at head-output set k (0 = the default tensors; 1 = a second pair, allocated on first use).
        The software-pipelined serving loop (pipeline.DetectStream) alternates between the two so that the NMS of batch
        i - 1 can read one set while the network of batch i writes the other."""
        if k == plan["head_set"]:
            return
        if k == 1 and "cls_alt" not in plan:
            plan["cls_alt"], plan["reg_alt"] = torch.empty_like(plan["cls"]), torch.empty_like(plan["reg"])
        for d, which, off in plan["pred_descs"]:
            d.y = plan[which + ("_alt" if k == 1 else "")].data_ptr() + off
        plan["head_set"] = k

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
        plan["image"] = x  # keep alive while kernels are in flight
        assert head_set == 0 or not decode, "the alternate head set is for decode=False callers"
        self._select_head_set(plan, head_set)
        main = stream if stream is not None else torch.cuda.current_stream(self.device)
        sp = _lib.stream_ptr(main)
        lib, h, chk = self.lib, self.handle, _lib.check
        plan["stem"].x = x.data_ptr()
        lane, waits, events = plan["lane"], plan["waits"], plan["events"]
        multi = self.n_lanes > 1 and max(lane) > 0
        if multi:
            if self._side is None:
                self._side = [torch.cuda.Stream(device=self.device) for _ in range(self.n_lanes - 1)]
            streams = [main] + self._side
            sps = [_lib.stream_ptr(t) for t in streams]
            plan["fork"].record(main)
            forked = set()
        for i, (kind, d) in enumerate(plan["calls"]):
            if hook is not None and i == hook[0]:
                hook[1]()
            if multi:
                t = lane[i]
                if t and t not in forked:        # a side stream starts after everything the caller queued before this forward
                    streams[t].wait_event(plan["fork"])
                    forked.add(t)
                for j in waits[i]:
                    streams[t].wait_event(events[j])
                sp = sps[t]
            self._launch(kind, d, sp)
            if multi and i in events:
                events[i].record(streams[lane[i]])
        if multi:                                  # join: the caller's stream continues after every lane
            for j in plan["tails"]:
                main.wait_event(events[j])
            sp = sps[0]
        g = self.g
        if not decode:
            if head_set == 1:
                return plan["cls_alt"], plan["reg_alt"], plan["sizes"]
            return plan["cls"], plan["reg"], plan["sizes"]
        chk(lib.yv6_head_decode(h, C.c_void_p(plan["cls"].data_ptr()), C.c_void_p(plan["reg"].data_ptr()),
                                C.c_void_p(plan["pred"].data_ptr()), N, g.num_classes, 4 * (g.reg_max + 1),
                                len(g.strides), plan["lvl_h"], plan["lvl_w"], plan["lvl_s"], sp))
        return plan["pred"]

    def _launch(self, kind, d, sp):
        lib, h, chk = self.lib, self.handle, _lib.check
        if kind == "conv":
            chk(lib.yv6_conv_fwd(h, C.byref(d), sp))
        elif kind == "stem":
            chk(lib.yv6_stem_fwd(h, C.byref(d), sp))
        elif kind == "pool":
            chk(lib.yv6_sppf_pool(h, C.c_void_p(d[0]), d[1], d[2], d[3], d[4], d[5], d[6], d[7], sp))
        elif kind == "dw":
            chk(lib.yv6_dwconv_fwd(h, C.byref(d), sp))
        elif kind == "se":
            chk(lib.yv6_se_fwd(h, C.byref(d), sp))
        elif kind == "shuffle":
            chk(lib.yv6_channel_shuffle(h, *d, sp))
        elif kind == "up":
            chk(lib.yv6_upsample2x(h, *d, sp))
        else:
            raise RuntimeError(f"no kernel for launch kind {kind!r}")

    def profile_calls(self, x, steps=20, stream=None):
        """Device time of every launch of one forward, each launched alone between CUDA events (serial, one stream):
        [(kind, op name, ms)], the median over `steps` runs."""
        x = x.contiguous()
        N, _, H, W = x.shape
        plan = self._plan(N, H, W, x.dtype if x.dtype == torch.uint8 else torch.float32)
        self.forward(x, stream)
        torch.cuda.synchronize()
        sp = _lib.stream_ptr(stream)
        rows = []
        for (kind, d), name in zip(plan["calls"], plan["call_names"]):
            ts = []
            for _ in range(steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                self._launch(kind, d, sp)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            rows.append((kind, name, sorted(ts)[len(ts) // 2]))
        return rows

    def head_outputs(self, N, H, W, in_dtype=torch.float32):
        """(cls [N,A,nc] post-sigmoid, reg [N,A,R] raw) of the last forward with this shape."""
        plan = self._plan(N, H, W, in_dtype)
        return plan["cls"], plan["reg"]

    def feature_maps(self, N, H, W, in_dtype=torch.float32):
        """Neck outputs as NCHW views (reference `featmaps`, yolo.py:37-39); bf16 (hi plane in fp32 mode)."""
        plan = self._plan(N, H, W, in_dtype)
        out = []
        for t in self.g.feat:
            buf = plan["bufs"][t.buf]
            buf = buf[0] if self.nsplit == 3 else buf
            out.append(buf[..., t.c_off:t.c_off + t.c].permute(0, 3, 1, 2))
        return out

    def profile_convs(self, x, steps=5, stream=None):
        """Roofline instrumentation for bench.py: CUDA events around every conv_igemm launch.
        Returns (conv-kernel ms per forward, algorithmic conv FLOPs per forward, launches per forward)."""
        x = x.contiguous()
        N, _, H, W = x.shape
        plan = self._plan(N, H, W, x.dtype if x.dtype == torch.uint8 else torch.float32)
        self.forward(x, stream)
        torch.cuda.synchronize()
        sp = _lib.stream_ptr(stream)
        convs = [d for kind, d in plan["calls"] if kind == "conv"]
        flops = sum(ci["flops"] for ci in plan["conv_info"])     # algorithmic (the column-pair view's zero taps do not count)
        # one event pair around the back-to-back conv launches of a forward (launch gaps between the
        # kernels are part of the step, so they stay in the denominator)
        total_ms = 0.0
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for d in convs:
                _lib.check(self.lib.yv6_conv_fwd(self.handle, C.byref(d), sp))
            e1.record()
            torch.cuda.synchronize()
            total_ms += e0.elapsed_time(e1)
        return total_ms / steps, flops, len(convs)

    def conv_bytes_per_launch(self, N, H, W):
        """Algorithmic HBM bytes of an average conv launch: each conv reads its input slice and writes its output
        slice once (bf16), weights once."""
        plan = self._plan(N, H, W, torch.float32)
        tot, n = 0.0, 0
        for ci in plan["conv_info"]:
            ysz = 4 if ci["y_f32"] else 2
            tot += N * (ci["h"] * ci["w"] * ci["cin"] * 2 + ci["ho"] * ci["wo"] * ci["cout"] * ysz) + ci["cout"] * ci["k"] ** 2 * ci["cin"] * 2
            n += 1
        return tot / max(n, 1)

    def profile_layers(self, x, iters=10, stream=None):
        """Per-launch timing table (name, shape, ms, TFLOP/s) with an L2 flush before every launch."""
        x = x.contiguous()
        N, _, H, W = x.shape
        plan = self._plan(N, H, W, x.dtype if x.dtype == torch.uint8 else torch.float32)
        self.forward(x, stream)
        torch.cuda.synchronize()
        sp = _lib.stream_ptr(stream)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=self.device)
        rows = []
        convs = [d for kind, d in plan["calls"] if kind == "conv"]
        for ci, d in zip(plan["conv_info"], convs):
            name = ci["name"]
            ts = []
            for _ in range(iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _lib.check(self.lib.yv6_conv_fwd(self.handle, C.byref(d), sp))
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            ms = ts[len(ts) // 2]
            ho, wo = ci["ho"], ci["wo"]
            fl = ci["flops"]
            by = 2.0 * d.N * (ci["h"] * ci["w"] * ci["cin"] + ho * wo * ci["cout"])
            rows.append(dict(name=name, cin=ci["cin"], cout=ci["cout"], k=ci["k"], s=ci["s"], hw=f"{ho}x{wo}", ms=ms,
                             tflops=fl / ms / 1e9, gbs=by / ms / 1e6, plan=ops.plan_of(d, self.device.index or 0)))
        return rows
