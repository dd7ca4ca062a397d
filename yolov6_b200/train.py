"""Training engine: train-form forward + backward of the conv stack on sm_90a kernels.

What autograd + cuDNN + ~130 BatchNorm / activation kernels do for the reference's
`Trainer.train_in_steps` (core/engine.py:142-176) over `Model.forward` in train mode
(models/yolo.py:33-41; ConvModule conv->BN->act, layers/common.py:46-49; RepVGGBlock's three BN-ed
branches, common.py:245-255), this engine does by walking the same layer graph as the inference
engine (arch.py):

  forward : raw convs on wgmma (yv6_conv_fwd, bf16 operands, fp32 accumulate, no bias/act)
            -> yv6_bn_stats_finalize (batch statistics of all branches of a block + running-stat update in
               one launch; eps 1e-3, momentum 0.03 as set by initialize_weights, torch_utils.py:38-48)
            -> yv6_bn_apply_fwd (sum of the BN-ed branches + activation, written into concat slices);
  backward: yv6_bn_bwd (activation + BatchNorm backward of all branches of a block in two passes)
            -> dgrad = yv6_conv_fwd with rotated / transposed weights, accumulating into the input
               gradient through the residual epilogue (stride-2 convs: four parity sub-convolutions)
            -> yv6_conv_wgrad (MN-major wgmma GEMM over pixels, fp32 split-K accumulation).

Step-level structure (SURVEY.md 8f N1): everything is planned once per input shape -- activation, raw-conv and
gradient buffers, one zero-initialised arena for all per-step accumulators (BatchNorm sums, fp32 KRSC weight
gradients, counters), and a list of C-ABI descriptors for the forward and the backward pass -- so a step is
    arena.zero_()  ->  yv6_xform (fp32 master weights -> every bf16 layout the kernels need, ONE launch)
    ->  forward descriptors  ->  loss  ->  backward descriptors  ->  yv6_xform (gradients -> flat fp32 buffer)
with no allocation, no host synchronisation and no per-layer PyTorch op; it can be captured in a CUDA graph
(step.py).  Parameters are views of one flat fp32 buffer and gradients land in one flat fp32 buffer in the
reference's tensor layouts (flat.py), laid out in the order the backward pass completes them, so the DDP
gradient all-reduce (core/engine.py:464-466) is a few large NCCL calls that overlap the rest of the backward
(dist.py) and SGD + EMA are one kernel (optim.py).  BottleRep shortcuts (M / L6, common.py:600-617) ride in
the BN apply / backward kernels (y = act(z) + alpha * x, alpha read from device memory).
"""
import ctypes as C
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib, ops
from ._lib import ACT_CODES, DT_F32, DT_U8, XF_BF16, XF_F32, XF_F64, XFORM_CHUNK, BnDesc, BnStatsDesc, QaDesc, WgradDesc, XformSeg
from .flat import FlatState

BN_EPS, BN_MOMENTUM = 1e-3, 0.03


def _p(t):
    return t.data_ptr() if t is not None else 0


def op_branches(op):
    """(prefix, kernel size) of the conv branches of a BN-ed block; k = 0 marks RepVGG's identity BatchNorm.  A QA block
    ('qa') has the two conv branches only: its identity / average-pool branches have no parameters (yv6_qa_fwd / _bwd)."""
    if op.layout == "qa":
        return [(op.name + ".rbr_dense", 3), (op.name + ".rbr_1x1", 1)]
    if op.layout == "rep":
        br = [(op.name + ".rbr_dense", 3), (op.name + ".rbr_1x1", 1)]
        if op.kind != "stem" and op.cin == op.cout and op.s == 1:
            br.append((op.name + ".rbr_identity", 0))
        return br
    if op.layout == "cm":        # bare ConvModule (MBLABlock.cv1 / cv2, common.py:671-677)
        return [(op.name, op.k)]
    return [(op.name + ".block", op.k)]


def conv_weight_name(op, prefix):
    """The weight of a conv branch: a ConvModule's `.conv.weight`, or the bare Conv2d `rbr_1x1.weight` of a QA block."""
    return prefix + (".weight" if op.layout == "qa" and prefix.endswith(".rbr_1x1") else ".conv.weight")


def branch_bn_names(op):
    """The BatchNorm of each conv branch of op_branches (None: none of its own) and, for a QA block, the post-sum BatchNorm."""
    if op.layout == "qa":
        return [op.name + ".rbr_dense.bn", None], op.name + ".bn"
    return [prefix + (".bn" if k else "") for prefix, k in op_branches(op)], None


def op_param_names(op):
    """Trainable parameters owned by a graph op, in the order their gradients are produced.  An op over rows w_row0 > 0 of a
    parameter (arch.Op.w_row0) writes its rows of the gradients, but the parameter belongs to the op over row 0: that op
    comes first in the forward pass, so the parameter's gradient is complete once that op's backward ran."""
    if op.kind == "pool" or op.w_row0:
        return []
    if op.kind == "pred":
        return [op.name + ".weight", op.name + ".bias"]
    if op.kind == "convT":
        return [op.name + ".upsample_transpose.weight", op.name + ".upsample_transpose.bias"]
    names = []
    bns, post = branch_bn_names(op)
    for (prefix, k), bn in zip(op_branches(op), bns):
        if k:
            names.append(conv_weight_name(op, prefix))
        if bn is not None:
            names += [bn + ".weight", bn + ".bias"]
    if post is not None:
        names += [post + ".weight", post + ".bias"]
    if op.alpha:
        names.append(op.alpha)
    return names


class XformTable:
    """Device tables of one yv6_xform launch."""

    def __init__(self, segs, dev):
        self.n = len(segs)
        arr = (XformSeg * max(self.n, 1))(*segs)
        raw = np.frombuffer(arr, dtype=np.uint8).copy()
        self.segs = torch.from_numpy(raw).to(dev)
        chunk_seg, chunk_first = [], []
        for i, s in enumerate(segs):
            total = s.n[0] * s.n[1] * s.n[2] * s.n[3]
            chunk_first.append(len(chunk_seg))
            chunk_seg += [i] * ((total + XFORM_CHUNK - 1) // XFORM_CHUNK)
        self.n_chunks = len(chunk_seg)
        self.chunk_seg = torch.tensor(chunk_seg or [0], dtype=torch.int32).to(dev)
        self.chunk_first = torch.tensor(chunk_first or [0], dtype=torch.int32).to(dev)

    def launch(self, lib, h, accumulate, sp):
        if self.n_chunks:
            _lib.check(lib.yv6_xform(h, self.segs.data_ptr(), self.chunk_seg.data_ptr(), self.chunk_first.data_ptr(), self.n_chunks,
                                     int(bool(accumulate)), sp))


def _seg(dst, src, n, ds, ss, dst_dtype, src_dtype):
    s = XformSeg()
    s.dst, s.src = dst, src
    n, ds, ss = list(n), list(ds), list(ss)
    while len(n) < 4:
        n.insert(0, 1)
        ds.insert(0, 0)
        ss.insert(0, 0)
    for i in range(4):
        s.n[i], s.ds[i], s.ss[i] = int(n[i]), int(ds[i]), int(ss[i])
    s.dst_dtype, s.src_dtype = dst_dtype, src_dtype
    return s


ALL = -1    # Launch.parity of a main-stream launch that waits for every pending weight gradient


@dataclass(eq=False)
class Write:
    """Channels [off, off + n) of gradient buffer `buf` written by a launch (at every pixel when `full`); `assign(True)` makes
    the launch overwrite them, `assign(False)` add to them.  The launches of one `group` share one decision."""
    buf: int
    off: int
    n: int
    full: bool
    assign: object
    group: tuple = None


@dataclass(eq=False)
class Launch(ops.Launch):
    """One launch of the training step (ops.Launch).  `side`: a weight gradient, run on the side stream next to the main
    stream; `parity`: the dc scratch pair it reads (side) or refills (main stream, ALL: everything the side stream may read).
    `snapshot` = (op index, incoming gradient slice) is copied into engine.dbg before the launch when engine.debug;
    `bucket` = k marks the unpack of gradient bucket k."""
    kernels: int = 1
    side: bool = False
    parity: int = None
    writes: tuple = ()
    snapshot: tuple = None
    bucket: int = None


def _desc_launch(kind, fn, d, **kw):
    return Launch(kind, fn, (C.byref(d),), desc=d, **kw)


class _Scratch:
    """Scratch of one planned shape.  dc: the BN-backward outputs (gradients w.r.t. the raw conv outputs), which live only until
    their dgrad / wgrad ran, two per op parity: the weight gradients of an op run on a side stream while the next op's BN
    backward refills the other pair.  Also the max-pool backward scratch, the ConvTranspose quadrant gradients and the head
    gradients dl; a buffer that grows keeps its smaller predecessors, which earlier launches still use."""

    def __init__(self, new, dc_elems):
        self.new = new
        self.dc = [new((dc_elems,), torch.bfloat16) for _ in range(4)]
        self.bn_ops = 0
        self.pool, self.quad, self.dl = [], [], []

    def dc_view(self, par, slot, shape):
        return self.dc[2 * par + slot][:int(np.prod(shape))].view(shape)

    def grown(self, pools, numel, count, dtype):
        """The last set of `count` buffers in `pools`, after appending a new set when it holds fewer than numel elements."""
        if not pools or pools[-1][0].numel() < numel:
            pools.append([self.new((numel,), dtype) for _ in range(count)])
        return pools[-1]


class _Arena:
    """The per-shape tensors of a multi-shape plan (`TrainEngine.plan_shapes`): every shape's plan carves its activations,
    gradients, head outputs and scratch from offset 0 of one byte buffer, in planning order, so the buffer is as large as the
    largest single plan and the shapes' plans overlap.  Only one shape is live at a time: the buffer is cleared whenever the
    live shape changes (`TrainEngine.make_live`), which leaves it as a fresh plan's torch.zeros would.  Over a meta tensor
    it only measures a plan."""
    ALIGN = 512                         # the caching allocator's granularity: a single plan's tensors start 512-aligned too

    def __init__(self, store):
        self.store, self.off, self.live = store, 0, None

    def take(self, shape, dtype):
        n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        o, self.off = self.off, self.off + (n + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        if self.off > self.store.numel():
            raise RuntimeError(f"multi-shape plan: {self.off} bytes exceed the shared buffer's {self.store.numel()}")
        return self.store[o:o + n].view(dtype).view(shape)


FWD_ARENA_KEYS = ("fsum", "fcnt", "qsum", "qcnt")     # the zero-arena slots the forward pass uses (batch-statistics sums)


class TrainEngine:
    """`teacher=True` plans the forward pass only, for the teacher of self-distillation (core/engine.py:429-441): batch-statistics
    BatchNorm with `track_running_stats = False` (the finalize launches get null running statistics, num_batches_tracked stays),
    no gradient buffers, scratch or backward launches, and no anchor-aided pred convs of a fuse_ab model (the distillation loss
    reads the anchor-free head, loss_distill.py:76).  step.TrainStep runs it next to the student's step."""
    teacher = False
    arena = None            # plan_shapes: the _Arena every planned shape's tensors are views into

    def __init__(self, model, n_buckets=1, teacher=False):
        self.teacher = bool(teacher)
        self.model = model
        self.g = model.graph
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError("yolov6_b200 training runs on sm_90a CUDA kernels only (no CPU fallback)")
        self.lib = _lib.lib()
        self.h = _lib.handle(self.dev.index or 0)
        self.n_buckets = max(1, int(n_buckets))
        self.debug = False      # tests: snapshot the incoming gradient of every op into self.dbg[op index]
        self.dbg = {}
        self._shape = None
        self.bucket_hook = None     # callable(k) invoked (eager mode) right after bucket k's gradients are unpacked
        self.overlap_wgrad = os.environ.get("YV6_WGRAD_OVERLAP", "1") != "0"   # weight gradients on a side stream (see backward)
        self._wg_stream = None
        # the neck outputs as differentiable outputs of the training forward (feature-map distillation, loss_distill.py:223-245):
        # off by default -- it changes the backward plan (every writer of those gradient slices accumulates onto the external one)
        self.external_feat_grads = False
        self._feat_grads = None
        self._build_state()

    # ================================================================== parameter-level state (shape independent)
    def _build_state(self):
        g, dev = self.g, self.dev
        order = [n for op in reversed(g.ops) for n in op_param_names(op)]
        self.flat = FlatState(self.model, order)
        self.params = dict(self.model.named_parameters())
        self.buffers_ = dict(self.model.named_buffers())
        fl = self.flat
        # ---- zero arena layout: per-step accumulators (float64 sums, counters, fp32 KRSC weight gradients)
        zoff, ztot = {}, 0

        def ztake(key, nbytes):
            nonlocal ztot
            if self.teacher and key[1] not in FWD_ARENA_KEYS:
                return
            zoff[key] = ztot
            ztot += (int(nbytes) + 15) // 16 * 16

        for i, op in enumerate(g.ops):
            if op.kind == "pool":
                continue
            if op.kind == "pred":
                chp = (op.cout + 15) // 16 * 16
                ztake((i, "bsum"), 16 * chp)
                ztake((i, "bcnt"), 16)
                ztake((i, "dw"), 4 * op.cout * op.cin)
            elif op.kind == "convT":
                ztake((i, "bsum"), 16 * op.cout)
                ztake((i, "bcnt"), 16)
                ztake((i, "dw"), 4 * 4 * op.cout * op.cin)
            else:
                br = op_branches(op)
                nb, c = len(br), op.cout
                ztake((i, "fsum"), 16 * nb * c)
                ztake((i, "fcnt"), 16)
                ztake((i, "s1"), 8 * c)
                ztake((i, "work"), 8 * nb * c)
                ztake((i, "s2"), 8 * nb * c)
                ztake((i, "dalpha"), 16)
                ztake((i, "bcnt"), 16)
                if op.layout == "qa":     # the post-sum BN's forward sums, and the backward of BN_d (rbr_dense.bn) on its own
                    ztake((i, "qsum"), 16 * c)
                    ztake((i, "qcnt"), 16)
                    for key, nbytes in (("s1d", 8 * c), ("s2d", 8 * c), ("workd", 8 * c), ("bcntd", 16)):
                        ztake((i, key), nbytes)
                for b, (prefix, k) in enumerate(br):
                    if k == 0:
                        continue
                    if op.kind == "stem":      # 1x1 wgrad over the im2col patches: [Cout][32] (27 taps + 5 zero columns)
                        ztake((i, "dw", b), 4 * op.cout * 32)
                    else:
                        ztake((i, "dw", b), 4 * op.cout * k * k * op.cin)
        self.zero_arena = torch.zeros(ztot, dtype=torch.uint8, device=dev)
        zbase = self.zero_arena.data_ptr()
        self._z = lambda *key: zbase + zoff[key]
        # ---- per-op fp32 outputs that need no clearing: BN statistics [nb][4][C] and backward coefficients [nb][2][C]
        self.stat_out, self.coef_out = {}, {}
        # ---- packed weights + the two xform tables
        pack, self.ctx, self.wts = [], [None] * len(g.ops), {}
        grad_segs, self.bucket_of_op = [], {}
        P = self.params

        bf16 = self._bf
        for i, op in enumerate(g.ops):
            if op.kind == "pool" or not self._planned(op):
                continue
            W = self.wts[i] = {}
            if op.kind == "pred":
                ch, cin, chp = op.cout, op.cin, (op.cout + 15) // 16 * 16
                W["w"] = bf16(ch, 1, 1, cin)
                W["bias"] = ops.bias_buffer(ch, dev)
                wsrc, bsrc = fl.ptr(op.name + ".weight"), fl.ptr(op.name + ".bias")
                pack.append(_seg(W["w"].data_ptr(), wsrc, [ch * cin], [1], [1], XF_BF16, XF_F32))
                pack.append(_seg(W["bias"].data_ptr(), bsrc, [ch], [1], [1], XF_F32, XF_F32))
                if not self.teacher:
                    W["wt"] = bf16(cin, 1, 1, chp)                               # dgrad: [Cin][ch_pad], zero padded
                    pack.append(_seg(W["wt"].data_ptr(), wsrc, [cin, ch], [chp, 1], [1, cin], XF_BF16, XF_F32))
                self.ctx[i] = dict(w=W["w"])
                continue
            if op.kind == "convT":
                co, ci = op.cout, op.cin
                W["w"] = bf16(4, co, 1, 1, ci)                                   # quadrant q = dy*2+dx: [Cout][Cin]
                W["bias"] = ops.bias_buffer(co, dev)
                wsrc = fl.ptr(op.name + ".upsample_transpose.weight")            # [Cin][Cout][2][2]
                pack.append(_seg(W["w"].data_ptr(), wsrc, [4, co, ci], [co * ci, ci, 1], [1, 4, co * 4], XF_BF16, XF_F32))
                if not self.teacher:
                    W["wt"] = bf16(4, ci, 1, 1, co)                              # dgrad of quadrant q: [Cin][Cout]
                    pack.append(_seg(W["wt"].data_ptr(), wsrc, [4, ci, co], [ci * co, co, 1], [1, co * 4, 4], XF_BF16, XF_F32))
                pack.append(_seg(W["bias"].data_ptr(), fl.ptr(op.name + ".upsample_transpose.bias"), [co], [1], [1], XF_F32, XF_F32))
                self.ctx[i] = dict(w=[W["w"][q] for q in range(4)])
                continue
            # ---- BN-ed blocks
            br = op_branches(op)
            nb, co, ci = len(br), op.cout, op.cin
            # QA blocks: stats [0] = BN_d (rbr_dense.bn), [1] = the post-sum bn; coef [0] / [1] = their backward coefficients
            self.stat_out[i] = torch.zeros(nb, 4, co, dtype=torch.float32, device=dev)
            if not self.teacher:
                self.coef_out[i] = torch.zeros(nb, 2, co, dtype=torch.float32, device=dev)
            W["br"] = []
            for b, (prefix, k) in enumerate(br):
                ent = dict(prefix=prefix, k=k, w=None)
                if k == 0:
                    W["br"].append(ent)
                    continue
                wsrc = fl.ptr(conv_weight_name(op, prefix)) + 4 * op.w_row0 * ci * k * k   # [Cout][Cin][k][k]
                if op.kind == "stem":
                    ent["w"] = torch.zeros(3, 3, 3, co, dtype=torch.float32, device=dev)   # [r][s][c][Cout], fp32 math
                    if k == 3:
                        pack.append(_seg(ent["w"].data_ptr(), wsrc, [9, 3, co], [3 * co, co, 1], [1, 9, 27], XF_F32, XF_F32))
                    else:       # 1x1 stride-2 branch = centre tap of a 3x3 stride-2 conv
                        pack.append(_seg(ent["w"].data_ptr() + 4 * (4 * 3 * co), wsrc, [3, co], [co, 1], [1, 3], XF_F32, XF_F32))
                    W["br"].append(ent)
                    continue
                kk = k * k
                ent["w"] = bf16(co, k, k, ci)                                    # forward: KRSC
                pack.append(_seg(ent["w"].data_ptr(), wsrc, [co, kk, ci], [kk * ci, ci, 1], [ci * kk, 1, kk], XF_BF16, XF_F32))
                W["br"].append(ent)
                if self.teacher:
                    continue
                if op.s == 1:   # dgrad = conv with the 180-degree rotated, transposed filter [Cin][k][k][Cout]
                    ent["wt"] = [bf16(ci, k, k, co)]
                    pack.append(_seg(ent["wt"][0].data_ptr(), wsrc + 4 * (kk - 1), [ci, kk, co], [kk * co, co, 1], [kk, -1, ci * kk],
                                     XF_BF16, XF_F32))
                elif k == 1:    # 1x1 stride 2 touches even positions only
                    ent["wt"] = [bf16(ci, 1, 1, co)]
                    pack.append(_seg(ent["wt"][0].data_ptr(), wsrc, [ci, co], [co, 1], [1, ci], XF_BF16, XF_F32))
                else:           # 3x3 stride 2: the input gradient at parity (ph, pw) is a 1- or 2-tap stride-1 conv
                    ent["wt"] = []
                    for ph in range(2):
                        for pw in range(2):
                            r0, dr, nr = (1, 0, 1) if ph == 0 else (2, -2, 2)    # tap t reads dc[i + t]: W[2] at t=0, W[0] at t=1
                            c0, dc, ncol = (1, 0, 1) if pw == 0 else (2, -2, 2)
                            wt = bf16(ci, nr, ncol, co)
                            pack.append(_seg(wt.data_ptr(), wsrc + 4 * (r0 * 3 + c0), [ci, nr, ncol, co],
                                             [nr * ncol * co, ncol * co, co, 1], [9, 3 * dr, dc, ci * 9], XF_BF16, XF_F32))
                            ent["wt"].append(wt)
            self.ctx[i] = dict(branches=[dict(prefix=e["prefix"], k=e["k"], w=e["w"], x=None) for e in W["br"]])
        self.pack_table = XformTable(pack, dev)
        self._zero_bytes = ztot
        if self.teacher:
            self.grad_tables, self.bucket_range = [], []
            return

        # ---- gradient unpack table, in backward order = flat gradient order; buckets = contiguous op ranges
        ops_with_params = [i for i in range(len(g.ops) - 1, -1, -1) if g.ops[i].kind != "pool"]
        total = fl.n_train
        bounds, acc, k = [], 0, 0
        per_bucket = [[] for _ in range(self.n_buckets)]
        self.bucket_range = []
        lo = 0
        for i in ops_with_params:
            op = g.ops[i]
            segs = self._grad_segs(i, op)
            size = sum(fl.slots[n][1] for n in op_param_names(op))
            per_bucket[k].extend(segs)
            self.bucket_of_op[i] = k
            acc += size
            if k < self.n_buckets - 1 and acc >= total * (k + 1) / self.n_buckets and op_param_names(op):
                hi = fl.slots[op_param_names(op)[-1]][0] + (fl.slots[op_param_names(op)[-1]][1] + 3) // 4 * 4
                self.bucket_range.append((lo, hi))
                lo = hi
                k += 1
        self.bucket_range.append((lo, total))
        while len(self.bucket_range) < self.n_buckets:
            self.bucket_range.append((total, total))
        self.grad_tables = [XformTable(s, dev) for s in per_bucket]
        self.last_op_of_bucket = {}
        for i in ops_with_params:
            self.last_op_of_bucket[self.bucket_of_op[i]] = i      # ops are visited in backward order: the last one wins

    def _grad_segs(self, i, op):
        """xform segments that move op i's gradients (fp32 KRSC arena / float64 sums) into the flat gradient buffer."""
        fl, z = self.flat, self._z
        segs = []
        if op.kind == "pred":
            ch, cin = op.cout, op.cin
            segs.append(_seg(fl.grad_ptr(op.name + ".weight"), z(i, "dw"), [ch * cin], [1], [1], XF_F32, XF_F32))
            segs.append(_seg(fl.grad_ptr(op.name + ".bias"), z(i, "bsum"), [ch], [1], [1], XF_F32, XF_F64))
            return segs
        if op.kind == "convT":
            co, ci = op.cout, op.cin
            segs.append(_seg(fl.grad_ptr(op.name + ".upsample_transpose.weight"), z(i, "dw"), [ci, co, 4], [co * 4, 4, 1],
                             [1, ci, co * ci], XF_F32, XF_F32))
            segs.append(_seg(fl.grad_ptr(op.name + ".upsample_transpose.bias"), z(i, "bsum"), [co], [1], [1], XF_F32, XF_F64))
            return segs
        br = op_branches(op)
        co, ci = op.cout, op.cin
        r0 = 4 * op.w_row0          # byte offset of the op's first row in per-channel vectors
        bns, post = branch_bn_names(op)
        for b, (prefix, k) in enumerate(br):
            wname = conv_weight_name(op, prefix)
            if k:
                if op.kind == "stem":
                    if k == 3:      # dw [Cout][32]: column (r*3+s)*3 + c -> [Cout][c][r][s]
                        segs.append(_seg(fl.grad_ptr(wname), z(i, "dw", b), [co, 3, 9], [27, 9, 1], [32, 1, 3],
                                         XF_F32, XF_F32))
                    else:           # the 1x1 stride-2 branch sees the centre tap (r = s = 1): columns 12..14
                        segs.append(_seg(fl.grad_ptr(wname), z(i, "dw", b) + 4 * 12, [co, 3], [3, 1], [32, 1], XF_F32, XF_F32))
                else:
                    kk = k * k      # dw [Cout][kk][Cin] -> [Cout][Cin][kk]
                    segs.append(_seg(fl.grad_ptr(wname) + r0 * ci * kk, z(i, "dw", b), [co, ci, kk], [ci * kk, kk, 1],
                                     [kk * ci, 1, ci], XF_F32, XF_F32))
            if post is not None:    # QA block: BN_d's sums come from its own backward launch
                if bns[b] is not None:
                    segs.append(_seg(fl.grad_ptr(bns[b] + ".weight"), z(i, "s2d"), [co], [1], [1], XF_F32, XF_F64))
                    segs.append(_seg(fl.grad_ptr(bns[b] + ".bias"), z(i, "s1d"), [co], [1], [1], XF_F32, XF_F64))
                continue
            bn = bns[b]
            segs.append(_seg(fl.grad_ptr(bn + ".weight") + r0, z(i, "s2") + 8 * b * co, [co], [1], [1], XF_F32, XF_F64))   # dgamma = sum dz * xhat
            segs.append(_seg(fl.grad_ptr(bn + ".bias") + r0, z(i, "s1"), [co], [1], [1], XF_F32, XF_F64))                 # dbeta = sum dz
        if post is not None:
            segs.append(_seg(fl.grad_ptr(post + ".weight"), z(i, "s2"), [co], [1], [1], XF_F32, XF_F64))
            segs.append(_seg(fl.grad_ptr(post + ".bias"), z(i, "s1"), [co], [1], [1], XF_F32, XF_F64))
        if op.alpha:
            segs.append(_seg(fl.grad_ptr(op.alpha), z(i, "dalpha"), [1], [1], [1], XF_F32, XF_F64))
        return segs

    # ================================================================== per-shape plan
    def _conv_desc(self, x, x_off, w, y, y_off=0, *, bias=None, y_strides=None, **kw):
        """y[..., y_off:+Cout] (+)= conv(x[..., x_off:+Cin], w) (ops.conv_desc).  x: [N,H,W,Ct] bf16, w: [Cout,kh,kw,Cin] bf16 KRSC,
        y: [N,Ho,Wo,Cyt] bf16 (or fp32 head tensor with explicit strides)."""
        return ops.conv_desc(x.data_ptr(), x.shape, w.data_ptr(), w.shape, y.data_ptr(), y_strides or y.stride()[:3], x_c_off=x_off,
                             y_c_off=y_off, bias=_p(bias), y_f32=y.dtype == torch.float32, **kw)

    def _wgrad_desc(self, x, x_off, cin, dy, dy_off, cout, k, stride, dw_ptr):
        d = WgradDesc()
        N, H, W, Ct = x.shape
        d.x = x.data_ptr() + x_off * 2
        d.N, d.H, d.W, d.Cin, d.x_c_total = N, H, W, cin, Ct
        d.dy = dy.data_ptr() + dy_off * 2
        d.Cout, d.dy_c_total = cout, dy.shape[3]
        d.kh = d.kw = k
        d.stride, d.pad = stride, k // 2
        d.dw = dw_ptr
        return d

    def _stats_desc(self, xs, c, pixels, sums_ptr, cnt_ptr, finalize=None, row0=0):
        """xs: [(tensor, channel offset)]; finalize: [(bn prefix, stats tensor [4][C])] or None (sums only); row0: the channels
        are rows [row0, row0 + c) of the BatchNorm."""
        d = BnStatsDesc()
        d.nb, d.C, d.pixels = len(xs), c, pixels
        for b, (t, off) in enumerate(xs):
            d.x[b] = t.data_ptr() + off * 2
            d.x_pitch[b] = t.shape[3]
        d.sums, d.counter, d.zeroed = sums_ptr, cnt_ptr, 1
        d.eps, d.momentum = BN_EPS, BN_MOMENTUM
        if finalize is not None:
            fl = self.flat
            for b, (prefix, st) in enumerate(finalize):
                d.gamma[b], d.beta[b] = fl.ptr(prefix + ".weight") + 4 * row0, fl.ptr(prefix + ".bias") + 4 * row0
                if not self.teacher:      # a teacher's running statistics stay as they are (null: no update)
                    d.running_mean[b] = fl.ptr(prefix + ".running_mean") + 4 * row0
                    d.running_var[b] = fl.ptr(prefix + ".running_var") + 4 * row0
                d.stats[b] = st.data_ptr()
        return d

    def _qa_desc(self, op, u, v, st, t, sums_ptr, cnt_ptr):
        """yv6_qa_fwd of a QA block: t = BN_d(u) + v (x / avg set by the caller), the post-sum bn finalised into st[1]."""
        fl, bn = self.flat, op.name + ".bn"
        q = QaDesc()
        q.N, q.H, q.W, q.C = t.shape
        q.u, q.u_pitch, q.v, q.v_pitch = u.data_ptr(), u.shape[3], v.data_ptr(), v.shape[3]
        q.scale_d, q.shift_d = st[0, 2].data_ptr(), st[0, 3].data_ptr()
        q.avg = int(op.avg)
        q.t, q.t_pitch = t.data_ptr(), t.shape[3]
        q.sums, q.counter, q.zeroed, q.eps, q.momentum = sums_ptr, cnt_ptr, 1, BN_EPS, BN_MOMENTUM
        q.gamma, q.beta = fl.ptr(bn + ".weight"), fl.ptr(bn + ".bias")
        q.stats = st[1].data_ptr()
        if not self.teacher:
            q.running_mean, q.running_var = fl.ptr(bn + ".running_mean"), fl.ptr(bn + ".running_var")
        return q

    def _dgrad_descs(self, dc, ent, stride, gsrc, g_off):
        """g(src)[..., g_off:+Cin] += conv_transpose(dc, w) as one (stride 1) or up to four (stride 2) accumulating convs: at
        stride 2 one conv per input parity (ph, pw), a 1- or 2-tap stride-1 conv each; a 1x1 conv touches parity (0, 0) only."""
        if stride == 1:
            return [self._conv_desc(dc, 0, ent["wt"][0], gsrc, g_off, accumulate=True)]
        n, hs, ws, gct = gsrc.shape
        return [self._conv_desc(dc, 0, wt, gsrc, g_off, pad=(0, 0), out_hw=tuple(dc.shape[1:3]), accumulate=True,
                                y_strides=(hs * ws * gct, 2 * ws * gct, 2 * gct), y_elem_off=(ph * ws + pw) * gct)
                for (ph, pw), wt in zip([(0, 0), (0, 1), (1, 0), (1, 1)], ent["wt"])]

    def _bf(self, *shape):
        return torch.zeros(*shape, dtype=torch.bfloat16, device=self.dev)

    def _new(self, shape, dtype=torch.bfloat16, zero=True):
        """A per-shape tensor of the plan: a view into the multi-shape arena, or a tensor of its own."""
        if self.arena is not None:
            return self.arena.take(tuple(shape), dtype)
        return (torch.zeros if zero else torch.empty)(*shape, dtype=dtype, device=self.dev)

    def _planned(self, op):
        """False for the pred convs a teacher leaves out: every head but the anchor-free cls / reg pair."""
        return not (self.teacher and op.kind == "pred" and op.head[0] not in ("cls", "reg"))

    def _view(self, t):
        return self.bufs[t.buf], self.gbufs[t.buf]

    def _dgrad_launch(self, d, op, full=True, group=None):
        """A dgrad conv accumulating into op's input gradient slice g(src)[..., c_off:+cin] (or, as its first writer, assigning)."""
        def assign(a):
            if a:           # y = conv(...) instead of y += conv(...): no residual read
                d.res, d.alpha = 0, 0.0
        return _desc_launch("conv", "yv6_conv_fwd", d, writes=[Write(op.src.buf, op.src.c_off, op.cin, full, assign, group)])

    def plan_shapes(self, N, shapes, in_dtype):
        """Multi-shape mode: one input buffer for the largest image and one arena for the per-shape tensors (activations,
        gradients, head outputs, scratch) sized for the largest single plan among `shapes` [(H, W)].  `_plan` then plans any
        of those shapes as views into the two buffers, at the same addresses every time."""
        if self.teacher:
            raise ValueError("a teacher's forward plan reads its student's input: it takes no shape list")
        shapes = [(int(h), int(w)) for h, w in shapes]
        self.x_store = torch.zeros(N * 3 * max(h * w for h, w in shapes), dtype=in_dtype, device=self.dev)
        need = 0
        for H, W in shapes:                   # measure each plan on a meta buffer: sizes only, no device memory
            self.arena, self._shape = _Arena(torch.empty(1 << 62, dtype=torch.uint8, device="meta")), None
            self._plan(N, H, W, in_dtype)
            need = max(need, self.arena.off)
        self.arena, self._shape = _Arena(torch.zeros(need, dtype=torch.uint8, device=self.dev)), None

    def make_live(self, H, W):
        """Multi-shape mode: clears the arena when (H, W) is not the shape whose tensors it holds (the input buffer is kept)."""
        if self.arena.live != (H, W):
            self.arena.store.zero_()
            self.arena.live = (H, W)

    def _plan(self, N, H, W, in_dtype, x_static=None):
        """Plans the step for one input shape.  x_static: an existing [N,3,H,W] input buffer for the stem to read (a teacher reads
        its student's), instead of one of the engine's own."""
        key = (N, H, W, in_dtype)
        if self._shape == key and (x_static is None or x_static is self.x_static):
            return
        g, dev = self.g, self.dev
        maxs = max(g.strides)
        if H % maxs or W % maxs or H <= 0 or W <= 0:      # as InferEngine._plan: every level's map must halve the previous one
            raise RuntimeError(f"input {H}x{W} must be a multiple of the largest stride {maxs}")
        self._shape = key
        if self.arena is not None:
            self.arena.off = 0
        self.bufs = [self._new((N, H >> b.level, W >> b.level, b.c_total)) for b in g.bufs]
        self.gbufs = [None] * len(self.bufs) if self.teacher else [self._new(t.shape) for t in self.bufs]
        self.sizes = [(H // s, W // s) for s in g.strides]
        self.offs = [0]
        for h, w in self.sizes:
            self.offs.append(self.offs[-1] + h * w)
        A = self.offs[-1]
        self.cls = self._new((N, A, g.num_classes), torch.float32, zero=False)
        self.reg = self._new((N, A, 4 * (g.reg_max + 1)), torch.float32, zero=False)
        if x_static is None and self.arena is not None:       # the largest shape's input buffer, outside the arena
            x_static = self.x_store[:N * 3 * H * W].view(N, 3, H, W)
        self.x_static = x_static if x_static is not None else torch.zeros(N, 3, H, W, dtype=in_dtype, device=dev)   # graph-stable address
        self.fwd_calls = []
        planners = {"pool": self._plan_pool, "pred": self._plan_pred, "convT": self._plan_convT}
        if self.teacher:                      # forward launches only: every planner returns no backward launches
            for i, op in enumerate(g.ops):
                if self._planned(op):
                    planners.get(op.kind, self._plan_bn_block)(i, op)
            self.bwd_calls, self.zero_gbufs = [], []
            return
        self.grad_cls = self._new(self.cls.shape, torch.float32)
        self.grad_reg = self._new(self.reg.shape, torch.float32)
        if getattr(g, "distill_ns", False):   # N / S distillation student: DFL logits next to the 4 lrtb distances
            self.reg_dist = self._new((N, A, g.dist_reg_ch), torch.float32, zero=False)
            self.grad_reg_dist = self._new(self.reg_dist.shape, torch.float32)
        if getattr(g, "fuse_ab", False):      # anchor-aided branch (effidehead_fuseab.py:94-140): 3 anchors per pixel, rows (level, anchor, pixel)
            from .arch import AB_ANCHORS
            self.cls_ab = self._new((N, AB_ANCHORS * A, g.num_classes), torch.float32, zero=False)
            self.reg_ab = self._new((N, AB_ANCHORS * A, 4), torch.float32, zero=False)
            self.grad_cls_ab = self._new(self.cls_ab.shape, torch.float32)
            self.grad_reg_ab = self._new(self.reg_ab.shape, torch.float32)
            self._ab = {}                     # level -> {"cls_ab" / "reg_ab": (fp32 conv output, bf16 gradient)}
        self.scratch = _Scratch(self._new, max([N * (H >> g.bufs[op.dst.buf].level) * (W >> g.bufs[op.dst.buf].level) * op.cout
                                          for op in g.ops if op.kind in ("conv", "stem")] + [1]))
        bwd_of_op = [planners.get(op.kind, self._plan_bn_block)(i, op) for i, op in enumerate(g.ops)]
        self.bwd_calls = []
        for i in range(len(g.ops) - 1, -1, -1):
            self.bwd_calls += bwd_of_op[i]
            k = self.bucket_of_op.get(i)
            if k is not None and self.last_op_of_bucket[k] == i:
                self.bwd_calls.append(Launch("bucket", None, kernels=0, parity=ALL, bucket=k))
        self._resolve_first_writers()
        if self.arena is not None and self.arena.store.device.type != "meta":
            self.arena.live = None            # a new plan starts from cleared tensors, as a single plan's torch.zeros
            self.make_live(H, W)

    # ------------------------------------------------------------------ one planner per op kind: each appends the op's forward
    # launches to self.fwd_calls and returns its backward launches
    def _plan_pool(self, i, op):
        """SPPF: y_j = maxpool5(y_{j-1}) into slice j of the concat, j = 1..3, in one launch; backward: three chained launches."""
        buf, gbuf = self._view(op.dst)
        n, h, w, ct = buf.shape
        c = op.cin
        self.fwd_calls.append(Launch("pool", "yv6_sppf_pool", (buf.data_ptr(), n, h, w, c, ct, 1, 0)))
        if self.teacher:
            return []
        scr = self.scratch.grown(self.scratch.pool, n * h * w * c, 1, torch.float32)[0]
        bwd = []
        for j in (3, 2, 1):
            args = [buf.data_ptr() + (j - 1) * c * 2, ct, gbuf.data_ptr() + j * c * 2, ct, n, h, w, c, scr.data_ptr(),
                    gbuf.data_ptr() + (j - 1) * c * 2, ct, 1]

            def assign(a, args=args):       # the last argument: accumulate into g(y_{j-1})
                args[-1] = 0 if a else 1
            bwd.append(Launch("pool_bwd", "yv6_maxpool5_bwd", args, kernels=2, writes=[Write(op.dst.buf, (j - 1) * c, c, True, assign)]))
        bwd[0].snapshot = (i, gbuf[..., :4 * c])
        return bwd

    def _plan_pred(self, i, op):
        """Head prediction conv (cls / reg / reg_dist, or a fuse_ab one); backward from the loss gradient of its head tensor."""
        src, _ = self._view(op.src)
        Wt, z = self.wts[i], self._z
        which, lvl = op.head
        N, A, ch = src.shape[0], self.offs[-1], op.cout
        lh, lw = self.sizes[lvl]
        chp = (ch + 15) // 16 * 16
        if not which.endswith("_ab"):
            out = {"cls": self.cls, "reg": self.reg, "reg_dist": getattr(self, "reg_dist", None)}[which]
            self.fwd_calls.append(_desc_launch("conv", "yv6_conv_fwd", self._conv_desc(src, op.src.c_off, Wt["w"], out, bias=Wt["bias"],
                                                                                      act=op.act, y_strides=(A * ch, lw * ch, ch),
                                                                                      y_elem_off=self.offs[lvl] * ch)))
            if self.teacher:
                return []
        dl = self._new((N, lh, lw, chp))               # bf16 gradient of the conv's output, zero padded to chp channels
        self.scratch.dl.append(dl)
        bwd = []
        if which.endswith("_ab"):
            # fuse_ab pred conv: natural NHWC output [N, hw, na * ch] (fp32, sigmoid fused on the class branch); the pack /
            # grad kernels (csrc/yv6_fuseab.cu) move between it and the reference's (level, anchor, pixel) row order
            raw = self._new((N, lh * lw, ch), torch.float32, zero=False)
            st = self._ab.setdefault(lvl, {})
            st[which] = (raw, dl)
            self.fwd_calls.append(_desc_launch("conv", "yv6_conv_fwd", self._conv_desc(src, op.src.c_off, Wt["w"], raw, bias=Wt["bias"],
                                                                                      act=op.act, y_strides=(lh * lw * ch, lw * ch, ch))))
            if which == "reg_ab":          # second of the level's pair in forward order, first in backward order
                from .arch import AB_ANCHORS
                (raw_c, dl_c), (raw_r, dl_r) = st["cls_ab"], st["reg_ab"]
                anchors = (C.c_float * 6)(*[v / float(self.g.strides[lvl]) for v in self.g.anchors_init[lvl]])   # effidehead_fuseab.py:35
                rows = (AB_ANCHORS, self.g.num_classes, anchors, AB_ANCHORS * self.offs[lvl], self.cls_ab.shape[1])
                self.fwd_calls.append(Launch("abp", "yv6_head_ab_pack", (raw_c.data_ptr(), raw_r.data_ptr(), N, lh * lw, *rows,
                                                                         self.cls_ab.data_ptr(), self.reg_ab.data_ptr())))
                bwd.append(Launch("abg", "yv6_head_ab_grad", (self.grad_cls_ab.data_ptr(), self.cls_ab.data_ptr(), self.grad_reg_ab.data_ptr(),
                                                              raw_r.data_ptr(), N, lh * lw, *rows, dl_c.shape[3], dl_r.shape[3],
                                                              dl_c.data_ptr(), dl_r.data_ptr())))
        else:
            grad = {"cls": self.grad_cls, "reg": self.grad_reg, "reg_dist": getattr(self, "grad_reg_dist", None)}[which]
            bwd.append(Launch("hgp", "yv6_head_grad_prep", (grad.data_ptr(), self.cls.data_ptr() if which == "cls" else 0, N, A, ch,
                                                             self.offs[lvl], lh * lw, chp, dl.data_ptr())))
        bwd.append(_desc_launch("wgrad", "yv6_conv_wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dl, 0, ch, 1, 1, z(i, "dw")), side=True))
        bwd.append(_desc_launch("stats", "yv6_bn_stats_finalize", self._stats_desc([(dl, 0)], chp, N * lh * lw, z(i, "bsum"), z(i, "bcnt"))))
        bwd.append(self._dgrad_launch(self._conv_desc(dl, 0, Wt["wt"], self.gbufs[op.src.buf], op.src.c_off, accumulate=True), op))
        return bwd

    def _plan_convT(self, i, op):
        """ConvTranspose2d(k=2, s=2): four 1x1 convs, one per output quadrant (dy, dx), in the forward and the backward."""
        src, gsrc = self._view(op.src)
        dst, gdst = self._view(op.dst)
        Wt, z = self.wts[i], self._z
        N, dh, dw, dct = dst.shape
        _, sh, sw, _ = src.shape
        for q in range(4):
            dy, dx = q // 2, q % 2
            self.fwd_calls.append(_desc_launch("conv", "yv6_conv_fwd", self._conv_desc(
                src, op.src.c_off, Wt["w"][q], dst, op.dst.c_off, bias=Wt["bias"], y_strides=(dh * dw * dct, 2 * dw * dct, 2 * dct),
                y_elem_off=(dy * dw + dx) * dct)))
        if self.teacher:
            return []
        gd = gdst[..., op.dst.c_off:op.dst.c_off + op.cout]
        # bias gradient = column sums of the whole upsampled gradient slice
        bwd = [_desc_launch("stats", "yv6_bn_stats_finalize", self._stats_desc([(gdst, op.dst.c_off)], op.cout, N * dh * dw, z(i, "bsum"),
                                                                                z(i, "bcnt")), snapshot=(i, gd))]
        need = N * sh * sw * op.cout
        pool = self.scratch.grown(self.scratch.quad, need, 4, torch.bfloat16)
        for q in range(4):
            dy, dx = q // 2, q % 2
            dq = pool[q][:need].view(N, sh, sw, op.cout)
            # the gradient of quadrant q, dense; the quadrant buffers are reused, so the copy waits for every weight gradient
            bwd.append(Launch("copy", lambda sp, dq=dq, s=gd[:, dy::2, dx::2, :]: dq.copy_(s), parity=ALL))
            bwd.append(_desc_launch("wgrad", "yv6_conv_wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dq, 0, op.cout, 1, 1,
                                                                                z(i, "dw") + 4 * q * op.cout * op.cin), side=True))
            bwd.append(self._dgrad_launch(self._conv_desc(dq, 0, Wt["wt"][q], gsrc, op.src.c_off, accumulate=True), op))
        return bwd

    def _plan_bn_block(self, i, op):
        """BatchNorm-ed block (stem / rep / cba / cm / qa): raw convs of its branches -> batch statistics -> BN apply +
        activation.  Backward: BN backward into the dc scratch pair of the block's parity, then _plan_branch_grads."""
        z = self._z
        dst, gdst = self._view(op.dst)
        src, gsrc = self._view(op.src) if op.kind != "stem" else (None, None)
        n, ho, wo, dct = dst.shape
        count = n * ho * wo
        br, st = self.wts[i]["br"], self.stat_out[i]
        xs = []
        for b, ent in enumerate(br):
            if ent["k"] == 0:
                xs.append((src, op.src.c_off))
            else:
                raw = self._new((n, ho, wo, op.cout))
                if op.kind == "stem":
                    N, H, W, in_dtype = self._shape
                    self.fwd_calls.append(_desc_launch("stem", "yv6_stem_fwd", ops.stem_desc(
                        self.x_static.data_ptr(), N, H, W, in_dtype == torch.uint8, ent["w"].data_ptr(), 0, op.cout, None, raw.data_ptr(),
                        fp32_math=1)))
                else:
                    self.fwd_calls.append(_desc_launch("conv", "yv6_conv_fwd", self._conv_desc(src, op.src.c_off, ent["w"], raw, stride=op.s)))
                xs.append((raw, 0))
            self.ctx[i]["branches"][b]["x"] = xs[-1][0]
        if op.layout == "qa":
            xs, st = self._plan_qa_fwd(i, op, xs, count), st[1:]
        else:
            fin = [(ent["prefix"] + (".bn" if ent["k"] else ""), st[b]) for b, ent in enumerate(br)]
            self.fwd_calls.append(_desc_launch("stats", "yv6_bn_stats_finalize", self._stats_desc(
                xs, op.cout, count, z(i, "fsum"), z(i, "fcnt"), fin, op.w_row0)))
        d = BnDesc()
        d.nb, d.act, d.C, d.pixels = len(xs), ACT_CODES[op.act], op.cout, count
        for b, (t, off) in enumerate(xs):
            d.x[b], d.x_pitch[b] = t.data_ptr() + off * 2, t.shape[3]
            d.mean[b], d.invstd[b] = st[b, 0].data_ptr(), st[b, 1].data_ptr()
            d.scale[b], d.shift[b] = st[b, 2].data_ptr(), st[b, 3].data_ptr()
        d.y, d.y_pitch = dst.data_ptr() + op.dst.c_off * 2, dct
        if op.res is not None:
            rbuf, grbuf = self._view(op.res)
            d.res, d.res_pitch, d.res_alpha = rbuf.data_ptr() + op.res.c_off * 2, rbuf.shape[3], 1.0
            if op.alpha in self.params:
                d.res_alpha_dev = self.flat.ptr(op.alpha)
        self.fwd_calls.append(_desc_launch("apply", "yv6_bn_apply_fwd", d))
        if self.teacher:
            return []
        sc = self.scratch        # the backward launch runs on the same descriptor
        par, sc.bn_ops = sc.bn_ops & 1, sc.bn_ops + 1
        dcs, writes = [], []     # writes: the gradient slices this launch writes besides the scratch tensors
        for b in range(len(xs)):
            d.s2[b] = z(i, "s2") + 8 * b * op.cout
            if br[b]["k"] == 0:      # identity branch: its input gradient goes straight into g(src)
                d.dx[b], d.dx_pitch[b], d.accumulate[b] = gsrc.data_ptr() + op.src.c_off * 2, gsrc.shape[3], 1

                def dx_assign(a, b=b):
                    d.accumulate[b] = 0 if a else 1
                writes.append(Write(op.src.buf, op.src.c_off, op.cin, True, dx_assign))
                dcs.append(None)
            else:
                dc = sc.dc_view(par, len([t for t in dcs if t is not None]), (n, ho, wo, op.cout))
                d.dx[b], d.dx_pitch[b], d.accumulate[b] = dc.data_ptr(), op.cout, 0
                dcs.append(dc)
        d.dy, d.dy_pitch = gdst.data_ptr() + op.dst.c_off * 2, dct
        d.s1 = z(i, "s1")
        d.work, d.counter, d.coef, d.zeroed = z(i, "work"), z(i, "bcnt"), self.coef_out[i].data_ptr(), 1
        if op.res is not None:
            d.dres, d.dres_pitch, d.dalpha = grbuf.data_ptr() + op.res.c_off * 2, grbuf.shape[3], z(i, "dalpha")
            writes.append(Write(op.res.buf, op.res.c_off, op.cout, True, lambda a: setattr(d, "dres_assign", int(a))))
        bwd = [_desc_launch("bn_bwd", "yv6_bn_bwd", d, kernels=2, parity=par, writes=writes,
                            snapshot=(i, gdst[..., op.dst.c_off:op.dst.c_off + op.cout]))]
        if op.layout == "qa":
            qa_bwd, dcs = self._plan_qa_bwd(i, op, dcs[0], par)
            bwd += qa_bwd
        return bwd + self._plan_branch_grads(i, op, dcs, par)

    def _plan_qa_fwd(self, i, op, xs, count):
        """QA block: BN_d statistics of u, then t = BN_d(u) + v [+ x [+ avg3x3 x]] with the post-sum bn's statistics in one
        launch.  Returns [(t, 0)]: from here on the block is a one-branch BatchNorm over t."""
        z, st = self._z, self.stat_out[i]
        (u, _), (v, _) = xs
        self.fwd_calls.append(_desc_launch("stats", "yv6_bn_stats_finalize", self._stats_desc(
            [xs[0]], op.cout, count, z(i, "fsum"), z(i, "fcnt"), [(op.name + ".rbr_dense.bn", st[0])])))
        tq = self._new(u.shape)
        q = self._qa_desc(op, u, v, st, tq, z(i, "qsum"), z(i, "qcnt"))
        if op.identity:
            src = self.bufs[op.src.buf]
            q.x, q.x_pitch = src.data_ptr() + op.src.c_off * 2, src.shape[3]
        self.fwd_calls.append(_desc_launch("qa", "yv6_qa_fwd", q))
        self.ctx[i].update(u=u, v=v, t=tq, stats_d=st[0], stats_p=st[1])
        return [(tq, 0)]

    def _plan_qa_bwd(self, i, op, dt, par):
        """QA block after the post-sum bn's backward: dt -> BN_d backward (no activation) -> du; dt also feeds the 1x1 branch and
        the parameter-free identity / average-pool branches (yv6_qa_bwd into g(x)).  Returns the launches and the gradients of
        the conv branches' outputs, [du, dt]."""
        z, ctx = self._z, self.ctx[i]
        du = self.scratch.dc_view(par, 1, dt.shape)
        sd = self.stat_out[i][0]
        d = BnDesc()
        d.nb, d.act, d.C, d.pixels = 1, ACT_CODES[None], op.cout, dt.numel() // op.cout
        d.x[0], d.x_pitch[0] = ctx["u"].data_ptr(), op.cout
        d.mean[0], d.invstd[0], d.scale[0], d.shift[0] = (sd[r].data_ptr() for r in range(4))
        d.s2[0], d.s1 = z(i, "s2d"), z(i, "s1d")
        d.dx[0], d.dx_pitch[0], d.accumulate[0] = du.data_ptr(), op.cout, 0
        d.dy, d.dy_pitch = dt.data_ptr(), op.cout
        d.work, d.counter, d.coef, d.zeroed = z(i, "workd"), z(i, "bcntd"), self.coef_out[i][1].data_ptr(), 1
        bwd = [_desc_launch("bn_bwd", "yv6_bn_bwd", d, kernels=2, parity=par)]
        if op.identity:
            gsrc = self.gbufs[op.src.buf]
            qb = self._qa_desc(op, ctx["u"], ctx["v"], self.stat_out[i], ctx["t"], 0, 0)
            qb.dt, qb.dt_pitch = dt.data_ptr(), op.cout
            qb.dx, qb.dx_pitch = gsrc.data_ptr() + op.src.c_off * 2, gsrc.shape[3]
            bwd.append(_desc_launch("qa_bwd", "yv6_qa_bwd", qb, writes=[Write(op.src.buf, op.src.c_off, op.cin, True,
                                                                               lambda a: setattr(qb, "accumulate", int(not a)))]))
        return bwd, [du, dt]

    def _plan_branch_grads(self, i, op, dcs, par):
        """Weight gradients (side stream; they read the dc pair `par`) and input gradients of the conv branches of a BN-ed block,
        from the gradients dcs[b] of the branches' raw outputs."""
        z, br = self._z, self.wts[i]["br"]
        bwd = []
        if op.kind == "stem":       # im2col once, then one tensor-core wgrad GEMM per branch
            N, H, W, in_dtype = self._shape
            patches, patches_lo = self._new((*dcs[0].shape[:3], 32)), self._new((*dcs[0].shape[:3], 32))     # image = hi + lo (bf16 planes)
            self._stem_patches = (patches, patches_lo)
            bwd.append(Launch("im2col", "yv6_stem_im2col", (self.x_static.data_ptr(), DT_U8 if in_dtype == torch.uint8 else DT_F32,
                                                            1.0 / 255.0, N, H, W, patches.data_ptr(), patches_lo.data_ptr())))
            for b in range(len(br)):
                for pl in (patches, patches_lo):
                    bwd.append(_desc_launch("wgrad", "yv6_conv_wgrad", self._wgrad_desc(pl, 0, 32, dcs[b], 0, op.cout, 1, 1, z(i, "dw", b)),
                                            side=True, parity=par))
            return bwd
        src, gsrc = self._view(op.src)
        for b, ent in enumerate(br):
            if ent["k"] == 0:
                continue
            bwd.append(_desc_launch("wgrad", "yv6_conv_wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dcs[b], 0, op.cout, ent["k"], op.s,
                                                                                z(i, "dw", b)), side=True, parity=par))
            # a stride-2 3x3 dgrad = four parity convolutions that together cover every pixel; 1x1 stride 2 covers one parity
            full = op.s == 1 or ent["k"] == 3
            for d in self._dgrad_descs(dcs[b], ent, op.s, gsrc, op.src.c_off):
                bwd.append(self._dgrad_launch(d, op, full, group=(i, b)))
        return bwd

    def _resolve_first_writers(self):
        """Gradient buffers are accumulated into by every consumer of a tensor.  Instead of clearing all of them at the start of
        the backward pass (one more pass over every activation gradient) the FIRST writer of a channel slice assigns and
        the later ones accumulate; only buffers whose first writer cannot assign (it covers part of the pixels, or part of
        a slice that is already partly written) are still cleared."""
        cov = [np.zeros(b.c_total, dtype=bool) for b in self.g.bufs]
        need_zero = set()
        group_decision = {}
        if self.external_feat_grads:         # backward() writes the external gradient (or zeros) into these slices first
            for t in self.g.feat:
                cov[t.buf][t.c_off:t.c_off + t.c] = True

        def decide(w):
            seg = cov[w.buf][w.off:w.off + w.n]
            if w.full and not seg.any():
                assign = True
            else:
                assign = False
                if not seg.all():
                    need_zero.add(w.buf)
            seg[:] = True
            return assign

        for launch in self.bwd_calls:
            for w in launch.writes:
                if w.group is None:
                    w.assign(decide(w))
                else:
                    if w.group not in group_decision:
                        group_decision[w.group] = decide(w)
                    w.assign(group_decision[w.group])
        for i, cv in enumerate(cov):        # slices nobody writes are read as zero gradients
            if not cv.all():
                need_zero.add(i)
        self.zero_gbufs = [self.gbufs[i] for i in sorted(need_zero)]

    # ================================================================== execution
    def launch_counts(self):
        """(forward, backward) kernel launches of the current plan, excluding the arena memset and the two repack launches; every
        gradient unpack table counts once."""
        return sum(c.kernels for c in self.fwd_calls), sum(c.kernels for c in self.bwd_calls) + len(self.grad_tables)

    def begin_step(self, sp=None):
        """Clears the per-step accumulators and repacks the master weights into the kernels' layouts."""
        sp = sp or _lib.stream_ptr()
        self.zero_arena.zero_()
        self.pack_table.launch(self.lib, self.h, False, sp)

    def forward(self, x):
        """x [N,3,H,W] fp32 in [0,1] (or uint8).  Returns (cls [N,A,nc] post-sigmoid, reg [N,A,R]) fp32 (engine-owned)."""
        if not self.flat.valid():
            raise RuntimeError("the model's tensors were replaced after the training engine was built (model.to / .half); "
                               "call model.train_engine(rebuild=True)")
        N, _, H, W = x.shape
        if x.dtype not in (torch.float32, torch.uint8):
            x = x.float()
        self._plan(N, H, W, x.dtype)
        if x.data_ptr() != self.x_static.data_ptr():
            self.x_static.copy_(x)
        sp = _lib.stream_ptr()
        self.begin_step(sp)
        if not self.teacher:
            self.flat.iflat.add_(1)                 # BatchNorm.num_batches_tracked
        self.run_forward(sp)
        return self.cls, self.reg

    def run_forward(self, sp):
        for c in self.fwd_calls:
            c.run(self.lib, self.h, sp)

    def backward(self, grad_cls, grad_reg, accumulate=False, first=0, last=None, grad_cls_ab=None, grad_reg_ab=None, grad_reg_dist=None):
        """Writes d(loss)/d(parameter) of every trainable parameter into the flat gradient buffer (`accumulate`: adds to it)
        given d(loss)/d(cls), d(loss)/d(reg) ([N,A,*] fp32).  `first`/`last` restrict the run to a slice of the call list
        (graph capture in bucket-sized segments)."""
        if grad_cls is not None and grad_cls.data_ptr() != self.grad_cls.data_ptr():
            self.grad_cls.copy_(grad_cls)
        if grad_reg is not None and grad_reg.data_ptr() != self.grad_reg.data_ptr():
            self.grad_reg.copy_(grad_reg)
        if getattr(self.g, "distill_ns", False) and first == 0 and grad_reg_dist is not None and grad_reg_dist.data_ptr() != self.grad_reg_dist.data_ptr():
            self.grad_reg_dist.copy_(grad_reg_dist)
        if getattr(self.g, "fuse_ab", False) and first == 0:      # None = the engine's own buffers were filled by the loss kernels
            for buf, gr in ((self.grad_cls_ab, grad_cls_ab), (self.grad_reg_ab, grad_reg_ab)):
                if gr is not None and gr.data_ptr() != buf.data_ptr():
                    buf.copy_(gr)
        lib, h = self.lib, self.h
        sp = _lib.stream_ptr()
        if first == 0:
            for gb in self.zero_gbufs:
                gb.zero_()
        if self.external_feat_grads and first == 0:       # after the clears above: these slices start from the external gradient
            fg = self._feat_grads or [None] * len(self.g.feat)
            for t, gr in zip(self.g.feat, fg):
                sl = self.gbufs[t.buf][..., t.c_off:t.c_off + t.c]
                if gr is None:
                    sl.zero_()
                else:
                    sl.copy_(gr.permute(0, 2, 3, 1))                 # NCHW fp32 -> NHWC bf16
            self._feat_grads = None
        calls = self.bwd_calls if last is None else self.bwd_calls[:last]
        # Weight gradients leave the critical path: a wgrad only feeds the gradient buffer, so it runs on a side stream next to
        # the dgrad of its own op and the (HBM-bound) BatchNorm backward of the next one.  Hazards: its dY operand lives in the
        # scratch pair of its op's parity (the BN backward two ops later waits for it), the transposed-conv quadrant copies reuse
        # their scratch (they wait for everything), and a bucket's unpack reads the accumulators (waits for everything).
        overlap = self.overlap_wgrad
        main = torch.cuda.current_stream(self.dev)
        if overlap and self._wg_stream is None:
            self._wg_stream = torch.cuda.Stream(device=self.dev)
        side = self._wg_stream
        ssp = _lib.stream_ptr(side) if overlap else sp
        pending = []             # (event recorded on the side stream after a wgrad, scratch parity or None)

        def wait_pending(par=ALL):
            for ev, q in pending:
                if par == ALL or q == par:
                    main.wait_event(ev)
            pending[:] = [(ev, q) for ev, q in pending if not (par == ALL or q == par)]

        for c in calls[first:]:
            if self.debug and c.snapshot is not None:
                self.dbg[c.snapshot[0]] = dict(gdst=c.snapshot[1].clone())
            if overlap and c.side:
                ev = torch.cuda.Event()
                ev.record(main)
                side.wait_event(ev)
                c.run(lib, h, ssp)
                done = torch.cuda.Event()
                done.record(side)
                pending.append((done, c.parity))
                continue
            if overlap and c.parity is not None:
                wait_pending(c.parity)
            if c.bucket is not None:
                self.grad_tables[c.bucket].launch(lib, h, accumulate, sp)
                if self.bucket_hook is not None:
                    self.bucket_hook(c.bucket)
            else:
                c.run(lib, h, sp)
        if overlap:
            wait_pending()      # every call (and every captured graph segment) ends joined

    def neck_outputs(self):
        """The neck outputs of the last forward as NCHW fp32 copies (the reference's `featmaps`, yolo.py:37-39)."""
        return [self.bufs[t.buf][..., t.c_off:t.c_off + t.c].permute(0, 3, 1, 2).float().contiguous() for t in self.g.feat]

    def bucket_call_index(self):
        """Indices into the backward call list right after each bucket's unpack (segment boundaries for graph capture)."""
        return [j + 1 for j, c in enumerate(self.bwd_calls) if c.bucket is not None]


class _HeadFn(torch.autograd.Function):
    """Connects the engine to autograd: forward returns the head tensors, backward runs the engine's backward pass and
    hands every parameter its gradient, so `loss.backward()`, GradScaler, gradient accumulation and the reducer hooks of
    DistributedDataParallel (core/engine.py:456-468) behave as they do for the reference's nn.Module."""

    @staticmethod
    def forward(ctx, engine, x, *params):
        ctx.engine = engine
        cls, reg = engine.forward(x)
        heads = [cls.clone(), reg.clone()]
        if getattr(engine.g, "fuse_ab", False):
            heads += [engine.cls_ab.clone(), engine.reg_ab.clone()]
        if getattr(engine.g, "distill_ns", False):
            heads += [engine.reg_dist.clone()]
        ctx.n_heads = len(heads)
        feats = engine.neck_outputs() if engine.external_feat_grads else []
        return (*heads, *feats)

    @staticmethod
    def backward(ctx, *grads):
        eng = ctx.engine
        g_cls, g_reg = grads[0], grads[1]
        extra = list(grads[2:ctx.n_heads])
        g_feats = list(grads[ctx.n_heads:])
        g_cls_ab = g_reg_ab = g_reg_dist = None
        if getattr(eng.g, "fuse_ab", False):
            g_cls_ab, g_reg_ab = extra[0], extra[1]
        if getattr(eng.g, "distill_ns", False):       # third output = the DFL branch
            g_reg_dist = torch.zeros_like(eng.grad_reg_dist) if extra[0] is None else extra[0].contiguous().float()
        f = lambda t: None if t is None else t.contiguous().float()   # noqa: E731
        # an output the loss did not use has no gradient: zero (None would mean "the engine's own buffer is already filled")
        g_cls = torch.zeros_like(eng.grad_cls) if g_cls is None else g_cls
        g_reg = torch.zeros_like(eng.grad_reg) if g_reg is None else g_reg
        if getattr(eng.g, "fuse_ab", False):
            g_cls_ab = torch.zeros_like(eng.grad_cls_ab) if g_cls_ab is None else g_cls_ab
            g_reg_ab = torch.zeros_like(eng.grad_reg_ab) if g_reg_ab is None else g_reg_ab
        if eng.external_feat_grads:
            eng._feat_grads = g_feats
        eng.backward(f(g_cls), f(g_reg), grad_cls_ab=f(g_cls_ab), grad_reg_ab=f(g_reg_ab), grad_reg_dist=g_reg_dist)
        flat = eng.flat
        g = flat.gflat.clone()          # autograd may keep (steal) what it is given; the flat buffer is reused next step
        grads = []
        for n in flat.names:
            o, k, shape = flat.slots[n]
            grads.append(g[o:o + k].view(shape))
        return (None, None, *grads)


def train_forward(engine, x):
    params = [engine.params[n] for n in engine.flat.names]
    return _HeadFn.apply(engine, x, *params)
