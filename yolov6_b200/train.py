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


class TrainEngine:
    def __init__(self, model, n_buckets=1):
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

        def bf16(*shape):
            return torch.zeros(*shape, dtype=torch.bfloat16, device=dev)

        for i, op in enumerate(g.ops):
            if op.kind == "pool":
                continue
            W = self.wts[i] = {}
            if op.kind == "pred":
                ch, cin, chp = op.cout, op.cin, (op.cout + 15) // 16 * 16
                W["w"] = bf16(ch, 1, 1, cin)
                W["bias"] = ops.bias_buffer(ch, dev)
                W["wt"] = bf16(cin, 1, 1, chp)                                   # dgrad: [Cin][ch_pad], zero padded
                wsrc, bsrc = fl.ptr(op.name + ".weight"), fl.ptr(op.name + ".bias")
                pack.append(_seg(W["w"].data_ptr(), wsrc, [ch * cin], [1], [1], XF_BF16, XF_F32))
                pack.append(_seg(W["bias"].data_ptr(), bsrc, [ch], [1], [1], XF_F32, XF_F32))
                pack.append(_seg(W["wt"].data_ptr(), wsrc, [cin, ch], [chp, 1], [1, cin], XF_BF16, XF_F32))
                self.ctx[i] = dict(w=W["w"])
                continue
            if op.kind == "convT":
                co, ci = op.cout, op.cin
                W["w"] = bf16(4, co, 1, 1, ci)                                   # quadrant q = dy*2+dx: [Cout][Cin]
                W["wt"] = bf16(4, ci, 1, 1, co)                                  # dgrad of quadrant q: [Cin][Cout]
                W["bias"] = ops.bias_buffer(co, dev)
                wsrc = fl.ptr(op.name + ".upsample_transpose.weight")            # [Cin][Cout][2][2]
                pack.append(_seg(W["w"].data_ptr(), wsrc, [4, co, ci], [co * ci, ci, 1], [1, 4, co * 4], XF_BF16, XF_F32))
                pack.append(_seg(W["wt"].data_ptr(), wsrc, [4, ci, co], [ci * co, co, 1], [1, co * 4, 4], XF_BF16, XF_F32))
                pack.append(_seg(W["bias"].data_ptr(), fl.ptr(op.name + ".upsample_transpose.bias"), [co], [1], [1], XF_F32, XF_F32))
                self.ctx[i] = dict(w=[W["w"][q] for q in range(4)])
                continue
            # ---- BN-ed blocks
            br = op_branches(op)
            nb, co, ci = len(br), op.cout, op.cin
            # QA blocks: stats [0] = BN_d (rbr_dense.bn), [1] = the post-sum bn; coef [0] / [1] = their backward coefficients
            self.stat_out[i] = torch.zeros(nb, 4, co, dtype=torch.float32, device=dev)
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
                W["br"].append(ent)
            self.ctx[i] = dict(branches=[dict(prefix=e["prefix"], k=e["k"], w=e["w"], x=None) for e in W["br"]])
        self.pack_table = XformTable(pack, dev)

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
        self._zero_bytes = ztot

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
        q.running_mean, q.running_var, q.stats = fl.ptr(bn + ".running_mean"), fl.ptr(bn + ".running_var"), st[1].data_ptr()
        return q

    def _dgrad_descs(self, dc, ent, k, stride, gsrc, g_off):
        """g(src)[..., g_off:+Cin] += conv_transpose(dc, w) as one (stride 1) or up to four (stride 2) accumulating convs."""
        if stride == 1:
            return [self._conv_desc(dc, 0, ent["wt"][0], gsrc, g_off, accumulate=True)]
        n, hs, ws, gct = gsrc.shape
        ho, wo = dc.shape[1], dc.shape[2]
        out = []
        j = 0
        for ph in range(2):
            for pw in range(2):
                if k == 1:
                    if ph or pw:
                        continue
                    wt = ent["wt"][0]
                else:
                    wt = ent["wt"][j]
                    j += 1
                out.append(self._conv_desc(dc, 0, wt, gsrc, g_off, pad=(0, 0), out_hw=(ho, wo), accumulate=True,
                                           y_strides=(hs * ws * gct, 2 * ws * gct, 2 * gct), y_elem_off=(ph * ws + pw) * gct))
        return out

    def _plan(self, N, H, W, in_dtype):
        key = (N, H, W, in_dtype)
        if self._shape == key:
            return
        self._shape = key
        g, dev, fl, z = self.g, self.dev, self.flat, self._z
        bf = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device=dev)   # noqa: E731
        self.bufs = [bf(N, H >> b.level, W >> b.level, b.c_total) for b in g.bufs]
        self.gbufs = [torch.zeros_like(t) for t in self.bufs]
        self.sizes = [(H // s, W // s) for s in g.strides]
        self.offs = [0]
        for h, w in self.sizes:
            self.offs.append(self.offs[-1] + h * w)
        A = self.offs[-1]
        self.cls = torch.empty(N, A, g.num_classes, dtype=torch.float32, device=dev)
        self.reg = torch.empty(N, A, 4 * (g.reg_max + 1), dtype=torch.float32, device=dev)
        self.grad_cls = torch.zeros_like(self.cls)
        self.grad_reg = torch.zeros_like(self.reg)
        if getattr(g, "distill_ns", False):   # N / S distillation student: DFL logits next to the 4 lrtb distances
            self.reg_dist = torch.empty(N, A, g.dist_reg_ch, dtype=torch.float32, device=dev)
            self.grad_reg_dist = torch.zeros_like(self.reg_dist)
        if getattr(g, "fuse_ab", False):      # anchor-aided branch (effidehead_fuseab.py:94-140): 3 anchors per pixel, rows (level, anchor, pixel)
            from .arch import AB_ANCHORS
            self.cls_ab = torch.empty(N, AB_ANCHORS * A, g.num_classes, dtype=torch.float32, device=dev)
            self.reg_ab = torch.empty(N, AB_ANCHORS * A, 4, dtype=torch.float32, device=dev)
            self.grad_cls_ab = torch.zeros_like(self.cls_ab)
            self.grad_reg_ab = torch.zeros_like(self.reg_ab)
            self._ab = {}                     # level -> dict(raw_cls, raw_reg, dl_cls, dl_reg, anchors)
        self.x_static = torch.zeros(N, 3, H, W, dtype=in_dtype, device=dev)   # the stem reads this buffer (graph-stable address)
        view = lambda t: (self.bufs[t.buf], self.gbufs[t.buf])   # noqa: E731
        # shared scratch: BN-backward outputs (gradients w.r.t. the raw conv outputs) live only until their dgrad / wgrad ran
        dc_elems = max([N * (H >> g.bufs[op.dst.buf].level) * (W >> g.bufs[op.dst.buf].level) * op.cout
                        for op in g.ops if op.kind in ("conv", "stem")] + [1])
        # (two per op parity: the weight gradients of an op run on a side stream while the next op's BN backward refills the other pair)
        dc_pool = [torch.zeros(dc_elems, dtype=torch.bfloat16, device=dev) for _ in range(4)]
        bn_ops = 0
        pool_scr, dq_pool = None, None
        fwd, bwd_rev = [], []        # bwd_rev[j] = list of calls of op j (assembled in reverse op order afterwards)
        x_dt = DT_U8 if in_dtype == torch.uint8 else DT_F32
        for i, op in enumerate(g.ops):
            calls = []
            if op.kind == "pool":
                buf, gbuf = view(op.dst)
                n, h, w, ct = buf.shape
                c = op.cin
                fwd.append(("pool", (buf.data_ptr(), n, h, w, c, ct, 1, 0)))
                if pool_scr is None or pool_scr.numel() < n * h * w * c:
                    pool_scr = torch.zeros(n * h * w * c, dtype=torch.float32, device=dev)
                calls.append(("dbg", (i, gbuf[..., :4 * c])))
                for j in (3, 2, 1):   # y_j = pool(y_{j-1}); slice j of the concat
                    calls.append(("pool_bwd", [buf.data_ptr() + (j - 1) * c * 2, ct, gbuf.data_ptr() + j * c * 2, ct, n, h, w, c,
                                               pool_scr, gbuf.data_ptr() + (j - 1) * c * 2, ct, 1],
                                  dict(buf=op.dst.buf, off=(j - 1) * c, n=c, full=True)))
                bwd_rev.append(calls)
                continue
            Wt = self.wts[i]
            if op.kind == "pred" and op.head[0].endswith("_ab"):
                # fuse_ab pred conv: natural NHWC output [N, hw, na * ch] (fp32, sigmoid fused on the class branch); the pack /
                # grad kernels (csrc/yv6_fuseab.cu) move between it and the reference's (level, anchor, pixel) row order
                from .arch import AB_ANCHORS
                src, gsrc = view(op.src)
                which, lvl = op.head
                lh, lw = self.sizes[lvl]
                ch, chp = op.cout, (op.cout + 15) // 16 * 16
                st = self._ab.setdefault(lvl, {})
                raw = torch.empty(N, lh * lw, ch, dtype=torch.float32, device=dev)
                dl = bf(N, lh, lw, chp)
                st["raw_" + which[:3]], st["dl_" + which[:3]] = raw, dl
                fwd.append(("conv", self._conv_desc(src, op.src.c_off, Wt["w"], raw, bias=Wt["bias"], act=op.act,
                                                    y_strides=(lh * lw * ch, lw * ch, ch))))
                if which == "reg_ab":          # second of the level's pair in forward order, first in backward order
                    anc = [v / float(g.strides[lvl]) for v in g.anchors_init[lvl]]          # effidehead_fuseab.py:35
                    st["anchors"] = (C.c_float * 6)(*anc)
                    fwd.append(("abp", lvl))
                    calls.append(("abg", lvl))
                calls.append(("wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dl, 0, ch, 1, 1, z(i, "dw"))))
                calls.append(("stats", self._stats_desc([(dl, 0)], chp, N * lh * lw, z(i, "bsum"), z(i, "bcnt"))))
                calls.append(("conv", self._conv_desc(dl, 0, Wt["wt"], gsrc, op.src.c_off, accumulate=True),
                              dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=True)))
                bwd_rev.append(calls)
                continue
            if op.kind == "pred":
                src, gsrc = view(op.src)
                which, lvl = op.head
                out, grad = {"cls": (self.cls, self.grad_cls), "reg": (self.reg, self.grad_reg),
                             "reg_dist": (getattr(self, "reg_dist", None), getattr(self, "grad_reg_dist", None))}[which]
                ch = out.shape[2]
                chp = (ch + 15) // 16 * 16
                lh, lw = self.sizes[lvl]
                fwd.append(("conv", self._conv_desc(src, op.src.c_off, Wt["w"], out, bias=Wt["bias"], act=op.act,
                                                    y_strides=(A * ch, lw * ch, ch), y_elem_off=self.offs[lvl] * ch)))
                dl = bf(N, lh, lw, chp)
                calls.append(("hgp", (grad.data_ptr(), self.cls.data_ptr() if which == "cls" else 0, N, A, ch, self.offs[lvl], lh * lw, chp,
                                      dl.data_ptr()), dl))
                calls.append(("wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dl, 0, ch, 1, 1, z(i, "dw"))))
                calls.append(("stats", self._stats_desc([(dl, 0)], chp, N * lh * lw, z(i, "bsum"), z(i, "bcnt"))))
                calls.append(("conv", self._conv_desc(dl, 0, Wt["wt"], gsrc, op.src.c_off, accumulate=True),
                              dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=True)))
                bwd_rev.append(calls)
                continue
            if op.kind == "convT":
                src, gsrc = view(op.src)
                dst, gdst = view(op.dst)
                _, dh, dw, dct = dst.shape
                _, sh, sw, _ = src.shape
                for q in range(4):
                    dy, dx = q // 2, q % 2
                    fwd.append(("conv", self._conv_desc(src, op.src.c_off, Wt["w"][q], dst, op.dst.c_off, bias=Wt["bias"],
                                                        y_strides=(dh * dw * dct, 2 * dw * dct, 2 * dct), y_elem_off=(dy * dw + dx) * dct)))
                gd = gdst[..., op.dst.c_off:op.dst.c_off + op.cout]
                calls.append(("dbg", (i, gd)))
                # bias gradient = column sums of the whole upsampled gradient slice
                calls.append(("stats", self._stats_desc([(gdst, op.dst.c_off)], op.cout, N * dh * dw, z(i, "bsum"), z(i, "bcnt"))))
                need = N * sh * sw * op.cout
                if dq_pool is None or dq_pool[0].numel() < need:
                    dq_pool = [torch.zeros(need, dtype=torch.bfloat16, device=dev) for _ in range(4)]
                for q in range(4):
                    dy, dx = q // 2, q % 2
                    dq = dq_pool[q][:need].view(N, sh, sw, op.cout)
                    calls.append(("copy", (dq, gd[:, dy::2, dx::2, :])))               # gradient of quadrant q, dense
                    calls.append(("wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dq, 0, op.cout, 1, 1, z(i, "dw") + 4 * q * op.cout * op.cin)))
                    calls.append(("conv", self._conv_desc(dq, 0, Wt["wt"][q], gsrc, op.src.c_off, accumulate=True),
                                  dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=True)))
                bwd_rev.append(calls)
                continue
            # ---- BN-ed blocks: stem / rep / cba ----
            dst, gdst = view(op.dst)
            n, ho, wo, dct = dst.shape
            count = n * ho * wo
            br = Wt["br"]
            nb = len(br)
            st = self.stat_out[i]
            xs = []
            for b, ent in enumerate(br):
                k = ent["k"]
                if k == 0:
                    src, _ = view(op.src)
                    xs.append((src, op.src.c_off))
                    self.ctx[i]["branches"][b]["x"] = src
                    continue
                raw = bf(n, ho, wo, op.cout)
                self.ctx[i]["branches"][b]["x"] = raw
                if op.kind == "stem":
                    fwd.append(("stem", ops.stem_desc(self.x_static.data_ptr(), N, H, W, in_dtype == torch.uint8, ent["w"].data_ptr(), 0,
                                                      op.cout, None, raw.data_ptr(), fp32_math=1)))
                else:
                    src, _ = view(op.src)
                    fwd.append(("conv", self._conv_desc(src, op.src.c_off, ent["w"], raw, stride=op.s)))
                xs.append((raw, 0))
            qa = op.layout == "qa"
            if qa:
                # BN_d statistics of u, then t = BN_d(u) + v [+ x [+ avg3x3 x]] with the post-sum bn's statistics in one launch;
                # from here on the block is a one-branch BatchNorm over t
                u, v = xs[0][0], xs[1][0]
                fwd.append(("stats", self._stats_desc([xs[0]], op.cout, count, z(i, "fsum"), z(i, "fcnt"), [(op.name + ".rbr_dense.bn", st[0])])))
                tq = bf(n, ho, wo, op.cout)
                q = self._qa_desc(op, u, v, st, tq, z(i, "qsum"), z(i, "qcnt"))
                if op.identity:
                    src, _ = view(op.src)
                    q.x, q.x_pitch = src.data_ptr() + op.src.c_off * 2, src.shape[3]
                fwd.append(("qa", q))
                self.ctx[i].update(u=u, v=v, t=tq, stats_d=st[0], stats_p=st[1])
                xs, st = [(tq, 0)], st[1:]
            else:
                fin = [(ent["prefix"] + (".bn" if ent["k"] else ""), st[b]) for b, ent in enumerate(br)]
                fwd.append(("stats", self._stats_desc(xs, op.cout, count, z(i, "fsum"), z(i, "fcnt"), fin, op.w_row0)))
            d = BnDesc()
            d.nb, d.act, d.C, d.pixels = len(xs), ACT_CODES[op.act], op.cout, count
            dcs = []
            for b, (t, off) in enumerate(xs):
                d.x[b], d.x_pitch[b] = t.data_ptr() + off * 2, t.shape[3]
                d.mean[b], d.invstd[b] = st[b, 0].data_ptr(), st[b, 1].data_ptr()
                d.scale[b], d.shift[b] = st[b, 2].data_ptr(), st[b, 3].data_ptr()
                d.s2[b] = z(i, "s2") + 8 * b * op.cout
                if br[b]["k"] == 0:      # identity branch: its input gradient goes straight into g(src)
                    _, gsrc = view(op.src)
                    d.dx[b], d.dx_pitch[b], d.accumulate[b] = gsrc.data_ptr() + op.src.c_off * 2, gsrc.shape[3], 1
                    dcs.append(None)
                else:
                    dc = dc_pool[2 * (bn_ops & 1) + len([t for t in dcs if t is not None])][:count * op.cout].view(n, ho, wo, op.cout)
                    d.dx[b], d.dx_pitch[b], d.accumulate[b] = dc.data_ptr(), op.cout, 0
                    dcs.append(dc)
            d.y, d.y_pitch = dst.data_ptr() + op.dst.c_off * 2, dct
            d.dy, d.dy_pitch = gdst.data_ptr() + op.dst.c_off * 2, dct
            d.s1 = z(i, "s1")
            d.work, d.counter, d.coef, d.zeroed = z(i, "work"), z(i, "bcnt"), self.coef_out[i].data_ptr(), 1
            if op.res is not None:
                rbuf, grbuf = view(op.res)
                d.res, d.res_pitch, d.res_alpha = rbuf.data_ptr() + op.res.c_off * 2, rbuf.shape[3], 1.0
                if op.alpha in self.params:
                    d.res_alpha_dev = fl.ptr(op.alpha)
                d.dres, d.dres_pitch, d.dalpha = grbuf.data_ptr() + op.res.c_off * 2, grbuf.shape[3], z(i, "dalpha")
            fwd.append(("apply", d))
            calls.append(("dbg", (i, gdst[..., op.dst.c_off:op.dst.c_off + op.cout])))
            wr = []      # gradient slices this launch writes besides the scratch tensors
            for b in range(nb):
                if br[b]["k"] == 0:
                    wr.append(dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=True, what=("dx", b)))
            if op.res is not None:
                wr.append(dict(buf=op.res.buf, off=op.res.c_off, n=op.cout, full=True, what=("dres", 0)))
            par = bn_ops & 1
            bn_ops += 1
            calls.append(("bn_bwd", d, wr, par))
            if qa:
                # dt (d.dx[0]) -> BN_d backward (no activation) -> du; dt also feeds the 1x1 branch and the parameter-free identity /
                # average-pool branches (yv6_qa_bwd into g(x)); the conv branches below then read dcs = [du, dt]
                dt = dcs[0]
                du = dc_pool[2 * par + 1][:count * op.cout].view(n, ho, wo, op.cout)
                sd_ = self.stat_out[i][0]
                d2 = BnDesc()
                d2.nb, d2.act, d2.C, d2.pixels = 1, ACT_CODES[None], op.cout, count
                d2.x[0], d2.x_pitch[0] = u.data_ptr(), op.cout
                d2.mean[0], d2.invstd[0], d2.scale[0], d2.shift[0] = (sd_[r].data_ptr() for r in range(4))
                d2.s2[0], d2.s1 = z(i, "s2d"), z(i, "s1d")
                d2.dx[0], d2.dx_pitch[0], d2.accumulate[0] = du.data_ptr(), op.cout, 0
                d2.dy, d2.dy_pitch = dt.data_ptr(), op.cout
                d2.work, d2.counter, d2.coef, d2.zeroed = z(i, "workd"), z(i, "bcntd"), self.coef_out[i][1].data_ptr(), 1
                calls.append(("bn_bwd", d2, [], par))
                if op.identity:
                    _, gsrc = view(op.src)
                    qb = self._qa_desc(op, u, v, self.stat_out[i], tq, 0, 0)
                    qb.dt, qb.dt_pitch = dt.data_ptr(), op.cout
                    qb.dx, qb.dx_pitch = gsrc.data_ptr() + op.src.c_off * 2, gsrc.shape[3]
                    calls.append(("qa_bwd", qb, dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=True)))
                dcs = [du, dt]
            if op.kind == "stem":       # im2col once, then one tensor-core wgrad GEMM per branch
                patches, patches_lo = bf(n, ho, wo, 32), bf(n, ho, wo, 32)     # image = hi + lo (bf16 planes)
                self._stem_patches = (patches, patches_lo)
                calls.append(("im2col", (self.x_static.data_ptr(), x_dt, 1.0 / 255.0, N, H, W, patches.data_ptr(), patches_lo.data_ptr())))
                for b in range(nb):
                    for pl in (patches, patches_lo):
                        calls.append(("wgrad", self._wgrad_desc(pl, 0, 32, dcs[b], 0, op.cout, 1, 1, z(i, "dw", b)), par))
            else:
                src, gsrc = view(op.src)
                for b, ent in enumerate(br):
                    if ent["k"] == 0:
                        continue
                    calls.append(("wgrad", self._wgrad_desc(src, op.src.c_off, op.cin, dcs[b], 0, op.cout, ent["k"], op.s, z(i, "dw", b)), par))
                    dds = self._dgrad_descs(dcs[b], ent, ent["k"], op.s, gsrc, op.src.c_off)
                    # a stride-2 3x3 dgrad = four parity convolutions that together cover every pixel; 1x1 stride 2 covers one parity
                    full = op.s == 1 or ent["k"] == 3
                    for gi, dd in enumerate(dds):
                        calls.append(("conv", dd, dict(buf=op.src.buf, off=op.src.c_off, n=op.cin, full=full, group=(i, b), first=gi == 0)))
            bwd_rev.append(calls)
        self.fwd_calls = fwd
        bwd = []
        for i in range(len(g.ops) - 1, -1, -1):
            bwd.extend(bwd_rev[i])
            k = self.bucket_of_op.get(i)
            if k is not None and self.last_op_of_bucket[k] == i:
                bwd.append(("bucket", k))
        self.bwd_calls = bwd
        self._keep = (dc_pool, pool_scr, dq_pool)
        self._resolve_first_writers()

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

        def decide(m):
            seg = cov[m["buf"]][m["off"]:m["off"] + m["n"]]
            if m["full"] and not seg.any():
                assign = True
            else:
                assign = False
                if not seg.all():
                    need_zero.add(m["buf"])
            seg[:] = True
            return assign

        for c in self.bwd_calls:
            kind = c[0]
            if kind == "conv" and len(c) > 2:
                m, d = c[2], c[1]
                if "group" in m:
                    if m["first"]:
                        group_decision[m["group"]] = decide(m)
                    assign = group_decision[m["group"]]
                else:
                    assign = decide(m)
                if assign:          # y = conv(...) instead of y += conv(...): no residual read
                    d.res, d.alpha = 0, 0.0
            elif kind == "bn_bwd":
                d = c[1]
                for m in c[2]:
                    assign = decide(m)
                    if m["what"][0] == "dx":
                        d.accumulate[m["what"][1]] = 0 if assign else 1
                    else:
                        d.dres_assign = 1 if assign else 0
            elif kind == "pool_bwd":
                c[1][11] = 0 if decide(c[2]) else 1
            elif kind == "qa_bwd":
                c[1].accumulate = 0 if decide(c[2]) else 1
        for i, cv in enumerate(cov):        # slices nobody writes are read as zero gradients
            if not cv.all():
                need_zero.add(i)
        self.zero_gbufs = [self.gbufs[i] for i in sorted(need_zero)]

    # ================================================================== execution
    def launch_counts(self):
        """(forward, backward) kernel launches of the current plan, excluding the arena memset and the two repack launches."""
        f = len(self.fwd_calls)
        b = 0
        for c in self.bwd_calls:
            kind = c[0]
            if kind == "bn_bwd" or kind == "pool_bwd":
                b += 2
            elif kind in ("dbg", "bucket"):
                continue
            else:
                b += 1
        return f, b + len(self.grad_tables)

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
        self.flat.iflat.add_(1)                     # BatchNorm.num_batches_tracked
        self.run_forward(sp)
        return self.cls, self.reg

    def run_forward(self, sp):
        lib, h, chk = self.lib, self.h, _lib.check
        for kind, d in self.fwd_calls:
            if kind == "conv":
                chk(lib.yv6_conv_fwd(h, C.byref(d), sp))
            elif kind == "stats":
                chk(lib.yv6_bn_stats_finalize(h, C.byref(d), sp))
            elif kind == "apply":
                chk(lib.yv6_bn_apply_fwd(h, C.byref(d), sp))
            elif kind == "stem":
                chk(lib.yv6_stem_fwd(h, C.byref(d), sp))
            elif kind == "qa":
                chk(lib.yv6_qa_fwd(h, C.byref(d), sp))
            elif kind == "abp":
                self._ab_call(d, False, sp)
            else:
                chk(lib.yv6_sppf_pool(h, C.c_void_p(d[0]), d[1], d[2], d[3], d[4], d[5], d[6], d[7], sp))

    def _ab_call(self, lvl, backward, sp):
        """fuse_ab level `lvl`: natural-order conv outputs -> (cls_ab, reg_ab) rows, or their gradients -> dense bf16 gradients."""
        from .arch import AB_ANCHORS
        st = self._ab[lvl]
        N = self.cls_ab.shape[0]
        lh, lw = self.sizes[lvl]
        nc, A3 = self.g.num_classes, self.cls_ab.shape[1]
        off3 = AB_ANCHORS * self.offs[lvl]
        if not backward:
            _lib.check(self.lib.yv6_head_ab_pack(self.h, _p(st["raw_cls"]), _p(st["raw_reg"]), N, lh * lw, AB_ANCHORS, nc, st["anchors"],
                                                 off3, A3, _p(self.cls_ab), _p(self.reg_ab), sp))
        else:
            _lib.check(self.lib.yv6_head_ab_grad(self.h, _p(self.grad_cls_ab), _p(self.cls_ab), _p(self.grad_reg_ab), _p(st["raw_reg"]), N,
                                                 lh * lw, AB_ANCHORS, nc, st["anchors"], off3, A3, st["dl_cls"].shape[3], st["dl_reg"].shape[3],
                                                 _p(st["dl_cls"]), _p(st["dl_reg"]), sp))

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
        lib, h, chk = self.lib, self.h, _lib.check
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

        def wait_pending(par=-1):
            keep = []
            for ev, q in pending:
                if par == -1 or q == par:
                    main.wait_event(ev)
                else:
                    keep.append((ev, q))
            pending[:] = keep

        for c in calls[first:]:
            kind, d = c[0], c[1]
            if kind == "conv":
                chk(lib.yv6_conv_fwd(h, C.byref(d), sp))
            elif kind == "wgrad":
                if overlap:
                    ev = torch.cuda.Event()
                    ev.record(main)
                    side.wait_event(ev)
                    chk(lib.yv6_conv_wgrad(h, C.byref(d), ssp))
                    done = torch.cuda.Event()
                    done.record(side)
                    pending.append((done, c[2] if len(c) > 2 else None))
                else:
                    chk(lib.yv6_conv_wgrad(h, C.byref(d), sp))
            elif kind == "bn_bwd":
                if overlap:
                    wait_pending(c[3])
                chk(lib.yv6_bn_bwd(h, C.byref(d), sp))
            elif kind == "stats":
                chk(lib.yv6_bn_stats_finalize(h, C.byref(d), sp))
            elif kind == "qa_bwd":
                chk(lib.yv6_qa_bwd(h, C.byref(d), sp))
            elif kind == "copy":
                if overlap:
                    wait_pending()
                d[0].copy_(d[1])
            elif kind == "abg":
                self._ab_call(d, True, sp)
            elif kind == "hgp":
                chk(lib.yv6_head_grad_prep(h, d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], d[8], sp))
            elif kind == "pool_bwd":
                chk(lib.yv6_maxpool5_bwd(h, d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], d[8].data_ptr(), d[9], d[10], d[11], sp))
            elif kind == "im2col":
                chk(lib.yv6_stem_im2col(h, *d, sp))
            elif kind == "bucket":
                if overlap:
                    wait_pending()
                self.grad_tables[d].launch(lib, h, accumulate, sp)
                if self.bucket_hook is not None:
                    self.bucket_hook(d)
            elif kind == "dbg":
                if self.debug:
                    self.dbg[d[0]] = dict(gdst=d[1].clone())
        if overlap:
            wait_pending()      # every call (and every captured graph segment) ends joined

    def bucket_call_index(self):
        """Indices into the backward call list right after each bucket's unpack (segment boundaries for graph capture)."""
        return [j + 1 for j, c in enumerate(self.bwd_calls) if c[0] == "bucket"]


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
        feats = []
        if engine.external_feat_grads:       # neck outputs, NCHW fp32 copies (reference `featmaps`, yolo.py:37-39)
            feats = [engine.bufs[t.buf][..., t.c_off:t.c_off + t.c].permute(0, 3, 1, 2).float().contiguous() for t in engine.g.feat]
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
