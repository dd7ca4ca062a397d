"""Every launch of the inference forward, run alone at the engine's own descriptors and checked per element against float64,
and the multi-lane forward and the captured serving graph checked bit for bit against a serial run of the same records.

Part 1 (test_every_inference_launch_record_matches_float64).  An InferEngine with seeded weights plans one input shape --
among them YOLOv6-S at 640 x 640, batch 32, in both precision modes: the shape bench.py times.  Every launch record of the
plan (stem, convs in all their forms, SPPF pool, depthwise conv, SE, channel shuffle, upsample) and the head decode run once
per distinct descriptor signature (pointers as (tensor kind, offset inside it)) on fresh seeded data:
  * every element of every plan buffer (activations, fused sibling outputs, head tensors, decoded output) first holds a finite
    sentinel, 2^100, in every plane; the launch's declared read spans (InferLaunch.reads) then get seeded random values (bf16,
    or the bf16x3 split of fp32 values in the fp32 mode);
  * after the launch the elements the descriptor writes are compared with float64 of the operation on the values that were in
    memory (packed weights, padded bias and alpha as the descriptor holds them); those elements must lie in the declared write
    spans (a head pred: the anchor rows of its level);
  * the read spans must be unchanged (except an in-place launch's), and every other element of every buffer must still hold
    the sentinel, bit for bit.  A kernel that reads a sentinel through a non-zero weight is off by ~2^100.
The conv launches of the Lite graphs read the 16-aligned channel window around their slice (engine.conv_window), wider than
the declared span; the check requires every weight column outside the span to be zero in every plane (the sentinel there
contributes 0), which is what the InferLaunch docstring allows.

Bars are per element.  R is the same operation on absolute values (|x| * |w| summed, plus |bias|), z the pre-activation:
  fp32 accumulation: slope * 1e-5 R, slope = the activation's largest slope (SiLU 1.1, Hardswish 1.5, sigmoid 0.25, else 1);
  bf16x3 products: the kernel drops the plane pairs (1, 2), (2, 1), (2, 2) (yv6_conv_igemm.cu kPairA / kPairB), < 2^-22 R;
  fp32 epilogue: bias add, activation (ex2 / rcp / expf approximations; the fp32 argument of the exponential is rounded, which
    grows with |z|) and residual add: 2^-22 (4 + |z|) |ref| + 2^-23 |alpha res|;
  SiLU of bf16 outputs goes through tanh.approx (h + h tanh(h), h = z / 2; PTX bounds its relative error by 2^-10.987), an
    absolute error <= 2^-10.987 |z| / 2 -- in the negative tail that is far above 2^-8 |ref|, and below the bf16 resolution
    of z itself;
  bf16 outputs: one round-to-nearest-even, 2^-8 of the value, on top of the terms above; three-plane outputs: the split is
    exact to 2^-24, inside the epilogue term;
  copies (shuffle, upsample), bf16 max-pool, the cls columns of the decode and its plain-ltrb boxes: bit for bit (the decode's
    boxes against an fp32 torch restatement of head_decode_kernel); the fp32-mode pool's planes sum to the fp32 maximum within
    2^-24 of it; DFL distances: 1e-5 of the distance (a sum of non-negative terms), boxes from them plus 2^-22 of the operands.
A wrong tap, a lost tile or a missing residual moves an element by O(|ref|), far above these bars.  The float64 reference runs
on the GPU through torch's float64 convolutions and matmuls (no code shared with this library); the first launch of each
conv form, of the stem, of the depthwise conv and of SE is cross-checked once against a float64 CPU computation on image 0.

Part 2 (test_lanes_and_serving_graph_match_a_serial_run).  The engine's default four-lane eager forward and one step of
pipeline.DetectStream (a captured CUDA graph) against a serial run of the same records (n_lanes = 1), bit for bit, over every
activation buffer, the fused sibling buffers and both head tensors.  The forward's kernels are deterministic: the conv kernel
walks a static tile schedule with no atomics and no split-K, the SE kernel sums in a fixed order in float64, the pool, stem,
depthwise, copy and decode kernels compute each output element in one thread.  A lane that starts before its producer has
finished reads the sentinel left in its input and is off by ~2^100.

Part 3 (test_every_training_forward_launch_matches_float64).  The same per-launch pattern over the training engine's forward
launch records (eng.fwd_calls) for YOLOv6-N / M / L6 (the backward test's set-up), N-QA, N with the fuse_ab head, S at
640, batch 32, and the N / S self-distillation student at the same shape (its reg_preds_dist pred conv writes fp32 rows of
A * 68).  Each distinct descriptor runs once on fresh seeded inputs; the elements it computes first hold the sentinel,
and every other element of the tensors it writes must keep its value bit for bit.  Kinds and references:
  raw branch conv (no bias, no activation, bf16), head / fuse_ab pred (bias, sigmoid, fp32), ConvTranspose quadrant: the
    conv bars above;
  fp32-math stem: fp32 image and weights, bf16 out;
  stats (bn_stats_finalize, after clearing the zero arena as every step does): sums 1e-5 R; mean, invstd, scale, shift and
    the running statistics in the flat parameter buffer through their formulas plus one fp32 rounding (the bars of
    test_bn_stats_finalize_matches_batchnorm2d);
  apply (bn_apply_fwd): act(sum_b scale_b x_b + shift_b) + alpha res, alpha read from the flat parameter buffer: the conv
    bars with R = sum |scale_b x_b| + |shift_b|;
  qa (qa_fwd): t = BN_d(u) + v [+ x + avg3x3(x)] at 1e-5 R plus one bf16 rounding, and the post-sum statistics of the stored
    t as for stats;
  SPPF pool: exact; fuse_ab row repack (head_ab_pack): class scores and box offsets exact, wh = (2 sigmoid(r))^2 anchor
    within 2^-20 of the value."""
import ctypes as C
import itertools
import time

import pytest
import torch
import torch.nn.functional as F

import test_gpu_backward_launches as bwd
from conftest import golden_keys
from oracle import fabricate as fab

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
F32_SUM, BF16_ULP = bwd.F32_SUM, bwd.BF16_ULP
DROPPED = 2.0 ** -22         # bf16x3 plane pairs the conv kernel leaves out, relative to R
EPI32 = 2.0 ** -22           # fp32 epilogue, relative to |ref| per unit of (4 + |z|)
EPS32 = 2.0 ** -23
TANH_APPROX = 2.0 ** -10.987
SENTINEL = 2.0 ** 100
ACT_NONE, ACT_RELU, ACT_SILU, ACT_SIGMOID, ACT_HARDSWISH = 0, 1, 2, 3, 4
SLOPE = {ACT_NONE: 1.0, ACT_RELU: 1.0, ACT_SILU: 1.1, ACT_SIGMOID: 0.25, ACT_HARDSWISH: 1.5}
GOLDEN_KEYS = ("yolov6n", "yolov6s", "yolov6m", "yolov6l6")

# name -> model config, batch, input height, width, precision, uint8 input
CONFIGS = {
    "yolov6s_640_b32_bf16": dict(cfg="yolov6s", N=32, H=640, W=640),
    "yolov6s_640_b32_fp32": dict(cfg="yolov6s", N=32, H=640, W=640, precision="fp32"),
    "yolov6l6_1280_b2": dict(cfg="yolov6l6", N=2, H=1280, W=1280),
    "yolov6n_384x640_b8_u8": dict(cfg="yolov6n", N=8, H=384, W=640, u8=True),
    "yolov6m_640_b2": dict(cfg="yolov6m", N=2, H=640, W=640),
    "yolov6s_mbla_256_b2": dict(cfg="yolov6s_mbla", N=2, H=256, W=256),
    "yolov6lite_s_128_bf16": dict(cfg="yolov6lite_s", N=2, H=128, W=128),
    "yolov6lite_s_128_fp32": dict(cfg="yolov6lite_s", N=2, H=128, W=128, precision="fp32"),
    "yolov6lite_l_192x320_bf16": dict(cfg="yolov6lite_l", N=2, H=192, W=320),
    "yolov6lite_l_192x320_fp32": dict(cfg="yolov6lite_l", N=2, H=192, W=320, precision="fp32"),
}


# ---------------------------------------------------------------------------------------------------------------- float64 references
def act64(z, act):
    if act == ACT_RELU:
        return z.clamp_min(0)
    if act == ACT_SILU:
        return z * torch.sigmoid(z)
    if act == ACT_SIGMOID:
        return torch.sigmoid(z)
    if act == ACT_HARDSWISH:
        return z * (z + 3).clamp(0, 6) / 6
    return z


def conv_ref(x, w, bias, stride, pad, act, res=None, alpha=1.0, groups=1):
    """(ref, R, z) of act(conv(x, w) + bias) (+ alpha * res) in float64, NHWC in and out; w [Cout, kh, kw, Cin / groups];
    R = the same conv on absolute values plus |bias|, z the pre-activation."""
    xs, ws = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    b = bias.double()
    z = F.conv2d(xs, ws, b, stride=stride, padding=pad, groups=groups).permute(0, 2, 3, 1)
    R = F.conv2d(xs.abs(), ws.abs(), b.abs(), stride=stride, padding=pad, groups=groups).permute(0, 2, 3, 1)
    ref = act64(z, act)
    if res is not None:
        ref = ref + alpha * res.double()
    return ref, R, z


def cross_check(form, fn, ref, R):
    """Once per form: the GPU float64 reference `ref` (R: its absolute-value sum) against fn() = the same computation on the
    CPU for image 0."""
    if form in XCHECKED:
        return
    XCHECKED.add(form)
    rc = fn()
    err = float(((ref[:1].cpu() - rc).abs() / (R[:1].cpu() + 1e-300)).max())
    assert err < 1e-12, f"{form}: GPU float64 reference differs from the CPU by {err:.2e} of R"


def out_bar(ref, R, z, act, *, bf16_out, planes3, fast_silu, res=None, alpha=1.0):
    """Per-element bar of one conv-like output (module docstring)."""
    acc = SLOPE[act] * (F32_SUM + (DROPPED if planes3 else 0.0)) * R + EPI32 * (4 + z.abs()) * ref.abs()
    if res is not None:
        acc = acc + EPS32 * (alpha * res.double()).abs()
    if fast_silu:
        acc = acc + TANH_APPROX * 0.5 * z.abs()
    return acc + BF16_ULP * (ref.abs() + acc) if bf16_out else acc


def sentinel_bits(dtype):
    return torch.tensor(SENTINEL, dtype=dtype).view(torch.int16 if dtype == BF16 else torch.int32).item()


def dirty(tensors):
    """Keys of the tensors in which some element does not hold the sentinel, bit for bit."""
    out = []
    for key, t in tensors.items():
        iv = t.view(torch.int16 if t.dtype == BF16 else torch.int32)
        if not bool((iv == sentinel_bits(t.dtype)).all()):
            out.append(key)
    return out


# ---------------------------------------------------------------------------------------------------------------- the plan
def build_engine(name, precision="bf16"):
    from yolov6_b200.engine import InferEngine
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = build_model(name, 80, dev)
    if name in GOLDEN_KEYS:
        m.load_state_dict(fab.fabricate_state_dict(golden_keys(name), seed=0))
    else:
        randomize_(m, seed=0)
    m.eval()
    return m, InferEngine(m.graph, m.state_dict(), dev, precision)


class Ctx:
    """One plan of an engine with every device tensor named: `tensors` {plan key: tensor} are the buffers the launches write
    (("buf", j), ("fused", i), ("head", "cls" | "reg"), ("pred",)); `mem` resolves any descriptor pointer, weights included."""

    def __init__(self, eng, N, H, W, u8=False):
        self.eng, self.N, self.H, self.W, self.P = eng, N, H, W, eng.nsplit
        dtype = torch.uint8 if u8 else F32
        self.plan = plan = eng._plan(N, H, W, dtype)
        self.img = torch.zeros(N, 3, H, W, dtype=dtype, device=eng.device)
        plan.stem.x = self.img.data_ptr()
        self.tensors = {("buf", j): t for j, t in enumerate(plan.bufs)}
        self.tensors.update({("fused", i): t for i, t in plan.fused.items()})
        self.tensors.update({("head", "cls"): plan.heads[0][0], ("head", "reg"): plan.heads[0][1], ("pred",): plan.pred})
        named = [(k[0], t) for k, t in self.tensors.items()] + [("img", self.img)]
        self.wkey = {}
        for i, ent in eng.weights.items():
            for k, v in ent.items():
                if k == "alpha":
                    continue
                for q, t in enumerate(v if isinstance(v, list) else [v]):
                    named.append((k, t))
                    self.wkey[t.data_ptr()] = (k, i, q)
        self.mem = bwd.Mem(named)
        self.key_of = {t.data_ptr(): k for k, t in self.tensors.items()}
        g = eng.g
        self.offs = list(itertools.accumulate(((H // s) * (W // s) for s in g.strides), initial=0))

    def locate(self, ptr):
        """(plan key, element offset inside one plane, channel pitch) of a pointer into a plan buffer."""
        f = self.mem.find(ptr)
        assert f is not None and f[1].data_ptr() in self.key_of, f"pointer {ptr:#x} is in no plan buffer"
        t = f[1]
        e = f[2] // t.element_size()
        plane = t[0].numel() if (self.P == 3 and t.dtype == BF16) else t.numel()
        return self.key_of[t.data_ptr()], e % plane, t.shape[-1]

    def span(self, key, lo, hi):
        if key[0] == "head":
            return self.tensors[key[:2]][:, self.offs[key[2]]:self.offs[key[2] + 1]]
        return self.tensors[key][..., lo:hi]

    def planes(self, ptr, shape, strides, plane_stride, dtype=BF16):
        n = self.P if plane_stride else 1
        return [self.mem.at(ptr + p * plane_stride * torch.empty(0, dtype=dtype).element_size(), dtype, shape, strides)
                for p in range(n)]

    def reset(self, keys=None):
        for k, t in self.tensors.items():
            if keys is None or k in keys:
                t.fill_(SENTINEL)


def val64(views):
    out = views[0].double()
    for v in views[1:]:
        out = out + v.double()
    return out


def nhwc_strides(H, W, pitch):
    return (H * W * pitch, W * pitch, pitch, 1)


def channels_in(ctx, ptr, n, spans, what):
    """Channel mask over [c0, c0 + n) of the pointer's buffer: which of them lie in the (key, lo, hi) spans."""
    key, e, pitch = ctx.locate(ptr)
    c0 = e % pitch
    mask = torch.zeros(n, dtype=torch.bool)
    for k, lo, hi in spans:
        if k == key:
            mask[max(lo - c0, 0):max(min(hi - c0, n), 0)] = True
    assert c0 + n <= pitch, f"{what}: channels [{c0}, {c0 + n}) leave the buffer pitch {pitch}"
    return key, mask


def assert_declared(ctx, ptr, n, spans, what):
    _, mask = channels_in(ctx, ptr, n, spans, what)
    assert bool(mask.all()), f"{what}: channels outside the declared spans {spans}"


# ---------------------------------------------------------------------------------------------------------------- per-kind checks
XCHECKED = set()     # conv forms whose GPU float64 reference was cross-checked on the CPU


def conv_form(r):
    d = r.desc
    if r.head is not None:
        return "pred"
    if "[" in r.conv["name"]:
        return "convT"
    if d.pair_view:
        return "pair_view"
    if r.writes[0][0][0] == "fused":
        return "fused"
    return "residual" if d.res else "plain"


def check_conv(ctx, r, out_views):
    from yolov6_b200._lib import DT_F32, PAD_SAME
    d, P = r.desc, ctx.P
    wk, i, _ = ctx.wkey[d.w]
    if d.pair_view:       # the original 3x3 stride-2 problem on the same memory, with the unpacked weights
        assert wk == "w_pair"
        N, H, W, Cin, xct = d.N, d.H, 2 * d.W, d.Cin // 2, d.x_c_total // 2
        wt = ctx.eng.weights[i]["w"][0]
        w = val64(list(wt) if P == 3 else [wt])
        kh = kw = 3
        stride, pad = (2, 2), (1, 1)
    else:
        N, H, W, Cin, xct, kh, kw = d.N, d.H, d.W, d.Cin, d.x_c_total, d.kh, d.kw
        w_planes = ctx.planes(d.w, (d.Cout, kh, kw, Cin), None, d.w_plane_stride)
        w = val64(w_planes)
        stride = (d.stride, d.stride_w or d.stride)
        pad = (d.pad, d.pad if d.pad_w == PAD_SAME else d.pad_w)
    Ho = (H + 2 * pad[0] - kh) // stride[0] + 1
    Wo = (W + 2 * pad[1] - kw) // stride[1] + 1
    assert d.out_h in (0, Ho) and d.out_w in (0, Wo), f"{r.name}: descriptor output size"
    Cout = d.Cout
    x = val64(ctx.planes(d.x, (N, H, W, Cin), nhwc_strides(H, W, xct), d.x_plane_stride))
    _, inside = channels_in(ctx, d.x, Cin, r.reads[:1], r.name)
    if not bool(inside.all()):        # the Lite 16-aligned window: zero weights outside the slice, in every plane
        out = ~inside.to(w.device)
        assert not d.pair_view
        for wp in w_planes:
            assert not bool((wp[..., out] != 0).any()), f"{r.name}: reads channels outside its span through non-zero weights"
        x[..., out] = 0.0             # sentinel * 0 = 0 in the kernel; kept out of the float64 convolution
    bias = ctx.mem.at(d.bias, F32, (Cout,)) if d.bias else torch.zeros(Cout, dtype=F32, device=x.device)
    res = None
    if d.res:
        assert_declared(ctx, d.res, Cout, r.reads[1:], r.name + " residual")
        res = val64(ctx.planes(d.res, (N, Ho, Wo, Cout), (d.res_img_stride, d.res_h_stride, d.res_w_stride, 1), d.res_plane_stride))
    y_f32 = d.y_dtype == DT_F32
    ydt = F32 if y_f32 else BF16
    yv = ctx.planes(d.y, (N, Ho, Wo, Cout), (d.y_img_stride, d.y_h_stride, d.y_w_stride, 1), d.y_plane_stride, ydt)
    key, e, pitch = ctx.locate(d.y)
    if r.head is not None:            # fp32 head rows [offs[lvl], offs[lvl + 1]) of the [N, A, ch] tensor
        (wkey, _, _), = r.writes
        lvl = wkey[2]
        assert key == ("head", r.head) and e == ctx.offs[lvl] * pitch and Ho * Wo == ctx.offs[lvl + 1] - ctx.offs[lvl]
        assert (d.y_img_stride, d.y_w_stride) == (ctx.offs[-1] * pitch, pitch) and Cout == pitch
    else:
        assert_declared(ctx, d.y, Cout, r.writes, r.name + " output")
    ref, R, z = conv_ref(x, w, bias[:Cout], stride, pad, d.act, res, d.alpha)
    cross_check(conv_form(r), lambda: conv_ref(x[:1].cpu(), w.cpu(), bias[:Cout].cpu(), stride, pad, d.act,
                                               None if res is None else res[:1].cpu(), d.alpha)[0], ref, R)
    bar = out_bar(ref, R, z, d.act, bf16_out=not y_f32, planes3=P == 3, fast_silu=d.act == ACT_SILU and not y_f32 and P == 1,
                  res=res, alpha=d.alpha)
    out_views += yv
    return bwd.ratio(val64(yv), ref, bar)


def check_stem(ctx, r, out_views):
    from yolov6_b200._lib import DT_U8
    d, P = r.desc, ctx.P
    N, H, W, Cout = d.N, d.H, d.W, d.Cout
    xf = ctx.img.float() * torch.tensor(d.in_scale, dtype=F32, device=ctx.img.device) if d.x_dtype == DT_U8 else ctx.img.clone()
    w = ctx.mem.at(d.w, F32, (3, 3, 3, Cout)).permute(3, 0, 1, 2)          # [Cout, r, s, c]
    b = ctx.mem.at(d.bias, F32, (Cout,)) if d.bias else torch.zeros(Cout, dtype=F32, device=w.device)
    bf16_math = P == 1 and not d.fp32_math
    if bf16_math:                     # tensor-core stem: bf16 image and weights, fp32 accumulation
        xf, w = xf.to(BF16), w.to(BF16)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    assert_declared(ctx, d.y, Cout, r.writes, r.name + " output")
    yv = ctx.planes(d.y, (N, Ho, Wo, Cout), nhwc_strides(Ho, Wo, Cout), d.y_plane_stride)
    ref, R, z = conv_ref(xf.permute(0, 2, 3, 1), w, b, 2, 1, d.act)
    cross_check("stem", lambda: conv_ref(xf[:1].cpu().permute(0, 2, 3, 1), w.cpu(), b.cpu(), 2, 1, d.act)[0], ref, R)
    bar = out_bar(ref, R, z, d.act, bf16_out=P == 1, planes3=False, fast_silu=False)
    out_views += yv
    return bwd.ratio(val64(yv), ref, bar)


def check_pool(ctx, r, out_views):
    y, N, H, W, Cc, ct, nsplit, plane = r.args
    views = ctx.planes(y, (N, H, W, ct), nhwc_strides(H, W, ct), plane)
    key, _, _ = ctx.locate(y)
    assert r.reads == [(key, 0, Cc)] and r.writes == [(key, Cc, 4 * Cc)]
    if nsplit == 3:                   # the kernel reads the fp32 sum of the planes in this order
        x = (views[0][..., :Cc].float() + views[1][..., :Cc].float()) + views[2][..., :Cc].float()
    else:
        x = views[0][..., :Cc].float()
    ys, t = [], x.permute(0, 3, 1, 2)
    for _ in range(3):
        t = F.max_pool2d(t, 5, 1, 2)
        ys.append(t.permute(0, 2, 3, 1))
    ref = torch.cat(ys, -1)
    out = [v[..., Cc:4 * Cc] for v in views]
    out_views += out
    if nsplit == 3:
        return bwd.ratio(val64(out), ref.double(), 2.0 ** -24 * ref.double().abs())
    assert bwd.bits_equal(out[0], ref.to(BF16)), f"{r.name}: bf16 max-pool is not exact"
    return 0.0


def check_dw(ctx, r, out_views):
    d, P = r.desc, ctx.P
    N, H, W, Cc, k, s = d.N, d.H, d.W, d.C, d.k, d.stride
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    assert_declared(ctx, d.x, Cc, r.reads, r.name + " input")
    assert_declared(ctx, d.y, Cc, r.writes, r.name + " output")
    if P == 3:                        # fp32 sum of the planes, as the kernel stages it
        xv = ctx.planes(d.x, (N, H, W, Cc), nhwc_strides(H, W, d.x_c_total), d.x_plane_stride)
        x = (xv[0].float() + xv[1].float()) + xv[2].float()
    else:
        x = ctx.planes(d.x, (N, H, W, Cc), nhwc_strides(H, W, d.x_c_total), 0)[0]
    w = ctx.mem.at(d.w, F32, (k * k, Cc)).t().reshape(Cc, k, k, 1)
    b = ctx.mem.at(d.bias, F32, (Cc,)) if d.bias else torch.zeros(Cc, dtype=F32, device=w.device)
    yv = ctx.planes(d.y, (N, Ho, Wo, Cc), nhwc_strides(Ho, Wo, d.y_c_total), d.y_plane_stride)
    ref, R, z = conv_ref(x, w, b, s, k // 2, d.act, groups=Cc)
    cross_check("dw", lambda: conv_ref(x[:1].cpu(), w.cpu(), b.cpu(), s, k // 2, d.act, groups=Cc)[0], ref, R)
    bar = out_bar(ref, R, z, d.act, bf16_out=P == 1, planes3=False, fast_silu=False)
    out_views += yv
    return bwd.ratio(val64(yv), ref, bar)


def check_se(ctx, r, out_views, x_before):
    d, P = r.desc, ctx.P
    N, HW, Cc, Cr = d.N, d.HW, d.C, d.Cr
    assert_declared(ctx, d.x, Cc, r.reads, r.name + " input")
    assert_declared(ctx, d.x, Cc, r.writes, r.name + " output")
    x = x_before.double().reshape(N, HW, Cc)
    w1, b1 = ctx.mem.at(d.w1, F32, (Cr, Cc)).double(), ctx.mem.at(d.b1, F32, (Cr,)).double()
    w2, b2 = ctx.mem.at(d.w2, F32, (Cc, Cr)).double(), ctx.mem.at(d.b2, F32, (Cc,)).double()
    def se64(x, w1, b1, w2, b2):
        hid = (x.mean(1) @ w1.t() + b1).clamp_min(0)
        return x * ((hid @ w2.t() + b2 + 3).clamp(0, 6) / 6)[:, None, :], hid

    m = x.mean(1)
    ref, hid = se64(x, w1, b1, w2, b2)
    cross_check("se", lambda: se64(*(t.cpu() for t in (x[:1], w1, b1, w2, b2)))[0], ref, x.abs())
    # fp32 FC sums (1e-5 of the sums of absolute terms) through the hard sigmoid (slope 1/6), then one fp32 product
    eh = F32_SUM * (m.abs() @ w1.abs().t() + b1.abs()) + EPS32 * m.abs().sum(1, keepdim=True)
    ez = F32_SUM * (hid @ w2.abs().t() + b2.abs()) + eh @ w2.abs().t()
    acc = x.abs() * (ez / 6)[:, None, :] + 2 * EPS32 * ref.abs()
    bar = acc + BF16_ULP * (ref.abs() + acc) if P == 1 else acc
    yv = ctx.planes(d.x, (N, HW, Cc), (HW * d.c_total, d.c_total, 1), d.plane_stride)
    out_views += yv
    return bwd.ratio(val64(yv), ref, bar)


def check_shuffle(ctx, r, out_views):
    a, ap, apl, b, bp, bpl, pix, Cc, y, yp, ypl, nsplit = r.args
    assert_declared(ctx, a, Cc, r.reads[:1], r.name + " a")
    assert_declared(ctx, b, Cc, r.reads[1:], r.name + " b")
    assert_declared(ctx, y, 2 * Cc, r.writes, r.name + " output")
    av, bv = ctx.planes(a, (pix, Cc), (ap, 1), apl), ctx.planes(b, (pix, Cc), (bp, 1), bpl)
    yv = ctx.planes(y, (pix, 2 * Cc), (yp, 1), ypl)
    for p in range(len(yv)):
        assert bwd.bits_equal(yv[p][:, 0::2], av[p]) and bwd.bits_equal(yv[p][:, 1::2], bv[p]), f"{r.name}: plane {p}"
    out_views += yv
    return 0.0


def check_up(ctx, r, out_views):
    x, xp, xpl, N, H, W, Cc, y, yp, ypl, nsplit = r.args
    assert_declared(ctx, x, Cc, r.reads, r.name + " input")
    assert_declared(ctx, y, Cc, r.writes, r.name + " output")
    xv = ctx.planes(x, (N, H, W, Cc), nhwc_strides(H, W, xp), xpl)
    yv = ctx.planes(y, (N, 2 * H, 2 * W, Cc), nhwc_strides(2 * H, 2 * W, yp), ypl)
    for p in range(len(yv)):
        assert bwd.bits_equal(yv[p], xv[p].repeat_interleave(2, 1).repeat_interleave(2, 2)), f"{r.name}: plane {p}"
    out_views += yv
    return 0.0


def decode_ref(ctx, cls, reg):
    """pred [N, A, 5 + nc] of head_decode_kernel restated in torch: plain ltrb boxes with the kernel's fp32 operation order (each
    op rounded once), DFL distances in float64.  Returns (pred, per-element bar or None when it must be bit-exact)."""
    g = ctx.eng.g
    N, A, Rr = reg.shape
    dev = reg.device
    lvl_ax, lvl_ay, lvl_s = [], [], []
    for lvl, s in enumerate(g.strides):
        h, w = ctx.H // s, ctx.W // s
        local = torch.arange(h * w, device=dev)
        lvl_ax.append((local % w).float() + 0.5)
        lvl_ay.append((local // w).float() + 0.5)
        lvl_s.append(torch.full((h * w,), float(s), device=dev))
    ax, ay, st = torch.cat(lvl_ax), torch.cat(lvl_ay), torch.cat(lvl_s)
    pred = torch.empty(N, A, 5 + cls.shape[2], dtype=F32, device=dev)
    pred[..., 5:] = cls
    pred[..., 4] = 1.0
    if Rr == 4:
        dl, dt, dr, db = reg.unbind(-1)
        x1, y1, x2, y2 = ax - dl, ay - dt, ax + dr, ay + db
        pred[..., 0] = ((x1 + x2) / 2) * st
        pred[..., 1] = ((y1 + y2) / 2) * st
        pred[..., 2] = (x2 - x1) * st
        pred[..., 3] = (y2 - y1) * st
        return pred, None
    nb = Rr // 4
    p = torch.softmax(reg.double().view(N, A, 4, nb), -1)
    dist = (p * torch.arange(nb, device=dev, dtype=F64)).sum(-1)
    dl, dt, dr, db = dist.unbind(-1)
    ax, ay, st = ax.double(), ay.double(), st.double()
    out = pred.double()
    out[..., 0], out[..., 1] = (2 * ax - dl + dr) / 2 * st, (2 * ay - dt + db) / 2 * st
    out[..., 2], out[..., 3] = (dl + dr) * st, (dt + db) * st
    bar = torch.zeros_like(out)
    eb = F32_SUM * dist                                    # a sum of non-negative terms: R = the distance
    bar[..., 0] = st * (eb[..., 0] + eb[..., 2]) + 2.0 ** -22 * st * (ax + dl + dr)
    bar[..., 2] = bar[..., 0]
    bar[..., 1] = st * (eb[..., 1] + eb[..., 3]) + 2.0 ** -22 * st * (ay + dt + db)
    bar[..., 3] = bar[..., 1]
    return out, bar


def check_decode(ctx, gen):
    from yolov6_b200 import _lib
    plan, eng = ctx.plan, ctx.eng
    cls, reg = plan.heads[0]
    ctx.reset()
    cls.copy_(torch.rand(cls.shape, generator=gen, device=cls.device))
    if reg.shape[2] == 4:
        reg.copy_(torch.rand(reg.shape, generator=gen, device=reg.device) * 20)
    else:
        reg.copy_(torch.randn(reg.shape, generator=gen, device=reg.device) * 3)
    c0, r0 = cls.clone(), reg.clone()
    plan.decode.run(eng.lib, eng.handle, _lib.stream_ptr())
    torch.cuda.synchronize()
    ref, bar = decode_ref(ctx, c0, r0)
    got = plan.pred
    assert torch.equal(got[..., 4:].contiguous().view(torch.int32), ref[..., 4:].float().contiguous().view(torch.int32)), \
        "decode: objectness / class columns"
    if bar is None:
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), "decode: boxes differ from the fp32 restatement"
        worst = 0.0
    else:
        worst = bwd.ratio(got[..., :4], ref[..., :4], bar[..., :4])
    assert torch.equal(cls, c0) and torch.equal(reg, r0), "decode wrote into its inputs"
    cls.fill_(SENTINEL), reg.fill_(SENTINEL), got.fill_(SENTINEL)
    assert not dirty(ctx.tensors), "decode wrote outside its output"
    return worst, "dfl" if bar is not None else "ltrb"


def launch_signature(ctx, r):
    if r.desc is not None:
        return (r.kind,) + bwd.signature(r.desc, ctx.mem)
    out = [r.kind]
    for a in r.args:
        f = ctx.mem.find(a) if isinstance(a, int) and a > 1 << 20 else None
        out.append(a if f is None else (f[0], f[2]))
    return tuple(out)


def plan_mode(d):
    from yolov6_b200 import ops
    from yolov6_b200._lib import DT_F32
    p = ops.plan_of(d)
    return dict(halo=p["halo"], resident=p["a_res"] % 10 if p["halo"] else None, cta_pair=p["a_res"] // 10 % 10,
                pair_view=d.pair_view, f32_out=d.y_dtype == DT_F32)


def fill_reads(ctx, r, gen):
    from yolov6_b200.ops import split3
    for key, lo, hi in r.reads:
        v = ctx.span(key, lo, hi)
        if ctx.P == 3 and v.dtype == BF16:
            v.copy_(split3(torch.randn(v.shape[1:], generator=gen, device=v.device)))
        else:
            v.copy_(torch.randn(v.shape, generator=gen, device=v.device).to(v.dtype))


def check_launch(ctx, r, gen):
    """Run one launch record alone on sentinel-filled buffers with random read spans; returns its worst error / bar ratio."""
    from yolov6_b200 import _lib
    from yolov6_b200._lib import DT_U8
    eng = ctx.eng
    ctx.reset()
    fill_reads(ctx, r, gen)
    written = {(k, lo, hi) for k, lo, hi in r.writes}
    snap = [(k, lo, hi, ctx.span(k, lo, hi).clone()) for k, lo, hi in r.reads if (k, lo, hi) not in written]
    x_before = val64([ctx.span(*r.reads[0])[p] for p in range(3)]) if (r.kind == "se" and ctx.P == 3) else (
        ctx.span(*r.reads[0]).double() if r.kind == "se" else None)
    out_views = []
    if r.kind == "stem":              # the image is the stem's input, outside the plan buffers
        assert r.desc.x == ctx.img.data_ptr()
        if r.desc.x_dtype == DT_U8:
            ctx.img.copy_(torch.randint(0, 256, ctx.img.shape, generator=gen, device=ctx.img.device, dtype=torch.uint8))
        else:
            ctx.img.copy_(torch.rand(ctx.img.shape, generator=gen, device=ctx.img.device))
    r.run(eng.lib, eng.handle, _lib.stream_ptr())
    torch.cuda.synchronize()
    ratio = {"stem": lambda: check_stem(ctx, r, out_views), "conv": lambda: check_conv(ctx, r, out_views),
             "pool": lambda: check_pool(ctx, r, out_views), "dw": lambda: check_dw(ctx, r, out_views),
             "se": lambda: check_se(ctx, r, out_views, x_before), "shuffle": lambda: check_shuffle(ctx, r, out_views),
             "up": lambda: check_up(ctx, r, out_views)}[r.kind]()
    settle(ctx.tensors, out_views, [ctx.span(k, lo, hi) for k, lo, hi in r.reads], [(ctx.span(k, lo, hi), b) for k, lo, hi, b in snap],
           f"{r.kind} {r.name}")
    return ratio


def settle(tensors, out_views, read_views, unchanged, what):
    """After a launch whose outputs were compared: the inputs it must not write still hold what they held (unchanged: [(view,
    copy from before)]); then the compared output elements and the read spans go back to the sentinel, and every tensor must
    hold the sentinel everywhere -- an element the launch wrote outside what its descriptor computes is left over."""
    for view, before in unchanged:
        iv = torch.int16 if before.dtype == BF16 else torch.int32
        assert torch.equal(view.view(iv), before.view(iv)), f"{what}: changed one of its inputs"
    for v in list(out_views) + list(read_views):
        v.fill_(SENTINEL)
    bad = dirty(tensors)
    assert not bad, f"{what}: wrote outside the elements its descriptor computes: " + "; ".join(stray(tensors[k], k) for k in bad)


def stray(t, key):
    """Where a tensor holds something other than the sentinel: channels, element count, a few values."""
    iv = t.view(torch.int16 if t.dtype == BF16 else torch.int32)
    m = iv != sentinel_bits(t.dtype)
    ch = m.reshape(-1, t.shape[-1]).any(0).nonzero().flatten().tolist()
    return f"{key} {tuple(t.shape)}: {int(m.sum())} elements in channels {ch}, values {t[m][:4].float().tolist()}"


KINDS = ("stem", "conv", "pool", "dw", "se", "shuffle", "up", "decode")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_inference_launch_record_matches_float64(config):
    from yolov6_b200 import _lib
    c = CONFIGS[config]
    t0 = time.time()
    m, eng = build_engine(c["cfg"], c.get("precision", "bf16"))
    ctx = Ctx(eng, c["N"], c["H"], c["W"], c.get("u8", False))
    gen = torch.Generator(device="cuda").manual_seed(20261016)
    worst = {k: 0.0 for k in KINDS}
    seen = {k: set() for k in KINDS}
    total = {k: 0 for k in KINDS}
    forms, modes = {}, set()
    for r in ctx.plan.launches:
        total[r.kind] += 1
        sig = launch_signature(ctx, r)
        if sig in seen[r.kind]:
            continue
        seen[r.kind].add(sig)
        ratio = check_launch(ctx, r, gen)
        assert ratio <= 1.0, f"{config}: {r.kind} {r.name}: error {ratio:.3f} x the bar"
        worst[r.kind] = max(worst[r.kind], ratio)
        if r.kind == "conv":
            f = conv_form(r)
            forms[f] = max(forms.get(f, 0.0), ratio)
            pm = plan_mode(r.desc)
            modes.add(tuple(sorted(pm.items())))
    ratio, how = check_decode(ctx, gen)
    worst["decode"], total["decode"] = ratio, 1
    seen["decode"].add(how)
    for k in ("stem", "conv", "decode"):
        assert seen[k], f"no {k} launch checked"
    print(f"\n{config}: distinct launches checked (of all in the plan): "
          + ", ".join(f"{k} {len(seen[k])}/{total[k]}" for k in KINDS if total[k]))
    print(f"{config}: worst error / bar: " + ", ".join(f"{k} {worst[k]:.3f}" for k in KINDS if total[k])
          + f" (decode: {how}); conv by form: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(forms.items())))
    summary = {}
    for md in modes:
        for k, v in md:
            summary.setdefault(k, set()).add(v)
    print(f"{config}: conv plan modes checked: " + ", ".join(f"{k} {sorted(v, key=str)}" for k, v in sorted(summary.items()))
          + f"; {time.time() - t0:.1f} s")
    del ctx, eng, m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- the schedule
SCHEDULE_CONFIGS = {"yolov6s_640_b32": dict(cfg="yolov6s", N=32, H=640, W=640),
                    "yolov6lite_l_192x320": dict(cfg="yolov6lite_l", N=2, H=192, W=320)}


@pytest.mark.parametrize("config", list(SCHEDULE_CONFIGS))
def test_lanes_and_serving_graph_match_a_serial_run(config):
    from yolov6_b200.pipeline import DetectStream
    c = SCHEDULE_CONFIGS[config]
    N, H, W = c["N"], c["H"], c["W"]
    m, eng = build_engine(c["cfg"])
    eng.n_lanes = 4
    ctx = Ctx(eng, N, H, W)
    assert max(ctx.plan.lane) > 0, "the schedule puts every launch on one lane"
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.rand(N, 3, H, W, generator=gen, device="cuda")
    net = {k: t for k, t in ctx.tensors.items() if k != ("pred",)}

    def run(lanes):
        eng.n_lanes = lanes
        ctx.reset()
        eng.forward(x)
        torch.cuda.synchronize()

    run(1)
    want = {k: t.clone() for k, t in ctx.tensors.items()}
    assert not any(bool((t.float().abs() >= SENTINEL).any()) for k, t in want.items() if k[0] != "buf"), "serial run left a sentinel"

    def compare(what, keys):
        diff = [k for k in keys if not torch.equal(ctx.tensors[k].view(torch.int16 if ctx.tensors[k].dtype == BF16 else torch.int32),
                                                   want[k].view(torch.int16 if want[k].dtype == BF16 else torch.int32))]
        assert not diff, f"{config}: {what} differs from the serial run in {diff}"

    run(4)
    compare("the four-lane forward", list(ctx.tensors))
    ds = DetectStream(m, N, H, W, host_input=False, engine=eng)      # warms both head sets up, captures the step graphs
    assert eng._plan(N, H, W, F32) is ctx.plan
    ctx.reset(set(net))                    # head set 1 keeps its scores: the step's NMS branch reads it
    ds.submit(x)
    torch.cuda.synchronize()
    compare("the captured serving step (head set 0)", list(net))
    print(f"\n{config}: {len(ctx.plan.launches)} launches on {max(ctx.plan.lane) + 1} lanes, {len(ctx.plan.events)} events: "
          f"the lanes and the captured step match the serial run bit for bit ({len(net)} tensors)")
    del ds, ctx, eng, m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- training forward
# name -> model config, image size, batch, fuse_ab.  N / M / L6 are the backward test's set-up.
TRAIN_CONFIGS = {
    "yolov6n": ("yolov6n", 128, 2, False), "yolov6m": ("yolov6m", 96, 2, False), "yolov6l6": ("yolov6l6", 128, 2, False),
    "yolov6n_qa": ("yolov6n_qa", 96, 2, False), "yolov6n_fuse_ab": ("yolov6n", 128, 2, True),
    "yolov6s_640_b32": ("yolov6s", 640, 32, False),
    # the N / S self-distillation student: a third pred conv per level (reg_preds_dist), fp32 rows of A * 68
    "yolov6s_640_b32_distill_ns": ("yolov6s", 640, 32, False, True),
}
TRAIN_KINDS = ("stem", "conv", "stats", "apply", "qa", "pool", "abp")


def train_engine(cfg, size, batch, fuse_ab, distill_ns=False):
    """The training engine of a model with seeded weights, planned for [batch, 3, size, size] fp32 images (as the backward test)."""
    dev = torch.device("cuda:0")
    m = bwd.seeded_model(cfg, dev, fuse_ab=fuse_ab, distill_ns=distill_ns)
    m.train()
    eng = m.train_engine()
    with torch.no_grad():
        eng.forward(fab.synthetic_images(batch, size, size, seed=11).to(dev))
    torch.cuda.synchronize()
    mem = bwd.engine_mem(eng)
    extra = [eng.cls_ab, eng.reg_ab] + [t for st in eng._ab.values() for t, _ in st.values()] if fuse_ab else []
    extra += [ctx["t"] for ctx in eng.ctx if ctx and "t" in ctx]

    def tensors(v):                   # every tensor of the packed weights (eng.wts: dicts and lists of them)
        if torch.is_tensor(v):
            yield v
        elif isinstance(v, dict):
            for u in v.values():
                yield from tensors(u)
        elif isinstance(v, (list, tuple)):
            for u in v:
                yield from tensors(u)
    for t in tensors(eng.wts):
        assert t.is_contiguous() and t.storage_offset() == 0
        mem.ts.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), "w", t))
    for t in extra:
        mem.ts.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), "out", t))
    return m, eng, mem


def guarded(mem, views, run):
    """The elements a launch computes (views) are set to the sentinel, the launch runs, and every other element of the tensors
    that hold the views must keep its value bit for bit.  Returns copies of the views after the launch."""
    ts = {mem.base(v.data_ptr()).data_ptr(): mem.base(v.data_ptr()) for v in views}
    for v in views:
        v.fill_(SENTINEL)
    before = {k: t.clone() for k, t in ts.items()}
    run()
    torch.cuda.synchronize()
    got = [v.clone() for v in views]
    for v in views:            # put the prior values back into the views, then the whole tensors must equal their copies
        t = mem.base(v.data_ptr())
        v.copy_(before[t.data_ptr()].as_strided(v.shape, v.stride(), v.storage_offset()))
    for k, t in ts.items():
        iv = torch.int16 if t.dtype == BF16 else torch.int32
        assert torch.equal(t.view(iv), before[k].view(iv)), "the launch wrote outside the elements its descriptor computes"
    return got


def fill(t, gen, scale=1.0, shift=0.0):
    t.copy_((torch.randn(t.shape, generator=gen, device=t.device) * scale + shift).to(t.dtype))


def stats_ratio(x, sums, st, gam, bet, rm0, rv0, rm, rv, momentum):
    """bn_stats_finalize's sums, mean / invstd / scale / shift and running statistics of x [P, C] against float64 (the bars of
    test_bn_stats_finalize_matches_batchnorm2d: sums 1e-5 R, the rest through their formulas plus one fp32 rounding)."""
    P = x.shape[0]
    R1, R2 = x.abs().sum(0), (x * x).sum(0)
    worst = max(bwd.ratio(sums[0], x.sum(0), F32_SUM * R1), bwd.ratio(sums[1], R2, F32_SUM * R2))
    if st is None:
        return worst
    mean, var = x.mean(0), x.var(0, unbiased=False)
    inv = 1.0 / torch.sqrt(var + bwd.BN_EPS)
    e_mean, e_var = F32_SUM * R1 / P, F32_SUM * (R2 / P + 2 * mean.abs() * R1 / P)
    e_inv = inv * 0.5 * e_var / (var + bwd.BN_EPS)
    g64, b64 = gam.double(), bet.double()
    sc, rel = g64 * inv, 2.0 ** -22
    st = st.double()
    worst = max(worst, bwd.ratio(st[0], mean, e_mean + rel * mean.abs()), bwd.ratio(st[1], inv, e_inv + rel * inv),
                bwd.ratio(st[2], sc, g64.abs() * e_inv + rel * sc.abs()),
                bwd.ratio(st[3], b64 - mean * sc, mean.abs() * g64.abs() * e_inv + sc.abs() * e_mean + rel * (b64.abs() + (mean * sc).abs())))
    if rm is not None:
        unb = P / (P - 1.0)
        worst = max(worst, bwd.ratio(rm, (1 - momentum) * rm0.double() + momentum * mean,
                                     momentum * e_mean + rel * (rm0.double().abs() + momentum * mean.abs())),
                    bwd.ratio(rv, (1 - momentum) * rv0.double() + momentum * unb * var,
                              momentum * unb * e_var + rel * (rv0.double().abs() + momentum * unb * var)))
    return worst


def tcheck_conv(lib, h, sp, mem, c, gen):
    """A training conv (raw branch: no bias, no activation, bf16 out; head pred / fuse_ab pred: bias and activation, fp32 out;
    ConvTranspose quadrant: bias, bf16) against float64."""
    from yolov6_b200._lib import DT_F32, PAD_SAME
    d = c.desc
    N, H, W, Cin, xct, Cout, kh, kw = d.N, d.H, d.W, d.Cin, d.x_c_total, d.Cout, d.kh, d.kw
    xt = mem.base(d.x)
    fill(xt, gen)
    stride, pad = (d.stride, d.stride_w or d.stride), (d.pad, d.pad if d.pad_w == PAD_SAME else d.pad_w)
    Ho, Wo = (H + 2 * pad[0] - kh) // stride[0] + 1, (W + 2 * pad[1] - kw) // stride[1] + 1
    x = mem.at(d.x, BF16, (N, H, W, Cin), nhwc_strides(H, W, xct)).double()
    w = mem.at(d.w, BF16, (Cout, kh, kw, Cin)).double()
    b = mem.at(d.bias, F32, (Cout,)) if d.bias else torch.zeros(Cout, dtype=F32, device=x.device)
    y_f32 = d.y_dtype == DT_F32
    yv = mem.at(d.y, F32 if y_f32 else BF16, (N, Ho, Wo, Cout), (d.y_img_stride, d.y_h_stride, d.y_w_stride, 1))
    got, = guarded(mem, [yv], lambda: bwd.check(lib.yv6_conv_fwd(h, C.byref(d), sp), lib))
    ref, R, z = conv_ref(x, w, b, stride, pad, d.act)
    return bwd.ratio(got, ref, out_bar(ref, R, z, d.act, bf16_out=not y_f32, planes3=False, fast_silu=d.act == ACT_SILU and not y_f32))


def tcheck_stem(lib, h, sp, mem, eng, c, gen):
    """The fp32-math stem: fp32 image and weights on CUDA cores, no bias or activation, bf16 raw output."""
    d = c.desc
    assert d.fp32_math == 1 and d.x == eng.x_static.data_ptr()
    eng.x_static.copy_(torch.rand(eng.x_static.shape, generator=gen, device=eng.x_static.device))
    N, H, W, Cout = d.N, d.H, d.W, d.Cout
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    w = mem.at(d.w, F32, (3, 3, 3, Cout)).permute(3, 0, 1, 2)
    b = mem.at(d.bias, F32, (Cout,)) if d.bias else torch.zeros(Cout, dtype=F32, device=w.device)
    yv = mem.at(d.y, BF16, (N, Ho, Wo, Cout))
    got, = guarded(mem, [yv], lambda: bwd.check(lib.yv6_stem_fwd(h, C.byref(d), sp), lib))
    ref, R, z = conv_ref(eng.x_static.permute(0, 2, 3, 1), w, b, 2, 1, d.act)
    return bwd.ratio(got, ref, out_bar(ref, R, z, d.act, bf16_out=True, planes3=False, fast_silu=False))


def tcheck_stats(lib, h, sp, mem, eng, c, gen):
    """bn_stats_finalize over fresh branch inputs, from a cleared zero arena (as every step starts), with the running statistics
    in the flat parameter buffer."""
    d = c.desc
    nb, Cc, P = d.nb, d.C, d.pixels
    xs = []
    for b in range(nb):
        fill(mem.base(d.x[b]), gen, 1 + b, 0.5 * b)
        xs.append(mem.at(d.x[b], BF16, (P, Cc), (d.x_pitch[b], 1)).double())
    rm0 = [mem.at(d.running_mean[b], F32, (Cc,)).clone() if d.running_mean[b] else None for b in range(nb)]
    rv0 = [mem.at(d.running_var[b], F32, (Cc,)).clone() if d.running_var[b] else None for b in range(nb)]
    eng.zero_arena.zero_()
    assert d.zeroed
    bwd.check(lib.yv6_bn_stats_finalize(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    sums = mem.at(d.sums, F64, (nb, 2, Cc))
    worst = 0.0
    for b in range(nb):
        st = mem.at(d.stats[b], F32, (4, Cc)) if d.stats[b] else None
        gam = mem.at(d.gamma[b], F32, (Cc,)) if d.stats[b] else None
        bet = mem.at(d.beta[b], F32, (Cc,)) if d.stats[b] else None
        rm = mem.at(d.running_mean[b], F32, (Cc,)) if rm0[b] is not None else None
        rv = mem.at(d.running_var[b], F32, (Cc,)) if rv0[b] is not None else None
        worst = max(worst, stats_ratio(xs[b], sums[b], st, gam, bet, rm0[b], rv0[b], rm, rv, d.momentum))
    return worst


def tcheck_apply(lib, h, sp, mem, c, gen):
    """bn_apply_fwd: act(sum_b scale_b x_b + shift_b) (+ alpha * res, alpha from the flat parameter buffer), bf16 out."""
    d = c.desc
    nb, Cc, P = d.nb, d.C, d.pixels
    z = torch.zeros(P, Cc, dtype=F64, device="cuda")
    R = torch.zeros_like(z)
    for b in range(nb):
        fill(mem.base(d.x[b]), gen)
        sc, sh = mem.at(d.scale[b], F32, (Cc,)), mem.at(d.shift[b], F32, (Cc,))
        sc.copy_(torch.rand(Cc, generator=gen, device="cuda") + 0.5)
        fill(sh, gen, 0.3)
        xb = mem.at(d.x[b], BF16, (P, Cc), (d.x_pitch[b], 1)).double()
        z += xb * sc.double() + sh.double()
        R += (xb * sc.double()).abs() + sh.double().abs()
    res, alpha = None, 1.0
    if d.res:
        fill(mem.base(d.res), gen)
        res = mem.at(d.res, BF16, (P, Cc), (d.res_pitch, 1)).double()
        if d.res_alpha_dev:
            assert mem.find(d.res_alpha_dev)[0] == "param"
            alpha = float(mem.at(d.res_alpha_dev, F32, (1,)).item())
        else:
            alpha = float(d.res_alpha)
    yv = mem.at(d.y, BF16, (P, Cc), (d.y_pitch, 1))
    got, = guarded(mem, [yv], lambda: bwd.check(lib.yv6_bn_apply_fwd(h, C.byref(d), sp), lib))
    ref = act64(z, d.act) + (alpha * res if res is not None else 0)
    return bwd.ratio(got, ref, out_bar(ref, R, z, d.act, bf16_out=True, planes3=False, fast_silu=False, res=res, alpha=alpha))


def tcheck_qa(lib, h, sp, mem, eng, c, gen):
    """qa_fwd: t = BN_d(u) + v [+ x + avg3x3(x)] (bf16), and the post-sum BatchNorm's statistics of the stored t."""
    q = c.desc
    N, H, W, Cc = q.N, q.H, q.W, q.C
    shape = (N, H, W, Cc)
    fill(mem.base(q.u), gen)
    fill(mem.base(q.v), gen)
    sc, sh = mem.at(q.scale_d, F32, (Cc,)), mem.at(q.shift_d, F32, (Cc,))
    sc.copy_(torch.rand(Cc, generator=gen, device="cuda") + 0.5)
    fill(sh, gen, 0.3)
    u = mem.at(q.u, BF16, shape, nhwc_strides(H, W, q.u_pitch)).double()
    v = mem.at(q.v, BF16, shape, nhwc_strides(H, W, q.v_pitch)).double()
    ref = u * sc.double() + sh.double() + v
    R = (u * sc.double()).abs() + sh.double().abs() + v.abs()
    if q.x:
        fill(mem.base(q.x), gen)
        x = mem.at(q.x, BF16, shape, nhwc_strides(H, W, q.x_pitch)).double()
        avg3 = lambda t: F.avg_pool2d(t.permute(0, 3, 1, 2), 3, 1, 1, count_include_pad=True).permute(0, 2, 3, 1)  # noqa: E731
        ref = ref + x + (avg3(x) if q.avg else 0)
        R = R + x.abs() + (avg3(x.abs()) if q.avg else 0)
    rm0, rv0 = mem.at(q.running_mean, F32, (Cc,)).clone(), mem.at(q.running_var, F32, (Cc,)).clone()
    eng.zero_arena.zero_()
    tv = mem.at(q.t, BF16, shape, nhwc_strides(H, W, q.t_pitch))
    got, = guarded(mem, [tv], lambda: bwd.check(lib.yv6_qa_fwd(h, C.byref(q), sp), lib))
    acc = F32_SUM * R
    worst = bwd.ratio(got, ref, acc + BF16_ULP * (ref.abs() + acc))
    tt = got.double().reshape(-1, Cc)
    return max(worst, stats_ratio(tt, mem.at(q.sums, F64, (2, Cc)), mem.at(q.stats, F32, (4, Cc)), mem.at(q.gamma, F32, (Cc,)),
                                  mem.at(q.beta, F32, (Cc,)), rm0, rv0, mem.at(q.running_mean, F32, (Cc,)),
                                  mem.at(q.running_var, F32, (Cc,)), q.momentum))


def tcheck_pool(lib, h, sp, mem, c, gen):
    """SPPF: the three chained 5x5 max-pools of channels [0, C) into [C, 4C) of one bf16 buffer: exact."""
    y, N, H, W, Cc, ct, nsplit, plane = c.args
    assert nsplit == 1
    buf = mem.at(y, BF16, (N, H, W, ct))
    fill(buf[..., :Cc], gen)
    t, ys = buf[..., :Cc].float().permute(0, 3, 1, 2), []
    for _ in range(3):
        t = F.max_pool2d(t, 5, 1, 2)
        ys.append(t.permute(0, 2, 3, 1))
    got, = guarded(mem, [buf[..., Cc:4 * Cc]], lambda: bwd.check(lib.yv6_sppf_pool(h, *c.args, sp), lib))
    assert bwd.bits_equal(got, torch.cat(ys, -1).to(BF16)), "training SPPF pool is not exact"
    return 0.0


def tcheck_abp(lib, h, sp, mem, c, gen):
    """head_ab_pack: NHWC [B, hw, na * ch] pred outputs -> rows (level, anchor, pixel); class scores and box offsets copied
    exactly, wh = (2 sigmoid(r))^2 * anchor against float64 (sigmoid through expf and one division, then three fp32
    products: 2^-20 of the value)."""
    raw_c, raw_r, B, hw, na, nc, anchors, row_off, rows, cls_ab, reg_ab = c.args
    rc, rr = mem.at(raw_c, F32, (B, hw, na, nc)), mem.at(raw_r, F32, (B, hw, na, 4))
    rc.copy_(torch.rand(rc.shape, generator=gen, device="cuda"))
    fill(rr, gen, 2.0)
    cv = mem.at(cls_ab + 4 * row_off * nc, F32, (B, na, hw, nc), (rows * nc, hw * nc, nc, 1))
    rv = mem.at(reg_ab + 4 * row_off * 4, F32, (B, na, hw, 4), (rows * 4, hw * 4, 4, 1))
    got_c, got_r = guarded(mem, [cv, rv], lambda: bwd.check(lib.yv6_head_ab_pack(h, *c.args, sp), lib))
    assert torch.equal(got_c, rc.permute(0, 2, 1, 3)), "head_ab_pack: class rows"
    assert torch.equal(got_r[..., :2], rr.permute(0, 2, 1, 3)[..., :2]), "head_ab_pack: box offsets"
    anc = torch.tensor(list(anchors), dtype=F64, device="cuda").view(na, 1, 2)
    wh = (2 * torch.sigmoid(rr.permute(0, 2, 1, 3)[..., 2:].double())) ** 2 * anc
    return bwd.ratio(got_r[..., 2:], wh, 2.0 ** -20 * wh.abs())


@pytest.mark.parametrize("name", list(TRAIN_CONFIGS))
def test_every_training_forward_launch_matches_float64(name):
    from yolov6_b200 import _lib
    t0 = time.time()
    m, eng, mem = train_engine(*TRAIN_CONFIGS[name])
    lib, h, sp = eng.lib, eng.h, _lib.stream_ptr()
    gen = torch.Generator(device="cuda").manual_seed(20261017)
    worst = {k: 0.0 for k in TRAIN_KINDS}
    seen = {k: set() for k in TRAIN_KINDS}
    total = {k: 0 for k in TRAIN_KINDS}
    for c in eng.fwd_calls:
        k = c.kind
        assert k in TRAIN_KINDS, k
        total[k] += 1
        sig = bwd.signature(c.desc, mem) if c.desc is not None else tuple(
            (mem.find(a)[0], mem.find(a)[2]) if isinstance(a, int) and a > 1 << 20 and mem.find(a) else
            (tuple(a) if isinstance(a, C.Array) else a) for a in c.args)
        if sig in seen[k]:
            continue
        seen[k].add(sig)
        r = {"conv": lambda: tcheck_conv(lib, h, sp, mem, c, gen), "stem": lambda: tcheck_stem(lib, h, sp, mem, eng, c, gen),
             "stats": lambda: tcheck_stats(lib, h, sp, mem, eng, c, gen), "apply": lambda: tcheck_apply(lib, h, sp, mem, c, gen),
             "qa": lambda: tcheck_qa(lib, h, sp, mem, eng, c, gen), "pool": lambda: tcheck_pool(lib, h, sp, mem, c, gen),
             "abp": lambda: tcheck_abp(lib, h, sp, mem, c, gen)}[k]()
        assert r <= 1.0, f"{name}: {k} launch {len(seen[k])}: error {r:.3f} x the bar"
        worst[k] = max(worst[k], r)
    for k in TRAIN_KINDS:
        if total[k]:
            assert seen[k]
    print(f"\n{name} (training forward): distinct launches checked (of all): "
          + ", ".join(f"{k} {len(seen[k])}/{total[k]}" for k in TRAIN_KINDS if total[k]))
    print(f"{name} (training forward): worst error / bar: " + ", ".join(f"{k} {worst[k]:.3f}" for k in TRAIN_KINDS if total[k])
          + f"; {time.time() - t0:.1f} s")
    del mem, eng, m
    torch.cuda.empty_cache()
