"""Every backward launch of the training engine, run alone on fresh seeded data and checked against float64.

`test_train_step_matches_reference_op_by_op` checks whole buffers at 1e-2 relative L2, which a wrong edge column or a wrong tap
in the border pixels of one dgrad parity does not move.  Here the engine plans a step -- YOLOv6-N / M / L6 at 96-128 px, N-QA
(the QA block's qa_bwd and its second bn_bwd on BN_d), N with the fuse_ab head (head_ab_grad), and the shapes the benchmark
trains: YOLOv6-S at 640, batch 32, uint8 input, and YOLOv6-M at 640, batch 8; the N / S self-distillation student at the
distillation benchmark's shape (S, 640, batch 32, uint8: the reg_preds_dist pred conv's 68-channel head gradient, its wgrad,
bias sums and a dgrad accumulating into the lrtb pred's input gradient); M with external neck-output gradients (every writer
of those slices accumulates) -- and every launch of its backward call list --
dgrad convs (grouped per op and branch: four parity launches for a 3x3 stride-2 conv, one for 1x1 stride 2), weight
gradients, BatchNorm backward (with the BottleRep shortcut), qa_bwd, the sums-only statistics of the pred and ConvTranspose
bias gradients, the head-gradient repacks, the SPPF max-pool backward chain and the stem im2col -- runs on its own descriptor:
every raw pointer is resolved to the engine tensor it lies in, so offsets and pitches are exactly the engine's.  Launches
with the same descriptor signature (fields, and pointer offsets inside their tensors) run once.

Engine memory.  Every tensor of the engine (activations, gradient buffers, dc / quadrant / pool scratch, head tensors and
gradients, statistics and coefficients, patches, fuse_ab and QA tensors) holds 2^100 before each launch, except the zero
arena, which holds zero as begin_step leaves it.  A check seeds the launch's inputs and the priors of its accumulating
outputs; an assigning output keeps the sentinel, so a pixel it fails to write is left at 2^100.  After the launch the inputs
must be unchanged, and once the inputs and outputs are put back every tensor must be at rest again, bit for bit.  The
gradient-buffer outputs of a launch are its Write records (train.Write: buffer, channel slice, every pixel when `full`), so
what a launch changes in the gradient buffers is held to what the first-writer resolution (train._resolve_first_writers)
was told.

Exact passes.  The flat master weights are integers in [-2, 2], repacked by begin_step into the forward and dgrad layouts
(the real-valued passes run on the fabricated weights).  dgrad, wgrad and the statistic sums also run on integer operands
in [-2, 2] (dgrad onto an integer prior when it
accumulates): every fp32 partial sum is then an integer below 2^24 (asserted per launch: K * max|a| * max|b| < 2^24), so
whatever the split-K, tiling or parity, wgrad must equal float64 plus the prior in fp32, dgrad float64 rounded once to bf16,
and the sums the float64 sums -- a lost or doubled split, tile or parity launch cannot hide in a rounding bar.

Real-valued passes, bars per element, R = the same operation on absolute values (the sum of absolute terms), u = 2^-24:
  dgrad, wgrad: 1e-5 R (fp32 accumulation of random terms), plus 2^-8 |ref| for a bf16 output;
  statistic sums: (L + 2) u R, L = the pixels one thread sums in fp32 before the float64 column sums (chan_run restates
    chan_grid of yv6_train.cu); the terms (bf16 values and their squares) are exact in fp32, so this bound is rigorous;
  bn_bwd: 1e-5 R for the pointwise fp32 work (activation backward, products, the apply pass) plus (L + 2) u R for the
    per-thread run of the reduce pass; dalpha sums 8 channels per pixel and a warp tree, a run of 8 L + 5; the premise
    L u < 2^-10 (first-order bound) is asserted per launch;
  qa_bwd: the 3x3 window sum of 9 terms, the product by 1/9 and two additions in fp32, 16 u of the absolute terms, plus one
    bf16 rounding;
  exact: head-gradient repack (g * (s * (1 - s)) in fp32, rounded once), head_ab_grad's class columns and box offsets,
    im2col (image -> bf16 hi + bf16 lo); head_ab_grad's w / h columns (sigmoid through expf): 2^-20 of |g * 8 anchor| s^2 plus
    one bf16 rounding;
  max-pool backward: sums of <= 25 quantised bf16 values are exact in fp32, so each launch's output is one bf16 rounding of
    the exact sum; the reference rounds each link of the chain the same way and the bar allows one bf16 rounding.
The float64 references run on the GPU (torch's float64 convolutions and autograd, no code shared with this library); the
first launch of each kind with a float64 reference is cross-checked once against the same computation on the CPU (image 0
where the operation is per image).  The printed numbers are the distinct and total launches per kind, the worst error / bar
ratio per kind, and the time taken."""
import ctypes as C
import functools
import math
import time

import pytest
import torch
import torch.nn.functional as F

from conftest import golden_keys
from oracle import fabricate as fab

pytestmark = pytest.mark.gpu

# name -> model config, image size, batch, fuse_ab head, uint8 input.  S and M at 640 are the shapes bench.py trains.
MODELS = {
    "yolov6n": dict(cfg="yolov6n", size=128, batch=2), "yolov6m": dict(cfg="yolov6m", size=96, batch=2),
    "yolov6l6": dict(cfg="yolov6l6", size=128, batch=2), "yolov6n_qa": dict(cfg="yolov6n_qa", size=96, batch=2),
    "yolov6n_fuse_ab": dict(cfg="yolov6n", size=128, batch=2, fuse_ab=True),
    "yolov6s_640_b32_u8": dict(cfg="yolov6s", size=640, batch=32, u8=True), "yolov6m_640_b8": dict(cfg="yolov6m", size=640, batch=8),
    # the N / S self-distillation student (third pred conv per level, reg_preds_dist) at the shape tools/bench_distill.py
    # trains, and M with the neck outputs' gradients injected by the channel-wise distillation term
    "yolov6s_640_b32_u8_distill_ns": dict(cfg="yolov6s", size=640, batch=32, u8=True, distill_ns=True),
    "yolov6m_96_b2_feat": dict(cfg="yolov6m", size=96, batch=2, feat=True),
}
GOLDEN_KEYS = ("yolov6n", "yolov6s", "yolov6m", "yolov6l6")
BN_EPS = 1e-3
F32_SUM = 1e-5           # fp32 accumulation, relative to the sum of absolute terms
BF16_ULP = 2.0 ** -8     # one round-to-nearest-even to bf16 (8 significant bits) moves a value by at most 2^-8 of it
U = 2.0 ** -24           # fp32 unit roundoff
SENTINEL = 2.0 ** 100
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
REST_EXEMPT = ("param", "img")   # master weights and the input image: not outputs of any backward launch


# ---------------------------------------------------------------------------------------------------------------- helpers
class Mem:
    """Device tensors by address range: turns a descriptor's raw pointer into a view of the tensor it lies in."""

    def __init__(self, named):
        self.ts = []
        for tag, t in named:
            if t is None:
                continue
            assert t.is_contiguous() and t.storage_offset() == 0, tag
            self.ts.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), tag, t))

    def find(self, ptr):
        for lo, hi, tag, t in self.ts:
            if lo <= ptr < hi:
                return tag, t, ptr - lo
        return None

    def at(self, ptr, dtype, shape, strides=None):
        f = self.find(ptr)
        assert f is not None, f"pointer {ptr:#x} lies in no known tensor"
        _, t, off = f
        esz = torch.empty(0, dtype=dtype).element_size()
        assert off % esz == 0
        if strides is None:
            strides = [1] * len(shape)
            for k in range(len(shape) - 2, -1, -1):
                strides[k] = strides[k + 1] * shape[k + 1]
        flat = t.reshape(-1).view(torch.uint8).view(dtype)
        assert off // esz + sum((s - 1) * st for s, st in zip(shape, strides)) < flat.numel(), "view leaves its tensor"
        return flat.as_strided(tuple(shape), tuple(strides), off // esz)

    def base(self, ptr):
        return self.find(ptr)[1]


class IO:
    """What one check did to engine memory: inputs it seeded (with a copy, they must come out unchanged) and outputs."""

    def __init__(self):
        self.seeded, self.ins, self.outs = [], [], []

    def seed(self, v):
        self.seeded.append(v)
        return v

    def freeze(self):
        """Right before the launch: copies of the seeded inputs."""
        self.ins = [(v, v.clone()) for v in self.seeded]

    def out(self, v):
        self.outs.append(v)
        return v


def int_view(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def at_rest(tag, t):
    if tag == "arena":
        return not bool(t.any())
    return bool((int_view(t) == int_view(torch.tensor([SENTINEL], dtype=t.dtype)).item()).all())


def poison(mem):
    """Every engine tensor to its rest state: the zero arena zero (as begin_step leaves it), everything else 2^100."""
    for _, _, tag, t in mem.ts:
        if tag == "arena":
            t.zero_()
        elif tag not in REST_EXEMPT:
            t.fill_(SENTINEL)


def settle(mem, ins, outs, what):
    """After a checked launch: its inputs still hold what was seeded; then inputs and outputs go back to rest, and every engine
    tensor must be at rest everywhere -- an element the launch wrote outside its declared outputs is left over."""
    for v, before in ins:
        assert torch.equal(int_view(v), int_view(before)), f"{what}: changed one of its inputs"
    for v in [v for v, _ in ins] + list(outs):
        if mem.find(v.data_ptr())[0] == "arena":
            v.zero_()
        else:
            v.fill_(SENTINEL)
    bad = [f"{tag} {tuple(t.shape)}" for _, _, tag, t in mem.ts if tag not in REST_EXEMPT and not at_rest(tag, t)]
    assert not bad, f"{what}: wrote outside the outputs it declares: " + "; ".join(bad)


def assert_full_write(v, what):
    """An assigning write started from the sentinel: every element must have been written."""
    left = v.float().abs() >= SENTINEL
    assert not bool(left.any()), f"{what}: not every pixel of a full write was written ({int(left.sum())} elements left)"


def assert_exact(got, exp, what):
    diff = got.double() != exp.double()
    assert not bool(diff.any()), (f"{what}: not exact: {int(diff.sum())} elements differ, worst by "
                                  f"{float((got.double() - exp.double()).abs().max()):.3g}")


def exact_k_bound(k, amax, bmax, prior=2):
    """Every fp32 partial sum of k products of integers |a| <= amax, |b| <= bmax onto an integer prior is exact."""
    return k * amax * bmax + prior < 2 ** 24


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def chan_run(pixels, c, per_sm, min_iters):
    """Pixels one thread of the channel-reduction kernels sums in fp32: chan_grid (yv6_train.cu) restated.  Threads per block
    cover C / 8 channel groups x prows pixel rows; the grid is capped at per_sm blocks per SM."""
    prows = max(1, 256 // (c // 8))
    grid = max(1, min(-(-pixels // (prows * min_iters)), num_sms() * per_sm))
    return -(-pixels // (grid * prows))


def run_bar(run):
    """fp32 sum of `run` terms, then converted into a float64 sum: (run + 2) u of the sum of absolute terms (first order)."""
    assert run * U < 2.0 ** -10, f"a run of {run} fp32 additions is outside the first-order bound"
    return (run + 2) * U


def signature(d, mem):
    """Descriptor fields, with each pointer replaced by (tensor kind, offset inside it); per-op accumulator slots in the zero
    arena and parameters compare equal whatever their offset."""
    out = [type(d).__name__]
    for fname, ty in d._fields_:
        v = getattr(d, fname)
        vals = list(v) if isinstance(v, C.Array) else [v]
        is_ptr = ty is C.c_void_p or (issubclass(ty, C.Array) and ty._type_ is C.c_void_p)
        for x in vals:
            if is_ptr:
                f = mem.find(x) if x else None
                out.append(None if f is None else (f[0], None if f[0] in ("arena", "param") else f[2]))
            else:
                out.append(x)
    return tuple(out)


def rnd(gen, *shape, dtype=BF16, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=gen, dtype=F64, device=gen.device) * scale + shift).to(dtype)


def ints(gen, *shape, dtype=BF16):
    return torch.randint(-2, 3, shape, generator=gen, device=gen.device).to(dtype)


def ratio(got, exp, bound):
    """max |got - exp| / bound; where the bound is 0 the values must be equal."""
    got, exp, bound = got.double(), exp.double(), bound.double()
    err = (got - exp).abs()
    assert not bool(torch.isnan(err).any()), "NaN where a value was expected"
    bad = (err > 0) & (bound <= 0)
    assert not bool(bad.any()), f"{int(bad.sum())} elements differ where they must be exact"
    r = err / bound.clamp_min(1e-300)
    r = torch.where(bound > 0, r, torch.zeros_like(r))
    return float(r.max()) if r.numel() else 0.0


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def nhwc_strides(H, W, pitch):
    return (H * W * pitch, W * pitch, pitch, 1)


def check(lib_rc, lib):
    assert lib_rc == 0, lib.yv6_last_error().decode()


XCHECKED = set()     # kinds whose GPU float64 reference was cross-checked on the CPU


def cross_check(kind, ref, R, fn):
    """Once per kind: the GPU float64 reference `ref` (R: its absolute-value sum) against fn() = the same on the CPU."""
    if kind in XCHECKED:
        return
    XCHECKED.add(kind)
    rc = fn()
    err = float(((ref.cpu() - rc).abs() / (R.cpu() + 1e-300)).max())
    assert err < 1e-12, f"{kind}: GPU float64 reference differs from the CPU by {err:.2e} of R"


# ---------------------------------------------------------------------------------------------------------------- per-kind checks
def check_dgrad(lib, h, sp, mem, descs, wf, stride, gbuf, meta, gen, io, exact):
    """One op's input gradient: g(src)[..., off:off + cin] (+)= conv2d_input(dc, W) over the launches of `descs` (all read the same
    dc).  An assigning group starts from the sentinel, an accumulating one from a prior; pixels no launch writes keep it."""
    d0 = descs[0]
    off, cin = meta.off, meta.n
    N, Hd, Wd, Cd, xct = d0.N, d0.H, d0.W, d0.Cin, d0.x_c_total
    assert all(d.x == d0.x for d in descs)
    acc = {bool(d.res) for d in descs}
    assert len(acc) == 1, "launches of one dgrad disagree on accumulate"
    acc = acc.pop()
    co, k, _, ci = wf.shape
    assert ci == cin
    if exact:
        assert exact_k_bound(co * k * k, 2, 2), "dgrad sum too long for exact integer operands"
    dcv = mem.at(d0.x, BF16, (N, Hd, Wd, Cd), (Hd * Wd * xct, Wd * xct, xct, 1))
    dcv.copy_(ints(gen, N, Hd, Wd, Cd) if exact else rnd(gen, N, Hd, Wd, Cd))
    io.seed(dcv)
    sl = io.out(gbuf[..., off:off + cin])
    if acc:
        sl.copy_(ints(gen, *sl.shape) if exact else rnd(gen, *sl.shape))
    before = sl.clone()
    io.freeze()
    for d in descs:
        check(lib.yv6_conv_fwd(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    # which pixels the launches write: element (n, i, j) of launch d sits at d.y + n*s0 + i*s1 + j*s2 (elements)
    n_, hs, ws, gct = gbuf.shape
    dev = gbuf.device
    written = torch.zeros(n_ * hs * ws, dtype=torch.bool, device=dev)
    base = gbuf.data_ptr()
    for d in descs:
        oh = d.out_h or (d.H + 2 * d.pad - d.kh) // d.stride + 1
        ow = d.out_w or (d.W + 2 * d.pad - d.kw) // d.stride + 1
        e0 = (d.y - base) // 2 - off
        idx = (e0 + torch.arange(d.N, device=dev).view(-1, 1, 1) * d.y_img_stride + torch.arange(oh, device=dev).view(1, -1, 1) * d.y_h_stride
               + torch.arange(ow, device=dev).view(1, 1, -1) * d.y_w_stride)
        assert bool((idx % gct == 0).all())
        written[(idx // gct).reshape(-1)] = True
    written = written.view(n_, hs, ws)
    assert not meta.full or bool(written.all()), "a full Write whose launches leave pixels out"
    w64 = nchw(wf).contiguous()
    dcn = nchw(dcv[..., :co])
    gin = torch.nn.grad.conv2d_input((n_, ci, hs, ws), w64, dcn, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    assert not bool(((gin != 0) & ~written[..., None]).any()), "the launches do not cover every pixel of the input gradient"
    got = sl.clone()
    assert torch.equal(int_view(got[~written]), int_view(before[~written])), "dgrad wrote pixels outside its launches"
    if not acc:
        assert_full_write(got[written], "dgrad")
    p = before[written].double() if acc else 0.0
    exp = p + gin[written]
    if exact:
        assert_exact(got[written], exp.to(BF16), "dgrad")
        return 0.0
    R = torch.nn.grad.conv2d_input((n_, ci, hs, ws), w64.abs(), dcn.abs(), stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    cross_check("dgrad", gin[:1], R[:1], lambda: torch.nn.grad.conv2d_input((1, ci, hs, ws), w64.cpu(), dcn[:1].cpu(), stride=stride,
                                                                            padding=k // 2).permute(0, 2, 3, 1))
    pa = p.abs() if acc else 0.0
    return ratio(got[written], exp, BF16_ULP * exp.abs() + F32_SUM * (R[written] + pa))


def wgrad_ref(x, dy, cout, k, stride, pad, absolute=True):
    """dW [Cout][k][k][Cin] of conv2d(x, W) against dy, and the same on absolute values (x, dy: NHWC)."""
    xs, ds = nchw(x), nchw(dy)
    shape = (cout, x.shape[3], k, k)
    ref = torch.nn.grad.conv2d_weight(xs, shape, ds, stride=stride, padding=pad).permute(0, 2, 3, 1)
    if not absolute:
        return ref, None
    R = torch.nn.grad.conv2d_weight(xs.abs(), shape, ds.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return ref, R


def check_wgrad(lib, h, sp, mem, d, gen, io, exact):
    """dW += wgrad(x, dY) on the descriptor's slices, onto a prior and onto zeros."""
    N, H, W, Cin, xct, Cout, dct, k = d.N, d.H, d.W, d.Cin, d.x_c_total, d.Cout, d.dy_c_total, d.kh
    Ho, Wo = (H + 2 * d.pad - k) // d.stride + 1, (W + 2 * d.pad - d.kw) // d.stride + 1
    if exact:
        assert exact_k_bound(N * Ho * Wo, 2, 2), "wgrad sum too long for exact integer operands"
    for ptr in (d.x, d.dy):     # whole tensors: channels outside the slices hold data too
        t = mem.base(ptr)
        t.copy_(ints(gen, *t.shape, dtype=t.dtype) if exact else rnd(gen, *t.shape, dtype=t.dtype))
        io.seed(t)
    x = mem.at(d.x, BF16, (N, H, W, Cin), (H * W * xct, W * xct, xct, 1))
    dy = mem.at(d.dy, BF16, (N, Ho, Wo, Cout), (Ho * Wo * dct, Wo * dct, dct, 1))
    dw = io.out(mem.at(d.dw, F32, (Cout, k, k, Cin)))
    ref, R = wgrad_ref(x, dy, Cout, k, d.stride, d.pad, absolute=not exact)
    if not exact:
        cross_check("wgrad", wgrad_ref(x[:1], dy[:1], Cout, k, d.stride, d.pad, absolute=False)[0],
                    wgrad_ref(x[:1], dy[:1], Cout, k, d.stride, d.pad)[1],
                    lambda: wgrad_ref(x[:1].cpu(), dy[:1].cpu(), Cout, k, d.stride, d.pad, absolute=False)[0])
    prior = ints(gen, Cout, k, k, Cin, dtype=F32) if exact else rnd(gen, Cout, k, k, Cin, dtype=F32)
    worst = 0.0
    for pr in (prior, torch.zeros_like(prior)):
        dw.copy_(pr)
        io.freeze()
        check(lib.yv6_conv_wgrad(h, C.byref(d), sp), lib)
        torch.cuda.synchronize()
        p = pr.double()
        if exact:
            assert_exact(dw, (p + ref).float(), "wgrad")
        else:
            worst = max(worst, ratio(dw, p + ref, F32_SUM * (R + p.abs())))
    return worst


def check_stats_sums(lib, h, sp, mem, d, gen, io, exact):
    """Sums only (no finalize): per-channel sum and sum of squares of an NHWC slice into a zeroed arena slot."""
    assert d.nb == 1 and not d.stats[0]
    P, Cc, pitch = d.pixels, d.C, d.x_pitch[0]
    t = mem.base(d.x[0])
    t.copy_(ints(gen, *t.shape, dtype=t.dtype) if exact else rnd(gen, *t.shape, dtype=t.dtype))
    io.seed(t)
    x = mem.at(d.x[0], BF16, (P, Cc), (pitch, 1)).double()
    sums = io.out(mem.at(d.sums, F64, (2, Cc)))
    io.out(mem.at(d.counter, torch.int32, (1,)))
    assert d.zeroed      # the arena slots are zero, as begin_step leaves them
    io.freeze()
    check(lib.yv6_bn_stats_finalize(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    q = x * x
    if exact:
        assert exact_k_bound(P, 2, 2), "statistic sums too long for exact integer operands"
        assert_exact(sums[0], x.sum(0), "stats sum")
        assert_exact(sums[1], q.sum(0), "stats sum of squares")
        return 0.0
    cross_check("stats", x.sum(0), x.abs().sum(0), lambda: x.cpu().sum(0))
    bar = run_bar(chan_run(P, Cc, 4, 16))
    return max(ratio(sums[0], x.sum(0), bar * x.abs().sum(0)), ratio(sums[1], q.sum(0), bar * q.sum(0)))


def bn_bwd_ref(xs, st, dy, act, res=None, alpha=0.0):
    """Autograd through act(sum_b BN_b(x_b)) (+ alpha * res) with batch-statistics BatchNorm, float64.  Returns (dz, dbeta,
    [dgamma_b], [dx_b], dres, dalpha)."""
    xr = [x.clone().requires_grad_(True) for x in xs]
    gr = [s["gam"].clone().requires_grad_(True) for s in st]
    br = [s["bet"].clone().requires_grad_(True) for s in st]
    z = 0
    for b in range(len(xs)):
        mu, var = xr[b].mean(0), xr[b].var(0, unbiased=False)
        z = z + (xr[b] - mu) / torch.sqrt(var + BN_EPS) * gr[b] + br[b]
    z.retain_grad()
    y = torch.relu(z) if act == 1 else (z * torch.sigmoid(z) if act == 2 else z)
    rr = al = None
    if res is not None:
        rr = res.double().requires_grad_(True)
        al = torch.tensor(alpha, dtype=F64, device=res.device, requires_grad=True)
        y = y + al * rr
    (y * dy.double()).sum().backward()
    return (z.grad, br[0].grad, [g.grad for g in gr], [x.grad for x in xr], None if rr is None else rr.grad,
            None if al is None else al.grad.view(1))


def check_bn_bwd(lib, h, sp, mem, d, gen, positive=False, io=None):
    """yv6_bn_bwd on fresh branch inputs with their true batch statistics in the stat slots, against float64 autograd through
    act(sum_b BN_b(x_b)) (+ alpha * res) with batch-statistics BatchNorm.  Returns {output: worst ratio}.  With `io` (engine
    memory) an assigning output starts from the sentinel and must be written everywhere."""
    nb, Cc, P, act = d.nb, d.C, d.pixels, d.act
    dev = gen.device
    host = lambda t: t.to(dev)     # noqa: E731
    view = lambda ptr, pitch: mem.at(ptr, BF16, (P, Cc), (pitch, 1))     # noqa: E731
    engine = io is not None
    io = io or IO()
    L = chan_run(P, Cc, 4, 16)           # the reduce pass's grid (yv6_bn_bwd: grid_r)
    rb = F32_SUM + run_bar(L)
    xs, st = [], []
    for b in range(nb):
        x = rnd(gen, P, Cc, scale=1 + b, shift=0.3 * b)
        io.seed(view(d.x[b], d.x_pitch[b])).copy_(x)
        xs.append(x.double())
    for b in range(nb):
        x = xs[b]
        gam = torch.rand(Cc, generator=gen, dtype=F64, device=dev) + 0.5
        bet = torch.randn(Cc, generator=gen, dtype=F64, device=dev) * 0.1
        mean, var = x.mean(0), x.var(0, unbiased=False)
        inv = 1.0 / torch.sqrt(var + BN_EPS)
        vals = [mean, inv, gam * inv, bet - mean * gam * inv]
        for ptr, v in zip((d.mean[b], d.invstd[b], d.scale[b], d.shift[b]), vals):
            io.seed(mem.at(ptr, F32, (Cc,))).copy_(v.float())
        st.append(dict(gam=gam, bet=bet, mean=mean.float().double(), inv=inv.float().double(), sc=(gam * inv).float().double(),
                       sh=(bet - mean * gam * inv).float().double()))
    dy = torch.randn(P, Cc, generator=gen, dtype=F64, device=dev)
    if positive:
        dy = dy.abs() + 0.1
    if act == 1:       # relu: where z is within fp32 rounding of 0 the kernel and float64 may disagree on the mask -- no gradient there
        z32 = sum(xs[b] * st[b]["sc"] + st[b]["sh"] for b in range(nb))
        tau = 1e-5 * (sum(st[b]["sh"].abs() for b in range(nb)) + sum((xs[b] * st[b]["sc"]).abs() for b in range(nb)))
        dy[z32.abs() < tau] = 0
    dy = dy.to(BF16)
    io.seed(view(d.dy, d.dy_pitch)).copy_(dy)
    has_res = bool(d.res)
    sentinel_assign = engine
    if has_res:
        res = rnd(gen, P, Cc)
        if positive:
            res = res.abs()
        io.seed(view(d.res, d.res_pitch)).copy_(res)
        alpha = float(mem.at(d.res_alpha_dev, F32, (1,)).item()) if d.res_alpha_dev else float(d.res_alpha)
        dres_prior = rnd(gen, P, Cc)
        dres_v = io.out(view(d.dres, d.dres_pitch))
        if not (sentinel_assign and d.dres_assign):
            dres_v.copy_(dres_prior)
    dx_prior = []
    for b in range(nb):
        pr = rnd(gen, P, Cc)
        v = io.out(view(d.dx[b], d.dx_pitch[b]))
        if not (sentinel_assign and not d.accumulate[b]):
            v.copy_(pr)
        dx_prior.append(pr)
    # accumulators: a caller arena with zeroed = 1 is cleared by the caller; otherwise the launch clears them (garbage here)
    caller = bool(d.work)
    garbage = lambda t: t.copy_(torch.randn(t.shape, generator=gen, dtype=F64, device=dev).to(t.dtype))   # noqa: E731
    s1 = io.out(mem.at(d.s1, F64, (Cc,)))
    s2 = [io.out(mem.at(d.s2[b], F64, (Cc,))) for b in range(nb)]
    for t in s2:
        garbage(t)
    da = io.out(mem.at(d.dalpha, F64, (1,))) if has_res else None
    if caller:
        work, cnt = io.out(mem.at(d.work, F64, (nb, Cc))), io.out(mem.at(d.counter, torch.int32, (1,)))
        coef = io.out(mem.at(d.coef, F32, (nb, 2, Cc)))
        garbage(coef)
    if caller and d.zeroed:
        for t in [s1, work, cnt] + ([da] if has_res else []):
            t.zero_()
    else:
        for t in [s1] + ([da] if has_res else []) + ([work] if caller else []):
            garbage(t)
    io.freeze()
    check(lib.yv6_bn_bwd(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()

    # ---- float64 reference
    dz, S1, S2s, dxs, dres_g, dal = bn_bwd_ref(xs, st, dy, act, res if has_res else None, alpha if has_res else 0.0)
    if "bn_bwd" not in XCHECKED and P * Cc <= 1 << 22:
        cpu = lambda t: None if t is None else t.cpu()     # noqa: E731
        ref_c = bn_bwd_ref([cpu(x) for x in xs], [{k: cpu(v) for k, v in s.items()} for s in st], cpu(dy), act,
                           cpu(res) if has_res else None, alpha if has_res else 0.0)
        cross_check("bn_bwd", dxs[0], torch.full_like(dxs[0], float(dxs[0].abs().max())), lambda: ref_c[3][0])
    out = {}
    R1 = dz.abs().sum(0)
    out["s1"] = ratio(host(s1), S1, rb * R1)
    worst_dx, worst_s2 = 0.0, 0.0
    for b in range(nb):
        s = st[b]
        R2 = s["inv"] * ((dz.abs() * xs[b].abs()).sum(0) + s["mean"].abs() * R1)
        worst_s2 = max(worst_s2, ratio(host(s2[b]), S2s[b], rb * R2))
        Bc = -s["sc"] * s["inv"] * S2s[b] / P
        Cb = -s["sc"] * S1 / P - Bc * s["mean"]
        xhat = (xs[b] - s["mean"]) * s["inv"]
        acc = bool(d.accumulate[b])
        p = dx_prior[b].double() * acc
        Rdx = ((s["sc"] * dz).abs() + Bc.abs() * xs[b].abs() + Cb.abs() + s["sc"].abs() * (R1 + xhat.abs() * R2) / P + p.abs())
        exp = p + dxs[b]
        got = host(view(d.dx[b], d.dx_pitch[b]))
        if sentinel_assign and not acc:
            assert_full_write(got, "bn_bwd dx")
        worst_dx = max(worst_dx, ratio(got, exp, BF16_ULP * exp.abs() + rb * Rdx))
        if caller:      # coefficients of the apply pass: the closed form of the kernel's comment on its own sums
            S1k, S2k = host(s1), host(s2[b])
            Bk = -s["sc"] * s["inv"] * S2k / P
            Ck = -s["sc"] * S1k / P - Bk * s["mean"]
            cf = host(coef).double()
            out["coef"] = max(out.get("coef", 0.0), ratio(cf[b, 0], Bk, 2.0 ** -22 * Bk.abs()),
                              ratio(cf[b, 1], Ck, 2.0 ** -22 * ((s["sc"] * S1k / P).abs() + (Bk * s["mean"]).abs())))
    out["s2"], out["dx"] = worst_s2, worst_dx
    if has_res:
        keep = 0.0 if d.dres_assign else 1.0
        p = dres_prior.double() * keep
        exp = p + dres_g
        got = host(view(d.dres, d.dres_pitch))
        if sentinel_assign and d.dres_assign:
            assert_full_write(got, "bn_bwd dres")
        out["dres"] = ratio(got, exp, BF16_ULP * exp.abs() + F32_SUM * ((alpha * dy.double()).abs() + p.abs()))
        out["dalpha"] = ratio(host(da), dal, (F32_SUM + run_bar(8 * L + 5)) * (dy.double() * res.double()).abs().sum().view(1))
    return out


def check_qa_bwd(lib, h, sp, mem, q, gen, io):
    """yv6_qa_bwd: dx (+)= dt + avg3x3^T(dt) (the adjoint of AvgPool2d(3, 1, 1) with count_include_pad is the same box filter)."""
    N, H, W, Cc = q.N, q.H, q.W, q.C
    dt = io.seed(mem.at(q.dt, BF16, (N, H, W, Cc), nhwc_strides(H, W, q.dt_pitch)))
    dt.copy_(rnd(gen, N, H, W, Cc))
    dx = io.out(mem.at(q.dx, BF16, (N, H, W, Cc), nhwc_strides(H, W, q.dx_pitch)))
    acc = bool(q.accumulate)
    if acc:
        dx.copy_(rnd(gen, N, H, W, Cc))
    p = dx.double() if acc else 0.0
    io.freeze()
    check(lib.yv6_qa_bwd(h, C.byref(q), sp), lib)
    torch.cuda.synchronize()
    d64 = dt.double()
    avg3 = lambda t: F.avg_pool2d(t.permute(0, 3, 1, 2), 3, 1, 1, count_include_pad=True).permute(0, 2, 3, 1)  # noqa: E731
    ref = p + d64 + (avg3(d64) if q.avg else 0.0)
    R = d64.abs() + (avg3(d64.abs()) if q.avg else 0.0) + (p.abs() if acc else 0.0)
    if q.avg:
        cross_check("qa_bwd", (d64 + avg3(d64))[:1], R[:1], lambda: d64[:1].cpu() + avg3(d64[:1].cpu()))
    if not acc:
        assert_full_write(dx, "qa_bwd dx")
    return ratio(dx, ref, 16 * U * R + BF16_ULP * ref.abs())     # window of 9 terms, x 1/9, two additions


def check_hgp(lib, h, sp, mem, args, gen, io):
    """dlogit = bf16(g * (s * (1 - s))) (or bf16(g)), repacked to NHWC with zero padded channels: bit for bit."""
    gp, sp_, B, A, ch, off, hw, chp, outp = args
    g = io.seed(mem.at(gp, F32, (B, A, ch)))
    g.copy_(torch.randn(B, A, ch, generator=gen, device=gen.device))
    if sp_:
        s = io.seed(mem.at(sp_, F32, (B, A, ch)))
        s.copy_(torch.rand(B, A, ch, generator=gen, device=gen.device))
    out = io.out(mem.at(outp, BF16, (B, hw, chp)))
    io.freeze()
    check(lib.yv6_head_grad_prep(h, gp, sp_, B, A, ch, off, hw, chp, outp, sp), lib)
    torch.cuda.synchronize()
    v = g[:, off:off + hw]
    if sp_:
        sv = s[:, off:off + hw]
        v = v * (sv * (1 - sv))
    exp = torch.zeros(B, hw, chp, dtype=F32, device=g.device)
    exp[..., :ch] = v
    assert bits_equal(out, exp.to(BF16)), "head_grad_prep differs from bf16(g * s * (1 - s))"
    return 0.0


def check_abg(lib, h, sp, mem, args, gen, io):
    """yv6_head_ab_grad: rows (level, anchor, pixel) of the fuse_ab gradients -> NHWC bf16 gradients of the raw pred outputs.
    Class columns bf16((g * s) * (1 - s)) and box offsets bf16(g) bit for bit; w / h: g * 8 anchor s^2 (1 - s), s = sigmoid of
    the raw output; padded channels zero."""
    gca, ca, gra, rawr, B, hw, na, nc, anchors, row_off, rows, cpad, rpad, dlc, dlr = args
    dev = gen.device
    gc, sc = io.seed(mem.at(gca, F32, (B, rows, nc))), io.seed(mem.at(ca, F32, (B, rows, nc)))
    gr, raw = io.seed(mem.at(gra, F32, (B, rows, 4))), io.seed(mem.at(rawr, F32, (B, hw, na * 4)))
    gc.copy_(torch.randn(gc.shape, generator=gen, device=dev))
    sc.copy_(torch.rand(sc.shape, generator=gen, device=dev))
    gr.copy_(torch.randn(gr.shape, generator=gen, device=dev))
    raw.copy_(torch.randn(raw.shape, generator=gen, device=dev) * 2)
    oc, orr = io.out(mem.at(dlc, BF16, (B, hw, cpad))), io.out(mem.at(dlr, BF16, (B, hw, rpad)))
    io.freeze()
    check(lib.yv6_head_ab_grad(h, *args, sp), lib)
    torch.cuda.synchronize()
    rows_of = lambda t, c: t[:, row_off:row_off + na * hw].reshape(B, na, hw, c).permute(0, 2, 1, 3)   # noqa: E731  [B, hw, na, c]
    g, s = rows_of(gc, nc), rows_of(sc, nc)
    exp_c = torch.zeros(B, hw, cpad, dtype=F32, device=dev)
    exp_c[..., :na * nc] = ((g * s) * (1 - s)).reshape(B, hw, na * nc)
    assert bits_equal(oc, exp_c.to(BF16)), "head_ab_grad: class columns"
    g4 = rows_of(gr, 4).double()                                   # [B, hw, na, 4]
    r4 = raw.view(B, hw, na, 4).double()
    anc = torch.tensor(list(anchors), dtype=F64, device=dev).view(1, 1, na, 2)
    sg = torch.sigmoid(r4[..., 2:])
    wh = g4[..., 2:] * anc * 8 * sg * sg * (1 - sg)
    got = orr[..., :na * 4].reshape(B, hw, na, 4)
    assert bits_equal(got[..., :2], g4[..., :2].float().to(BF16)), "head_ab_grad: box offsets"
    assert not bool(orr[..., na * 4:].any()), "head_ab_grad: padded channels"
    return ratio(got[..., 2:], wh, BF16_ULP * wh.abs() + 2.0 ** -20 * (g4[..., 2:] * anc * 8).abs() * sg * sg)


def check_pool_chain(lib, h, sp, eng, mem, calls, gen, io):
    """The three chained MaxPool2d(5, 1, 2) backward launches of one SPPF against torch's max-pool backward in float64 (scatter to
    the first maximum in row-major window order), on operands quantised to a few levels so that ties are everywhere.  Each
    launch changes exactly the slice of its Write record; an assigning launch starts from the sentinel."""
    n, hh, ww, c = calls[0].args[4:8]
    bi = calls[0].writes[0].buf
    buf, gbuf = eng.bufs[bi], eng.gbufs[bi]
    cg = torch.Generator().manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=gen, device=gen.device)))
    ys = [torch.randint(0, 4, (n, c, hh, ww), generator=cg).double()]
    for _ in range(3):
        ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
    for j in range(4):
        buf[..., j * c:(j + 1) * c] = ys[j].permute(0, 2, 3, 1).to(BF16).to(buf.device)
    io.seed(buf)
    prior = torch.randint(-3, 4, (n, hh, ww, 4 * c), generator=cg).to(BF16)
    io.seed(gbuf[..., 3 * c:4 * c]).copy_(prior[..., 3 * c:])           # the incoming gradient of the last pooled slice
    for call in calls:
        w = call.writes[0]
        assert w.full and w.n == c
        if call.args[11]:            # accumulates: starts from a prior; an assigning launch starts from the sentinel
            gbuf[..., w.off:w.off + c] = prior[..., w.off:w.off + c].to(gbuf.device)
        io.out(mem.base(call.args[8]))
    io.out(gbuf[..., :3 * c])
    io.freeze()
    G = [nchw(prior[..., j * c:(j + 1) * c]) for j in range(4)]
    for call in calls:
        d, w = call.args, call.writes[0]
        j = w.off // c + 1
        assert d[0] == buf.data_ptr() + (j - 1) * c * 2 and d[2] == gbuf.data_ptr() + j * c * 2
        before = gbuf.clone()
        check(lib.yv6_maxpool5_bwd(h, *d, sp), lib)
        torch.cuda.synchronize()
        keep = torch.ones(gbuf.shape[-1], dtype=torch.bool, device=gbuf.device)
        keep[w.off:w.off + w.n] = False
        assert torch.equal(int_view(gbuf[..., keep]), int_view(before[..., keep])), "pool_bwd wrote outside its Write record"
        if not d[11]:
            assert_full_write(gbuf[..., w.off:w.off + c], "pool_bwd")
        y = ys[j - 1].clone().requires_grad_(True)
        F.max_pool2d(y, 5, 1, 2).backward(G[j])
        G[j - 1] = (G[j - 1] * d[11] + y.grad).to(BF16).double()
    got = gbuf[..., :4 * c].cpu()
    exp = torch.cat([g.permute(0, 2, 3, 1) for g in G], -1)
    return ratio(got, exp, BF16_ULP * exp.abs())


def im2col_ref(img, scale):
    """patches [N, Ho, Wo, 32] fp32: column (r*3+s)*3+c = x[n, c, 2ho+r-1, 2wo+s-1] (zero outside), columns 27..31 zero."""
    x = img.float() * torch.tensor(scale, dtype=F32, device=img.device) if img.dtype == torch.uint8 else img.float()
    N, _, H, W = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x, (1, 1, 1, 1))
    v = torch.zeros(N, Ho, Wo, 32, dtype=F32, device=img.device)
    for r in range(3):
        for s in range(3):
            for c in range(3):
                v[..., (r * 3 + s) * 3 + c] = xp[:, c, r:r + 2 * Ho - 1:2, s:s + 2 * Wo - 1:2]
    hi = v.to(BF16)
    return hi, (v - hi.float()).to(BF16)


def check_im2col(lib, h, sp, img_ptr, img, x_dt, scale, N, H, W, patches, patches_lo, gen, io=None):
    """Bit for bit.  With `io` (engine memory) the patches start from the sentinel, so every element must be written."""
    if io is None:
        patches.copy_(rnd(gen, *patches.shape).to(patches.device))
        patches_lo.copy_(rnd(gen, *patches_lo.shape).to(patches.device))
    else:
        io.out(patches), io.out(patches_lo)
    check(lib.yv6_stem_im2col(h, img_ptr, x_dt, C.c_float(scale), N, H, W, patches.data_ptr(), patches_lo.data_ptr(), sp), lib)
    torch.cuda.synchronize()
    hi, lo = im2col_ref(img, C.c_float(scale).value)
    assert bits_equal(patches.to(hi.device), hi), "im2col: bf16 patches"
    assert bits_equal(patches_lo.to(hi.device), lo), "im2col: bf16 residual plane"
    return 0.0


# ---------------------------------------------------------------------------------------------------------------- the engine's launches
def seeded_model(cfg, dev, fuse_ab=False, distill_ns=False, dfl=False):
    """The model with seeded weights: the fabricated golden state of its config where golden keys exist, else randomize_.  A
    distill_ns student (and a DFL-head teacher, `dfl`) has the DFL head: its weights are fabricated over the model's own keys."""
    from yolov6_b200 import configs
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    spec = cfg
    if distill_ns or dfl:
        spec = configs.get_config(cfg)
        spec["head"]["use_dfl"], spec["head"]["reg_max"] = True, 16
    m = build_model(spec, 80, dev, fuse_ab=fuse_ab, distill_ns=distill_ns)
    if distill_ns or dfl:
        m.load_state_dict(fab.fabricate_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=0))
    elif cfg in GOLDEN_KEYS:
        m.load_state_dict(fab.fabricate_state_dict(golden_keys(cfg + ("_fuseab" if fuse_ab else "")), seed=0))
    else:
        randomize_(m, seed=0)
    return m


@functools.lru_cache(maxsize=1)
def _engine(name):
    """The model's training engine, planned at the configuration's shape, and its master weights: the fabricated ones and
    integers in [-2, 2] (use_weights repacks one set or the other)."""
    c = MODELS[name]
    size, batch = c["size"], c["batch"]
    dev = torch.device("cuda:0")
    m = seeded_model(c["cfg"], dev, fuse_ab=c.get("fuse_ab", False), distill_ns=c.get("distill_ns", False))
    m.train()
    eng = m.train_engine()
    eng.external_feat_grads = bool(c.get("feat"))      # before planning, as TrainStep sets it for distill_feat
    x = fab.synthetic_images(batch, size, size, seed=11)
    if c.get("u8"):
        x = (x * 255).round().to(torch.uint8)
    with torch.no_grad():
        eng.forward(x.to(dev))                   # plans the step
    gen = torch.Generator(device=dev).manual_seed(3)
    fl = eng.flat.pflat
    eng.weight_sets = {False: fl.clone(), True: torch.randint(-2, 3, fl.shape, generator=gen, device=dev).to(fl.dtype)}
    eng.weights_now = False
    torch.cuda.synchronize()
    return m, eng


def use_weights(eng, integer):
    """Master weights for the next checks: integers (exact passes) or the fabricated ones (real-valued passes, and the
    BottleRep shortcut weight that bn_bwd reads from the parameter buffer); begin_step repacks them into the forward and
    dgrad layouts and clears the zero arena, which is its rest state."""
    if eng.weights_now is not integer:
        eng.flat.pflat.copy_(eng.weight_sets[integer])
        eng.begin_step()
        torch.cuda.synchronize()
        eng.weights_now = integer


def engine_mem(eng):
    sc = eng.scratch
    named = [("buf", t) for t in eng.bufs] + [("gbuf", t) for t in eng.gbufs] + [("arena", eng.zero_arena)]
    named += [("dc", t) for t in sc.dc] + [("dq", t) for q in sc.quad for t in q] + [("poolscr", t) for p in sc.pool for t in p]
    named += [("stat", t) for t in eng.stat_out.values()] + [("coef", t) for t in eng.coef_out.values()]
    named += [("head", t) for t in (eng.cls, eng.reg, eng.grad_cls, eng.grad_reg)] + [("img", eng.x_static)]
    if getattr(eng.g, "distill_ns", False):
        named += [("head", t) for t in (eng.reg_dist, eng.grad_reg_dist)]
    named += [("dl", t) for t in sc.dl]
    named += [("patch", t) for t in getattr(eng, "_stem_patches", ())]
    named += [("raw", br["x"]) for ctx in eng.ctx if ctx and "branches" in ctx for br in ctx["branches"] if br["k"]]
    named += [("qa_t", ctx["t"]) for ctx in eng.ctx if ctx and "t" in ctx]
    if getattr(eng.g, "fuse_ab", False):
        named += [("ab", t) for t in (eng.cls_ab, eng.reg_ab, eng.grad_cls_ab, eng.grad_reg_ab)]
        named += [("ab_raw", raw) for st in eng._ab.values() for raw, _ in st.values()]
    named += [("gflat", eng.flat.gflat), ("param", eng.flat.pflat)]
    return Mem(named)


def dgrad_weights(eng):
    """dgrad weight pointer -> (op index, forward KRSC weight, forward stride)."""
    out = {}
    for i, W in eng.wts.items():
        op = eng.g.ops[i]
        if op.kind == "pred":
            out[W["wt"].data_ptr()] = (i, W["w"], 1)
        elif op.kind == "convT":
            for q in range(4):
                out[W["wt"][q].data_ptr()] = (i, W["w"][q], 1)
        elif op.kind != "stem":
            for ent in W["br"]:
                for wt in ent.get("wt", []):
                    out[wt.data_ptr()] = (i, ent["w"], op.s)
    return out


def assert_write_view(eng, w, ptr, pitch, c, pixels, what):
    """A launch's output view (ptr, channel pitch, C channels, pixels) is exactly the slice its Write record declares."""
    g = eng.gbufs[w.buf]
    assert ptr == g.data_ptr() + 2 * w.off and pitch == g.shape[3] and c == w.n, f"{what}: output view is not its Write record"
    assert w.full and pixels == g.numel() // g.shape[3], f"{what}: a full Write over part of the pixels"


KINDS = ("conv", "wgrad", "bn_bwd", "stats", "hgp", "pool_bwd", "im2col", "qa_bwd", "abg")


@pytest.mark.parametrize("name", list(MODELS))
def test_every_backward_launch_record_matches_float64_autograd(name):
    from yolov6_b200 import _lib
    from yolov6_b200._lib import DT_F32, DT_U8
    t0 = time.time()
    m, eng = _engine(name)
    lib, h, sp = eng.lib, eng.h, _lib.stream_ptr()
    mem = engine_mem(eng)
    poison(mem)
    ops = eng.g.ops
    gen = torch.Generator(device="cuda").manual_seed(20261015)
    worst = {k: 0.0 for k in KINDS}
    bn_worst = {}
    seen = {k: set() for k in KINDS}
    total = {k: 0 for k in KINDS}
    exact = {k: 0 for k in ("conv", "wgrad", "stats")}

    def first_time(kind, sig):
        total[kind] += 1
        if sig in seen[kind]:
            return False
        seen[kind].add(sig)
        return True

    def run(kind, what, fn):
        io = IO()
        r = fn(io)
        settle(mem, io.ins, io.outs, f"{name}: {kind} {what}")
        return r

    # dgrads: one group per (op, branch) or per dgrad weight; the four parity launches of a stride-2 3x3 conv together
    wmap = dgrad_weights(eng)
    groups, pools = {}, {}
    for c in eng.bwd_calls:
        if c.kind == "conv":
            d, wr = c.desc, c.writes[0]
            key = wr.group or ("w", d.w)
            groups.setdefault(key, (wr, []))[1].append(d)
        elif c.kind == "pool_bwd":
            pools.setdefault(c.writes[0].buf, []).append(c)
    for key, (meta, descs) in groups.items():
        i, wf, stride = wmap[descs[0].w]
        assert all(wmap[d.w][0] == i for d in descs)
        gbuf = eng.gbufs[meta.buf]
        if not first_time("conv", tuple(signature(d, mem) for d in descs) + (tuple(gbuf.shape),)):
            continue
        for ex in (False, True):
            use_weights(eng, ex)
            r = run("dgrad", ops[i].name, lambda io: check_dgrad(lib, h, sp, mem, descs, wf, stride, gbuf, meta, gen, io, ex))
            assert r <= 1.0, f"{ops[i].name}: dgrad error {r:.2f} x the bar ({len(descs)} launches)"
            worst["conv"] = max(worst["conv"], r)
        exact["conv"] += 1
    for bi, calls in pools.items():
        assert len(calls) == 3
        if not first_time("pool_bwd", tuple(tuple(c.args) for c in calls)):
            continue
        r = run("pool_bwd", bi, lambda io: check_pool_chain(lib, h, sp, eng, mem, calls, gen, io))
        assert r <= 1.0, f"pool backward of buffer {bi}: error {r:.2f} x the bar"
        worst["pool_bwd"] = max(worst["pool_bwd"], r)
    for c in eng.bwd_calls:
        kind, d = c.kind, c.desc
        if kind == "wgrad":
            if first_time(kind, signature(d, mem)):
                for ex in (False, True):
                    r = run(kind, (d.N, d.H, d.W, d.Cin, d.Cout, d.kh), lambda io: check_wgrad(lib, h, sp, mem, d, gen, io, ex))
                    assert r <= 1.0, f"wgrad {(d.N, d.H, d.W, d.Cin, d.Cout, d.kh, d.stride)}: error {r:.2f} x the bar"
                    worst[kind] = max(worst[kind], r)
                exact[kind] += 1
        elif kind == "bn_bwd":
            if first_time(kind, signature(d, mem)):
                for w in c.writes:          # identity-branch dx and the shortcut's dres: exactly their Write records
                    dx_ptrs = [(d.dx[b], d.dx_pitch[b]) for b in range(d.nb) if d.dx[b] == eng.gbufs[w.buf].data_ptr() + 2 * w.off]
                    ptr, pitch = dx_ptrs[0] if dx_ptrs else (d.dres, d.dres_pitch)
                    assert_write_view(eng, w, ptr, pitch, d.C, d.pixels, f"bn_bwd launch {total[kind]}")
                use_weights(eng, False)
                out = run(kind, f"launch {total[kind]} (C={d.C}, nb={d.nb})", lambda io: check_bn_bwd(lib, h, sp, mem, d, gen, io=io))
                for k, r in out.items():
                    bn_worst[k] = max(bn_worst.get(k, 0.0), r)
                    assert r <= 1.0, f"bn_bwd C={d.C} nb={d.nb} act={d.act} res={bool(d.res)}: {k} error {r:.2f} x the bar"
        elif kind == "qa_bwd":
            if first_time(kind, signature(d, mem)):
                w, = c.writes
                assert_write_view(eng, w, d.dx, d.dx_pitch, d.C, d.N * d.H * d.W, f"qa_bwd launch {total[kind]}")
                r = run(kind, f"launch {total[kind]} (C={d.C})", lambda io: check_qa_bwd(lib, h, sp, mem, d, gen, io))
                assert r <= 1.0, f"qa_bwd C={d.C}: error {r:.2f} x the bar"
                worst[kind] = max(worst[kind], r)
        elif kind == "stats":
            if first_time(kind, signature(d, mem)):
                for ex in (False, True):
                    r = run(kind, (d.C, d.pixels), lambda io: check_stats_sums(lib, h, sp, mem, d, gen, io, ex))
                    assert r <= 1.0, f"stats C={d.C} pixels={d.pixels}: error {r:.2f} x the bar"
                    worst[kind] = max(worst[kind], r)
                exact[kind] += 1
        elif kind == "hgp":
            if first_time(kind, (bool(c.args[1]),) + tuple(c.args[2:8])):
                run(kind, c.args[2:8], lambda io: check_hgp(lib, h, sp, mem, c.args, gen, io))
        elif kind == "abg":
            if first_time(kind, tuple(c.args[4:8]) + tuple(c.args[9:13])):
                r = run(kind, c.args[4:8], lambda io: check_abg(lib, h, sp, mem, c.args, gen, io))
                assert r <= 1.0, f"head_ab_grad: error {r:.2f} x the bar"
                worst[kind] = max(worst[kind], r)
        elif kind == "im2col":
            if first_time(kind, tuple(c.args[1:6])):
                x_ptr, x_dt, scale, N, H, W, pp, plo = c.args
                img = eng.x_static
                assert x_ptr == img.data_ptr() and x_dt == (DT_U8 if img.dtype == torch.uint8 else DT_F32)
                patches, lo = eng._stem_patches
                assert pp == patches.data_ptr() and plo == lo.data_ptr()

                def im2col(io):
                    if img.dtype == torch.uint8:
                        img.copy_(torch.randint(0, 256, img.shape, generator=gen, device=img.device, dtype=torch.uint8))
                        other = torch.rand(img.shape, generator=gen, device=img.device)
                        other[0, :, 0, :] = 1.0 / 3.0                  # values with a non-zero bf16 residual
                    else:
                        img.copy_(torch.rand(img.shape, generator=gen, device=img.device))
                        img[0, :, 0, :] = 1.0 / 3.0
                        other = torch.randint(0, 256, img.shape, generator=gen, device=img.device, dtype=torch.uint8)
                    check_im2col(lib, h, sp, x_ptr, img, x_dt, scale, N, H, W, patches, lo, gen, io)
                    check_im2col(lib, h, sp, other.data_ptr(), other, DT_F32 if other.dtype == F32 else DT_U8, scale, N, H, W,
                                 patches, lo, gen, io)
                    return 0.0
                run(kind, (N, H, W), im2col)
    worst["bn_bwd"] = max(bn_worst.values()) if bn_worst else 0.0
    kinds_made = {c.kind for c in eng.bwd_calls}
    for k in KINDS:
        if k in kinds_made:
            assert seen[k], f"no {k} launch checked"
    made = [k for k in KINDS if total[k]]
    print(f"\n{name}: distinct launches checked (of all in the plan): " + ", ".join(f"{k} {len(seen[k])}/{total[k]}" for k in made))
    print(f"{name}: exact integer passes (error 0): " + ", ".join(f"{k} {v}" for k, v in exact.items())
          + "; worst error / bar of the real-valued passes: "
          + ", ".join(f"{k} {worst[k]:.3f}" for k in made if k not in ("hgp", "im2col"))
          + " (hgp, im2col: bit-exact); bn_bwd by output: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(bn_worst.items()))
          + f"; {time.time() - t0:.1f} s")
    del mem, eng, m
    _engine.cache_clear()
    torch.cuda.empty_cache()

# ---------------------------------------------------------------------------------------------------------------- edges outside the engine's shapes
@pytest.mark.parametrize("nb,ch,pixels,pitch_extra,zeroed", [
    (1, 8, 100003, 8, 1), (2, 48, 50001, 16, 0), (3, 96, 20011, 0, 1), (1, 384, 9001, 64, 0), (2, 1024, 3001, 0, 1),
    (1, 2048, 4001, 8, 0), (3, 384, 12345, 8, 1)])
def test_bn_stats_finalize_matches_batchnorm2d(nb, ch, pixels, pitch_extra, zeroed):
    """yv6_bn_stats_finalize (sums of up to three branches, then mean / invstd / scale / shift and the running statistics in the
    block that finishes last) against float64 sums and nn.BatchNorm2d(eps=1e-3, momentum=0.03) in train mode, with channel
    slices of wider tensors, many blocks, and both a caller-cleared (zeroed = 1) and a self-cleared (zeroed = 0) arena.
    Bars: sums 1e-5 R; mean, invstd, scale, shift and the running statistics follow from the sums' bar through their formulas,
    plus the fp32 rounding of the outputs (2^-22 relative)."""
    from yolov6_b200 import _lib
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(ch + nb)
    d = _lib.BnStatsDesc()
    d.nb, d.C, d.pixels, d.zeroed, d.eps, d.momentum = nb, ch, pixels, zeroed, BN_EPS, 0.03
    keep, xs = [], []
    for b in range(nb):
        pitch = ch + pitch_extra * (b + 1)
        off = pitch_extra * (b + 1) // 2 // 8 * 8
        t = rnd(gen, pixels, pitch, scale=1 + b, shift=2.0 * b).to(dev)
        xs.append(t[:, off:off + ch].cpu().double())
        d.x[b], d.x_pitch[b] = t.data_ptr() + 2 * off, pitch
        gam, bet = torch.rand(ch, generator=gen) + 0.5, torch.randn(ch, generator=gen) * 0.1
        rm, rv = torch.randn(ch, generator=gen) * 0.1, torch.rand(ch, generator=gen) + 0.5
        dt = [v.to(dev) for v in (gam, bet, rm, rv)] + [torch.full((4, ch), float("nan"), device=dev)]
        d.gamma[b], d.beta[b], d.running_mean[b], d.running_var[b], d.stats[b] = (v.data_ptr() for v in dt)
        keep.append((t, dt, (gam, bet, rm, rv)))
    sums = torch.randn(nb * 2 * ch + 2, dtype=F64).to(dev)          # [nb][2][ch] sums, then the counter
    d.sums, d.counter = sums.data_ptr(), sums.data_ptr() + 8 * nb * 2 * ch
    if zeroed:
        sums.zero_()
    check(lib.yv6_bn_stats_finalize(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    got = sums.cpu()[:nb * 2 * ch].view(nb, 2, ch)
    worst = 0.0
    for b in range(nb):
        x = xs[b]
        (gam, bet, rm, rv), dt = keep[b][2], keep[b][1]
        R1, R2 = x.abs().sum(0), (x * x).sum(0)
        worst = max(worst, ratio(got[b, 0], x.sum(0), F32_SUM * R1), ratio(got[b, 1], (x * x).sum(0), F32_SUM * R2))
        bn = torch.nn.BatchNorm2d(ch, eps=BN_EPS, momentum=0.03).double().train()
        with torch.no_grad():
            bn.weight.copy_(gam.double()), bn.bias.copy_(bet.double())
            bn.running_mean.copy_(rm.double()), bn.running_var.copy_(rv.double())
            bn(x.t().reshape(1, ch, pixels, 1))
        mean, var = x.mean(0), x.var(0, unbiased=False)
        inv = 1.0 / torch.sqrt(var + BN_EPS)
        e_mean = F32_SUM * R1 / pixels
        e_var = F32_SUM * (R2 / pixels + 2 * mean.abs() * R1 / pixels)
        e_inv = inv * 0.5 * e_var / (var + BN_EPS)
        sc, g64 = gam.double() * inv, gam.double()
        rel = 2.0 ** -22
        st = dt[4].cpu().double()
        worst = max(worst, ratio(st[0], mean, e_mean + rel * mean.abs()), ratio(st[1], inv, e_inv + rel * inv),
                    ratio(st[2], sc, g64 * e_inv + rel * sc.abs()),
                    ratio(st[3], bet.double() - mean * sc, mean.abs() * g64 * e_inv + sc.abs() * e_mean
                          + rel * (bet.double().abs() + (mean * sc).abs())))
        unb = pixels / (pixels - 1.0)
        worst = max(worst, ratio(dt[2].cpu(), bn.running_mean, 0.03 * e_mean + rel * (rm.double().abs() + 0.03 * mean.abs())),
                    ratio(dt[3].cpu(), bn.running_var, 0.03 * unb * e_var + rel * (rv.double().abs() + 0.03 * unb * var)))
    print(f"bn_stats_finalize nb={nb} ch={ch} pixels={pixels}: worst error / bar {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("ch,nb,act,alpha_dev,caller,pixels,positive", [
    (48, 1, "silu", 0, 1, 20000, 0), (48, 2, "relu", 1, 0, 20000, 1), (64, 2, "relu", 1, 1, 20000, 0), (64, 1, "silu", 0, 0, 9000, 1),
    (96, 3, "relu", 0, 1, 8000, 0), (96, 1, "silu", 1, 1, 8000, 1), (192, 1, "silu", 1, 0, 6000, 0), (192, 2, "relu", 0, 1, 6000, 1),
    (384, 1, "silu", 0, 1, 6000, 0), (384, 2, "relu", 1, 0, 5000, 1), (384, 1, "silu", 1, 1, 7000, 1)])
def test_bn_bwd_shortcut_matches_autograd(ch, nb, act, alpha_dev, caller, pixels, positive):
    """yv6_bn_bwd with a BottleRep shortcut (y = act(sum_b BN_b(x_b)) + alpha * res) at the channel counts whose block is not a
    whole number of warps (48, 96: 252 threads; 192, 384: 240) and at 64 (256) as a control; alpha from the host and from device
    memory; the handle's scratch and a caller arena; many blocks.  With `positive` dY and res are positive, so that dalpha =
    sum dY * res has no cancellation and a lost or doubled part of a warp's partial sum is a large error.  Bars as in the module
    docstring (dalpha 1e-5 of the sum of |dY * res|)."""
    from yolov6_b200 import _lib
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(7 * ch + nb)
    pitch = ch + 16
    named = []

    def t(tag, *shape, dtype=BF16):
        x = torch.zeros(*shape, dtype=dtype, device=dev)
        named.append((tag, x))
        return x

    d = _lib.BnDesc()
    d.nb, d.act, d.C, d.pixels = nb, _lib.ACT_CODES[act], ch, pixels
    stats = t("stat", nb, 4, ch, dtype=F32)
    s2 = t("s2", nb, ch, dtype=F64)
    for b in range(nb):
        xb = t("x", pixels, pitch)
        d.x[b], d.x_pitch[b] = xb.data_ptr() + 16, pitch                 # channel offset 8
        d.mean[b], d.invstd[b], d.scale[b], d.shift[b] = (stats[b, k].data_ptr() for k in range(4))
        d.s2[b] = s2[b].data_ptr()
        dx = t("dx", pixels, ch + 8 * b)
        d.dx[b], d.dx_pitch[b], d.accumulate[b] = dx.data_ptr(), ch + 8 * b, b % 2
    gy, r, gr = t("dy", pixels, pitch), t("res", pixels, pitch), t("dres", pixels, 2 * ch)
    d.dy, d.dy_pitch = gy.data_ptr(), pitch
    d.res, d.res_pitch = r.data_ptr() + 32, pitch                          # channel offset 16
    d.dres, d.dres_pitch, d.dres_assign = gr.data_ptr() + 2 * ch, 2 * ch, int(positive)
    acc = t("acc", 2 + ch, dtype=F64)                                     # dalpha, counter, s1
    d.dalpha, d.counter, d.s1 = acc[0].data_ptr(), acc[1].data_ptr(), acc[2].data_ptr()
    if alpha_dev:
        al = t("param", 4, dtype=F32)
        al.fill_(0.6875)
        d.res_alpha, d.res_alpha_dev = 123.0, al.data_ptr()               # the device value wins
    else:
        d.res_alpha = 0.6875
    if caller:
        work, coef = t("work", nb, ch, dtype=F64), t("coef", nb, 2, ch, dtype=F32)
        d.work, d.coef, d.zeroed = work.data_ptr(), coef.data_ptr(), 1
    out = check_bn_bwd(lib, h, sp, Mem(named), d, gen, positive=bool(positive))
    print(f"bn_bwd ch={ch} nb={nb} {act} alpha_dev={alpha_dev} caller={caller}: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(out.items())))
    for k, v in out.items():
        assert v <= 1.0, f"{k}: error {v:.2f} x the bar"


@pytest.mark.parametrize("N,H,W", [(3, 37, 41), (1, 2, 1), (2, 64, 33)])
def test_stem_im2col_odd_sizes(N, H, W):
    """im2col of the stem (3x3 stride 2, pad 1) at odd and tiny image sizes, fp32 and uint8 images: bit for bit."""
    from yolov6_b200 import _lib
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    gen = torch.Generator().manual_seed(H * W)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    patches = torch.zeros(N, Ho, Wo, 32, dtype=BF16, device="cuda")
    lo = torch.zeros_like(patches)
    img = torch.rand(N, 3, H, W, generator=gen)
    dimg = img.cuda()
    check_im2col(lib, h, sp, dimg.data_ptr(), img, _lib.DT_F32, 1.0 / 255.0, N, H, W, patches, lo, gen)
    img8 = torch.randint(0, 256, (N, 3, H, W), generator=gen, dtype=torch.uint8)
    d8 = img8.cuda()
    check_im2col(lib, h, sp, d8.data_ptr(), img8, _lib.DT_U8, 1.0 / 255.0, N, H, W, patches, lo, gen)
    assert math.isfinite(float(patches.float().sum()))
