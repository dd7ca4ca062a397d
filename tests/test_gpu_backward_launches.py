"""Every backward launch of the training engine, run alone on fresh seeded data and checked against float64 autograd on the CPU.

`test_train_step_matches_reference_op_by_op` checks whole buffers at 1e-2 relative L2, which a wrong edge column or a wrong tap
in the border pixels of one dgrad parity does not move.  Here the engine (YOLOv6-N / M / L6) plans a step, and every launch of
its backward call list -- dgrad convs (grouped per op and branch: four parity launches for a 3x3 stride-2 conv, one for 1x1
stride 2), weight gradients, BatchNorm backward (with the BottleRep shortcut), the sums-only statistics of the pred and
ConvTranspose bias gradients, the head-gradient repack, the SPPF max-pool backward chain and the stem im2col -- runs on its own
descriptor: every raw pointer is resolved to the engine tensor it lies in, so offsets and pitches are exactly the engine's.
Launches with the same descriptor signature (fields, and pointer offsets inside their tensors) run once.

Bars are per element and scale with R = the same operation on absolute values (the sum of absolute terms):
  fp32 accumulation (wgrad, BatchNorm sums, dalpha): |got - ref| <= 1e-5 R.  K <= 2^13 products or pixel partials are summed in
    fp32 (per-thread runs of <= ~16 pixels, then float64 or split-K fp32 atomics), which costs a few 2^-24 sqrt(K) R at most;
  bf16 outputs (dgrad, dx, dres): 2^-8 |ref| (one round-to-nearest-even to bf16, 8 significant bits) on top of the fp32 bar;
  exact: the head-gradient repack (g * (s * (1 - s)) in fp32, rounded once) and im2col (fp32 image -> bf16 hi + bf16 lo);
  max-pool backward: sums of <= 25 quantised bf16 values are exact in fp32, so each launch's output is one bf16 rounding of
    the exact sum; the reference rounds each link of the chain the same way and the bar allows one bf16 rounding.
A wrong tap, a lost pixel tile or a doubled half-warp changes elements by O(|ref|), far above these bars.  The printed numbers
are the worst error / bar ratio per launch kind."""
import ctypes as C
import functools
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import golden_keys
from oracle import fabricate as fab

pytestmark = pytest.mark.gpu

MODELS = {"yolov6n": (128, 2), "yolov6m": (96, 2), "yolov6l6": (128, 2)}     # name: (image size, batch)
BN_EPS = 1e-3
F32_SUM = 1e-5           # fp32 accumulation, relative to the sum of absolute terms
BF16_ULP = 2.0 ** -8     # one round-to-nearest-even to bf16 (8 significant bits) moves a value by at most 2^-8 of it
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64


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
    return (torch.randn(*shape, generator=gen, dtype=F64) * scale + shift).to(dtype)


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


def check(lib_rc, lib):
    assert lib_rc == 0, lib.yv6_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------- per-kind checks
def check_dgrad(lib, h, sp, mem, descs, wf, stride, gbuf, off, cin, gen):
    """One op's input gradient: g(src)[..., off:off + cin] (+)= conv2d_input(dc, W) over the launches of `descs` (all read the same
    dc).  Elements outside the slice, and pixels no launch writes, keep the prior bit for bit."""
    d0 = descs[0]
    N, Hd, Wd, Cd, xct = d0.N, d0.H, d0.W, d0.Cin, d0.x_c_total
    assert all(d.x == d0.x for d in descs)
    acc = {bool(d.res) for d in descs}
    assert len(acc) == 1, "launches of one dgrad disagree on accumulate"
    acc = acc.pop()
    dc = rnd(gen, N, Hd, Wd, Cd)
    mem.at(d0.x, BF16, (N, Hd, Wd, Cd), (Hd * Wd * xct, Wd * xct, xct, 1)).copy_(dc)
    prior = rnd(gen, *gbuf.shape)
    gbuf.copy_(prior)
    for d in descs:
        check(lib.yv6_conv_fwd(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    got = gbuf.cpu()
    # which pixels the launches write: element (n, i, j) of launch d sits at d.y + n*s0 + i*s1 + j*s2 (elements)
    n_, hs, ws, gct = gbuf.shape
    written = torch.zeros(n_ * hs * ws, dtype=torch.bool)
    base = gbuf.data_ptr()
    for d in descs:
        oh = d.out_h or (d.H + 2 * d.pad - d.kh) // d.stride + 1
        ow = d.out_w or (d.W + 2 * d.pad - d.kw) // d.stride + 1
        e0 = (d.y - base) // 2 - off
        idx = (e0 + torch.arange(d.N).view(-1, 1, 1) * d.y_img_stride + torch.arange(oh).view(1, -1, 1) * d.y_h_stride
               + torch.arange(ow).view(1, 1, -1) * d.y_w_stride)
        assert bool((idx % gct == 0).all())
        written[(idx // gct).reshape(-1)] = True
    written = written.view(n_, hs, ws, 1)
    co, k, _, ci = wf.shape
    assert ci == cin
    w64 = nchw(wf.cpu()).contiguous()
    dcn = nchw(dc[..., :co])
    gin = torch.nn.grad.conv2d_input((n_, ci, hs, ws), w64, dcn, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    R = torch.nn.grad.conv2d_input((n_, ci, hs, ws), w64.abs(), dcn.abs(), stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    assert not bool(((gin != 0) & ~written).any()), "the launches do not cover every pixel of the input gradient"
    p = prior[..., off:off + cin].double()
    exp = torch.where(written, p * acc + gin, p)
    bound = torch.where(written, BF16_ULP * exp.abs() + F32_SUM * (R + acc * p.abs()), torch.zeros_like(p))
    r = ratio(got[..., off:off + cin], exp, bound)
    outside = torch.ones(gct, dtype=torch.bool)
    outside[off:off + cin] = False
    assert bits_equal(got[..., outside], prior[..., outside]), "dgrad wrote outside its channel slice"
    return r


def wgrad_ref(x, dy, cout, k, stride, pad):
    """dW [Cout][k][k][Cin] of conv2d(x, W) against dy, and the same on absolute values (x, dy: NHWC)."""
    xs, ds = nchw(x), nchw(dy)
    shape = (cout, x.shape[3], k, k)
    ref = torch.nn.grad.conv2d_weight(xs, shape, ds, stride=stride, padding=pad).permute(0, 2, 3, 1)
    R = torch.nn.grad.conv2d_weight(xs.abs(), shape, ds.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return ref, R


def check_wgrad(lib, h, sp, mem, d, gen):
    """dW += wgrad(x, dY) on the descriptor's slices, onto a random prior and onto zeros."""
    N, H, W, Cin, xct, Cout, dct, k = d.N, d.H, d.W, d.Cin, d.x_c_total, d.Cout, d.dy_c_total, d.kh
    Ho, Wo = (H + 2 * d.pad - k) // d.stride + 1, (W + 2 * d.pad - d.kw) // d.stride + 1
    for ptr in (d.x, d.dy):     # whole tensors: channels outside the slices hold data too
        t = mem.base(ptr)
        t.copy_(rnd(gen, *t.shape))
    x = mem.at(d.x, BF16, (N, H, W, Cin), (H * W * xct, W * xct, xct, 1)).cpu()
    dy = mem.at(d.dy, BF16, (N, Ho, Wo, Cout), (Ho * Wo * dct, Wo * dct, dct, 1)).cpu()
    dw = mem.at(d.dw, F32, (Cout, k, k, Cin))
    ref, R = wgrad_ref(x, dy, Cout, k, d.stride, d.pad)
    prior = rnd(gen, Cout, k, k, Cin, dtype=F32)
    worst = 0.0
    for pr in (prior, torch.zeros_like(prior)):
        dw.copy_(pr)
        check(lib.yv6_conv_wgrad(h, C.byref(d), sp), lib)
        torch.cuda.synchronize()
        p = pr.double()
        worst = max(worst, ratio(dw.cpu(), p + ref, F32_SUM * (R + p.abs())))
    return worst


def check_stats_sums(lib, h, sp, mem, d, gen):
    """Sums only (no finalize): per-channel sum and sum of squares of an NHWC slice into a zeroed arena slot."""
    assert d.nb == 1 and not d.stats[0]
    P, Cc, pitch = d.pixels, d.C, d.x_pitch[0]
    t = mem.base(d.x[0])
    t.copy_(rnd(gen, *t.shape))
    x = mem.at(d.x[0], BF16, (P, Cc), (pitch, 1)).cpu().double()
    sums = mem.at(d.sums, F64, (2, Cc))
    cnt = mem.at(d.counter, torch.int32, (1,))
    assert d.zeroed
    sums.zero_()
    cnt.zero_()
    check(lib.yv6_bn_stats_finalize(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()
    got = sums.cpu()
    q = x * x
    return max(ratio(got[0], x.sum(0), F32_SUM * x.abs().sum(0)), ratio(got[1], q.sum(0), F32_SUM * q.sum(0)))


def check_bn_bwd(lib, h, sp, mem, d, gen, positive=False):
    """yv6_bn_bwd on fresh branch inputs with their true batch statistics in the stat slots, against autograd through
    act(sum_b BN_b(x_b)) (+ alpha * res) with batch-statistics BatchNorm.  Returns {output: worst ratio}."""
    nb, Cc, P, act = d.nb, d.C, d.pixels, d.act
    view = lambda ptr, pitch: mem.at(ptr, BF16, (P, Cc), (pitch, 1))     # noqa: E731
    xs, st = [], []
    for b in range(nb):
        x = rnd(gen, P, Cc, scale=1 + b, shift=0.3 * b)
        view(d.x[b], d.x_pitch[b]).copy_(x)
        xs.append(x.double())
    for b in range(nb):
        x = xs[b]
        gam = torch.rand(Cc, generator=gen, dtype=F64) + 0.5
        bet = torch.randn(Cc, generator=gen, dtype=F64) * 0.1
        mean, var = x.mean(0), x.var(0, unbiased=False)
        inv = 1.0 / torch.sqrt(var + BN_EPS)
        vals = [mean, inv, gam * inv, bet - mean * gam * inv]
        for ptr, v in zip((d.mean[b], d.invstd[b], d.scale[b], d.shift[b]), vals):
            mem.at(ptr, F32, (Cc,)).copy_(v.float())
        st.append(dict(gam=gam, bet=bet, mean=mean.float().double(), inv=inv.float().double(), sc=(gam * inv).float().double(),
                       sh=(bet - mean * gam * inv).float().double()))
    dy = torch.randn(P, Cc, generator=gen, dtype=F64)
    if positive:
        dy = dy.abs() + 0.1
    if act == 1:       # relu: where z is within fp32 rounding of 0 the kernel and float64 may disagree on the mask -- no gradient there
        z32 = sum(xs[b] * st[b]["sc"] + st[b]["sh"] for b in range(nb))
        tau = 1e-5 * (sum(st[b]["sh"].abs() for b in range(nb)) + sum((xs[b] * st[b]["sc"]).abs() for b in range(nb)))
        dy[z32.abs() < tau] = 0
    dy = dy.to(BF16)
    view(d.dy, d.dy_pitch).copy_(dy)
    has_res = bool(d.res)
    if has_res:
        res = rnd(gen, P, Cc)
        if positive:
            res = res.abs()
        view(d.res, d.res_pitch).copy_(res)
        alpha = float(mem.at(d.res_alpha_dev, F32, (1,)).item()) if d.res_alpha_dev else float(d.res_alpha)
        dres_prior = rnd(gen, P, Cc)
        view(d.dres, d.dres_pitch).copy_(dres_prior)
    dx_prior = []
    for b in range(nb):
        pr = rnd(gen, P, Cc)
        view(d.dx[b], d.dx_pitch[b]).copy_(pr)
        dx_prior.append(pr)
    # accumulators: a caller arena with zeroed = 1 is cleared by the caller; otherwise the launch clears them (garbage here)
    caller = bool(d.work)
    garbage = lambda t: t.copy_(torch.randn(t.shape, generator=gen, dtype=F64).to(t.dtype))   # noqa: E731
    s1 = mem.at(d.s1, F64, (Cc,))
    s2 = [mem.at(d.s2[b], F64, (Cc,)) for b in range(nb)]
    for t in s2:
        garbage(t)
    da = mem.at(d.dalpha, F64, (1,)) if has_res else None
    if caller:
        work, cnt, coef = mem.at(d.work, F64, (nb, Cc)), mem.at(d.counter, torch.int32, (1,)), mem.at(d.coef, F32, (nb, 2, Cc))
        garbage(coef)
    if caller and d.zeroed:
        for t in [s1, work, cnt] + ([da] if has_res else []):
            t.zero_()
    else:
        for t in [s1] + ([da] if has_res else []) + ([work] if caller else []):
            garbage(t)
    check(lib.yv6_bn_bwd(h, C.byref(d), sp), lib)
    torch.cuda.synchronize()

    # ---- float64 reference
    xr = [x.clone().requires_grad_(True) for x in xs]
    gr = [s["gam"].clone().requires_grad_(True) for s in st]
    br = [s["bet"].clone().requires_grad_(True) for s in st]
    z = 0
    for b in range(nb):
        mu, var = xr[b].mean(0), xr[b].var(0, unbiased=False)
        z = z + (xr[b] - mu) / torch.sqrt(var + BN_EPS) * gr[b] + br[b]
    z.retain_grad()
    y = torch.relu(z) if act == 1 else (z * torch.sigmoid(z) if act == 2 else z)
    if has_res:
        rr = res.double().requires_grad_(True)
        al = torch.tensor(alpha, dtype=F64, requires_grad=True)
        y = y + al * rr
    (y * dy.double()).sum().backward()
    dz = z.grad
    out = {}
    R1 = dz.abs().sum(0)
    S1 = br[0].grad
    out["s1"] = ratio(s1.cpu(), S1, F32_SUM * R1)
    worst_dx, worst_s2 = 0.0, 0.0
    for b in range(nb):
        s = st[b]
        R2 = s["inv"] * ((dz.abs() * xs[b].abs()).sum(0) + s["mean"].abs() * R1)
        S2 = gr[b].grad
        worst_s2 = max(worst_s2, ratio(s2[b].cpu(), S2, F32_SUM * R2))
        Bc = -s["sc"] * s["inv"] * S2 / P
        Cb = -s["sc"] * S1 / P - Bc * s["mean"]
        xhat = (xs[b] - s["mean"]) * s["inv"]
        acc = bool(d.accumulate[b])
        p = dx_prior[b].double() * acc
        Rdx = ((s["sc"] * dz).abs() + Bc.abs() * xs[b].abs() + Cb.abs() + s["sc"].abs() * (R1 + xhat.abs() * R2) / P + p.abs())
        exp = p + xr[b].grad
        worst_dx = max(worst_dx, ratio(view(d.dx[b], d.dx_pitch[b]).cpu(), exp, BF16_ULP * exp.abs() + F32_SUM * Rdx))
        if caller:      # coefficients of the apply pass: the closed form of the kernel's comment on its own sums
            S1k, S2k = s1.cpu(), s2[b].cpu()
            Bk = -s["sc"] * s["inv"] * S2k / P
            Ck = -s["sc"] * S1k / P - Bk * s["mean"]
            cf = coef.cpu().double()
            out["coef"] = max(out.get("coef", 0.0), ratio(cf[b, 0], Bk, 2.0 ** -22 * Bk.abs()),
                              ratio(cf[b, 1], Ck, 2.0 ** -22 * ((s["sc"] * S1k / P).abs() + (Bk * s["mean"]).abs())))
    out["s2"], out["dx"] = worst_s2, worst_dx
    if has_res:
        keep = 0.0 if d.dres_assign else 1.0
        p = dres_prior.double() * keep
        exp = p + rr.grad
        out["dres"] = ratio(view(d.dres, d.dres_pitch).cpu(), exp, BF16_ULP * exp.abs() + F32_SUM * ((alpha * dy.double()).abs() + p.abs()))
        out["dalpha"] = ratio(da.cpu(), al.grad.view(1), F32_SUM * (dy.double() * res.double()).abs().sum().view(1))
    return out


def check_hgp(lib, h, sp, mem, args, gen):
    """dlogit = bf16(g * (s * (1 - s))) (or bf16(g)), repacked to NHWC with zero padded channels: bit for bit."""
    gp, sp_, B, A, ch, off, hw, chp, outp = args
    g = mem.at(gp, F32, (B, A, ch))
    g.copy_(torch.randn(B, A, ch, generator=gen))
    if sp_:
        s = mem.at(sp_, F32, (B, A, ch))
        s.copy_(torch.rand(B, A, ch, generator=gen))
    out = mem.at(outp, BF16, (B, hw, chp))
    out.copy_(rnd(gen, B, hw, chp))
    check(lib.yv6_head_grad_prep(h, gp, sp_, B, A, ch, off, hw, chp, outp, sp), lib)
    torch.cuda.synchronize()
    v = g.cpu()[:, off:off + hw]
    if sp_:
        sv = s.cpu()[:, off:off + hw]
        v = v * (sv * (1 - sv))
    exp = torch.zeros(B, hw, chp, dtype=F32)
    exp[..., :ch] = v
    assert bits_equal(out.cpu(), exp.to(BF16)), "head_grad_prep differs from bf16(g * s * (1 - s))"
    return 0.0


def check_pool_chain(lib, h, sp, eng, calls, gen):
    """The three chained MaxPool2d(5, 1, 2) backward launches of one SPPF against torch's max-pool backward in float64 (scatter to
    the first maximum in row-major window order), on operands quantised to a few levels so that ties are everywhere."""
    a = calls[0][1]
    n, hh, ww, c = a[4], a[5], a[6], a[7]
    bi = calls[0][2]["buf"]
    buf, gbuf = eng.bufs[bi], eng.gbufs[bi]
    ys = [torch.randint(0, 4, (n, c, hh, ww), generator=gen).double()]
    for _ in range(3):
        ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
    for j in range(4):
        buf[..., j * c:(j + 1) * c] = ys[j].permute(0, 2, 3, 1).to(BF16).to(buf.device)
    prior = torch.randint(-3, 4, tuple(gbuf.shape), generator=gen).to(BF16)
    gbuf.copy_(prior)
    G = [nchw(prior[..., j * c:(j + 1) * c]) for j in range(4)]
    for call in calls:
        d = call[1]
        j = call[2]["off"] // c + 1
        assert d[0] == buf.data_ptr() + (j - 1) * c * 2 and d[2] == gbuf.data_ptr() + j * c * 2
        check(lib.yv6_maxpool5_bwd(h, d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], d[8].data_ptr(), d[9], d[10], d[11], sp), lib)
        y = ys[j - 1].clone().requires_grad_(True)
        F.max_pool2d(y, 5, 1, 2).backward(G[j])
        G[j - 1] = (G[j - 1] * d[11] + y.grad).to(BF16).double()
    torch.cuda.synchronize()
    got = gbuf.cpu()
    exp = torch.cat([g.permute(0, 2, 3, 1) for g in G], -1)
    r = ratio(got[..., :4 * c], exp, BF16_ULP * exp.abs())
    assert bits_equal(got[..., 4 * c:], prior[..., 4 * c:])
    return r


def im2col_ref(img, scale):
    """patches [N, Ho, Wo, 32] fp32: column (r*3+s)*3+c = x[n, c, 2ho+r-1, 2wo+s-1] (zero outside), columns 27..31 zero."""
    x = img.float() * torch.tensor(scale, dtype=F32) if img.dtype == torch.uint8 else img.float()
    N, _, H, W = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x, (1, 1, 1, 1))
    v = torch.zeros(N, Ho, Wo, 32, dtype=F32)
    for r in range(3):
        for s in range(3):
            for c in range(3):
                v[..., (r * 3 + s) * 3 + c] = xp[:, c, r:r + 2 * Ho - 1:2, s:s + 2 * Wo - 1:2]
    hi = v.to(BF16)
    return hi, (v - hi.float()).to(BF16)


def check_im2col(lib, h, sp, img_ptr, img_cpu, x_dt, scale, N, H, W, patches, patches_lo, gen):
    patches.copy_(rnd(gen, *patches.shape))
    patches_lo.copy_(rnd(gen, *patches_lo.shape))
    check(lib.yv6_stem_im2col(h, img_ptr, x_dt, C.c_float(scale), N, H, W, patches.data_ptr(), patches_lo.data_ptr(), sp), lib)
    torch.cuda.synchronize()
    hi, lo = im2col_ref(img_cpu, C.c_float(scale).value)
    assert bits_equal(patches.cpu(), hi), "im2col: bf16 patches"
    assert bits_equal(patches_lo.cpu(), lo), "im2col: bf16 residual plane"
    return 0.0


# ---------------------------------------------------------------------------------------------------------------- the engine's launches
@functools.lru_cache(maxsize=1)
def _engine(name):
    from yolov6_b200.model import build_model
    size, batch = MODELS[name]
    dev = torch.device("cuda:0")
    m = build_model(name, 80, dev)
    m.load_state_dict(fab.fabricate_state_dict(golden_keys(name), seed=0))
    m.train()
    eng = m.train_engine()
    with torch.no_grad():
        eng.forward(fab.synthetic_images(batch, size, size, seed=11).to(dev))     # plans the step, packs the weights
    torch.cuda.synchronize()
    return eng


def engine_mem(eng):
    dc_pool, pool_scr, dq_pool = eng._keep
    named = [("buf", t) for t in eng.bufs] + [("gbuf", t) for t in eng.gbufs] + [("arena", eng.zero_arena)]
    named += [("dc", t) for t in dc_pool] + [("dq", t) for t in (dq_pool or [])] + [("poolscr", pool_scr)]
    named += [("stat", t) for t in eng.stat_out.values()] + [("coef", t) for t in eng.coef_out.values()]
    named += [("head", t) for t in (eng.cls, eng.reg, eng.grad_cls, eng.grad_reg)] + [("img", eng.x_static)]
    named += [("dl", c[2]) for c in eng.bwd_calls if c[0] == "hgp"]
    named += [("dq", c[1][0]) for c in eng.bwd_calls if c[0] == "copy"]       # ConvTranspose quadrants (earlier, smaller pools)
    named += [("patch", t) for t in getattr(eng, "_stem_patches", ())]
    named += [("raw", br["x"]) for ctx in eng.ctx if ctx and "branches" in ctx for br in ctx["branches"] if br["k"]]
    named += [("param", eng.flat.pflat)]
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


KINDS = ("conv", "wgrad", "bn_bwd", "stats", "hgp", "pool_bwd", "im2col")


@pytest.mark.parametrize("name", list(MODELS))
def test_every_backward_launch_matches_float64_autograd(name):
    from yolov6_b200 import _lib
    from yolov6_b200._lib import DT_F32, DT_U8
    eng = _engine(name)
    lib, h, sp = eng.lib, eng.h, _lib.stream_ptr()
    mem = engine_mem(eng)
    ops = eng.g.ops
    gen = torch.Generator().manual_seed(20261015)
    worst = {k: 0.0 for k in KINDS}
    bn_worst = {}
    seen = {k: set() for k in KINDS}
    total = {k: 0 for k in KINDS}

    def first_time(kind, sig):
        total[kind] += 1
        if sig in seen[kind]:
            return False
        seen[kind].add(sig)
        return True

    # dgrads: one group per (op, branch) or per dgrad weight; the four parity launches of a stride-2 3x3 conv together
    wmap = dgrad_weights(eng)
    groups, pools = {}, {}
    for c in eng.bwd_calls:
        if c[0] == "conv":
            d, meta = c[1], c[2]
            key = meta.get("group", ("w", d.w))
            groups.setdefault(key, (meta, []))[1].append(d)
        elif c[0] == "pool_bwd":
            pools.setdefault(c[2]["buf"], []).append(c)
    for key, (meta, descs) in groups.items():
        i, wf, stride = wmap[descs[0].w]
        assert all(wmap[d.w][0] == i for d in descs)
        gbuf = eng.gbufs[meta["buf"]]
        if not first_time("conv", tuple(signature(d, mem) for d in descs) + (tuple(gbuf.shape),)):
            continue
        r = check_dgrad(lib, h, sp, mem, descs, wf, stride, gbuf, meta["off"], meta["n"], gen)
        assert r <= 1.0, f"{ops[i].name}: dgrad error {r:.2f} x the bar ({len(descs)} launches)"
        worst["conv"] = max(worst["conv"], r)
    for bi, calls in pools.items():
        assert len(calls) == 3
        if not first_time("pool_bwd", tuple(tuple(x if not torch.is_tensor(x) else None for x in c[1]) for c in calls)):
            continue
        r = check_pool_chain(lib, h, sp, eng, calls, gen)
        assert r <= 1.0, f"pool backward of buffer {bi}: error {r:.2f} x the bar"
        worst["pool_bwd"] = max(worst["pool_bwd"], r)
    for c in eng.bwd_calls:
        kind = c[0]
        if kind == "wgrad":
            d = c[1]
            if first_time(kind, signature(d, mem)):
                r = check_wgrad(lib, h, sp, mem, d, gen)
                assert r <= 1.0, f"wgrad {(d.N, d.H, d.W, d.Cin, d.Cout, d.kh, d.stride)}: error {r:.2f} x the bar"
                worst[kind] = max(worst[kind], r)
        elif kind == "bn_bwd":
            d = c[1]
            if first_time(kind, signature(d, mem)):
                out = check_bn_bwd(lib, h, sp, mem, d, gen)
                for k, r in out.items():
                    bn_worst[k] = max(bn_worst.get(k, 0.0), r)
                    assert r <= 1.0, f"bn_bwd C={d.C} nb={d.nb} act={d.act} res={bool(d.res)}: {k} error {r:.2f} x the bar"
        elif kind == "stats":
            d = c[1]
            if first_time(kind, signature(d, mem)):
                r = check_stats_sums(lib, h, sp, mem, d, gen)
                assert r <= 1.0, f"stats C={d.C} pixels={d.pixels}: error {r:.2f} x the bar"
                worst[kind] = max(worst[kind], r)
        elif kind == "hgp":
            if first_time(kind, (bool(c[1][1]),) + tuple(c[1][2:8])):
                check_hgp(lib, h, sp, mem, c[1], gen)
        elif kind == "im2col":
            if first_time(kind, tuple(c[1][1:6])):
                x_ptr, x_dt, scale, N, H, W, pp, plo = c[1]
                assert x_dt == DT_F32 and x_ptr == eng.x_static.data_ptr()
                patches, lo = eng._stem_patches
                assert pp == patches.data_ptr() and plo == lo.data_ptr()
                img = torch.rand(N, 3, H, W, generator=gen)
                img[0, :, 0, :] = 1.0 / 3.0                          # values with a non-zero bf16 residual
                eng.x_static.copy_(img)
                check_im2col(lib, h, sp, x_ptr, img, x_dt, scale, N, H, W, patches, lo, gen)
                img8 = torch.randint(0, 256, (N, 3, H, W), generator=gen, dtype=torch.uint8)
                d8 = img8.cuda()
                check_im2col(lib, h, sp, d8.data_ptr(), img8, DT_U8, scale, N, H, W, patches, lo, gen)
    worst["bn_bwd"] = max(bn_worst.values()) if bn_worst else 0.0
    kinds_made = {c[0] for c in eng.bwd_calls}
    for k in KINDS:
        if k in kinds_made:
            assert seen[k], f"no {k} launch checked"
    print(f"\n{name}: distinct launches checked (of all in the plan): "
          + ", ".join(f"{k} {len(seen[k])}/{total[k]}" for k in KINDS))
    print(f"{name}: worst error / bar: " + ", ".join(f"{k} {worst[k]:.3f}" for k in KINDS if k not in ("hgp", "im2col"))
          + " (hgp, im2col: bit-exact); bn_bwd by output: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(bn_worst.items())))


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
