"""GPU parity of the training engine (train-form forward + backward through conv / wgrad / BN kernels).

The kernels compute in bf16 (operands and stored activations) with fp32 accumulation, like the
reference's own GPU training which runs convs under fp16 autocast (core/engine.py:150).  The forward
is compared with the oracle's train-mode network (bf16 storage, float64 arithmetic; head outputs
within 5e-2); the backward is compared op by op with torch autograd in float64 (1e-2 relative L2),
see the test's docstring for why.  Measured values are printed."""
import numpy as np
import pytest
import torch

from conftest import golden_keys
from oracle import fabricate as fab
from oracle import model as om

pytestmark = pytest.mark.gpu


def oracle_forward(name, sd, x):
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad(), om.train_mode(), om.bf16_storage():   # same storage precision as the kernels (bf16 in HBM)
        cls, reg, _ = om.forward(sd64, om.CONFIGS[name], x.double(), train_outputs=True)
    return cls, reg


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).double()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _bn_train(t, gamma, beta):
    mu, var = t.mean(dim=(0, 2, 3)), t.var(dim=(0, 2, 3), unbiased=False)
    sc = gamma / torch.sqrt(var + 1e-3)
    return t * sc.view(1, -1, 1, 1) + (beta - mu * sc).view(1, -1, 1, 1)


def _q(t):
    """bf16 storage of an intermediate with a straight-through gradient (what the kernels write to HBM)."""
    return t + (t.to(torch.bfloat16).double() - t).detach()


@pytest.mark.parametrize("name,size,batch,variant", [("yolov6n", 128, 4, ""), ("yolov6s", 96, 2, ""), ("yolov6m", 96, 2, ""),
                                                     ("yolov6l6", 128, 2, ""), ("yolov6n", 128, 2, "fuse_ab"), ("yolov6n", 128, 2, "distill_ns")])
def test_train_step_matches_reference_op_by_op(name, size, batch, variant):
    """Forward against the oracle's train-mode network; backward op by op.

    Train-mode BatchNorm over randomly initialised weights is chaotic: the float64 oracle and the same oracle
    with bf16 storage already disagree on parameter gradients with cosine ~0.3 (measured, DESIGN.md), so an
    end-to-end gradient comparison measures rounding noise, not the kernels.  Instead every op of the
    engine's backward pass is checked against torch autograd (float64, on the engine's own forward
    tensors and incoming gradient): parameter gradients, the forward value, and -- summed over all
    consumers of a tensor -- the input gradients.  Bars: 1e-2 relative L2 (bf16 gradient storage), 3e-2 for
    the per-channel BatchNorm sums."""
    import torch.nn.functional as F
    from yolov6_b200.model import build_model
    dev = torch.device("cuda:0")
    fuse_ab, distill_ns = variant == "fuse_ab", variant == "distill_ns"
    sd = fab.fabricate_state_dict(golden_keys(name + ("_fuseab" if fuse_ab else "_distill_ns" if distill_ns else "")), seed=0)
    for k in sd:      # batch-stat BN makes the features unit-variance; keep the head logits O(1)
        if (".cls_preds" in k or ".reg_preds" in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
        if k.endswith(".alpha"):
            sd[k] = sd[k] * 0.75
    cfg = name
    if distill_ns:       # the N / S distillation student is configured with a DFL branch (configs/yolov6n.py: "set to True / 16 ...")
        from yolov6_b200 import configs
        cfg = configs.get_config(name)
        cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
    m = build_model(cfg, 80, dev, fuse_ab=fuse_ab, distill_ns=distill_ns)
    m.load_state_dict(sd)
    m.train()
    eng = m.train_engine()
    eng.debug = True
    x = fab.synthetic_images(batch, size, size, seed=11)
    xd = x.to(dev)
    g = torch.Generator().manual_seed(5)
    if fuse_ab:       # anchor-aided branch (effidehead_fuseab.py:94-140): five training outputs, all of them in the scalar
        (feats, cls_ab, reg_ab, cls, reg), _ = m(xd)
    elif distill_ns:  # effidehead_distill_ns.py:104: (x, cls, reg_distri, reg_lrtb)
        (feats, cls, reg_dist, reg), _ = m(xd)
    else:
        (feats, cls, reg), _ = m(xd)
    wc, wr = torch.randn(cls.shape, generator=g).to(dev), torch.randn(reg.shape, generator=g).to(dev)
    L = (cls * wc).sum() + (reg * wr).sum()
    if fuse_ab:
        w1, w2 = torch.randn(cls_ab.shape, generator=g).to(dev), torch.randn(reg_ab.shape, generator=g).to(dev)
        L = L + (cls_ab * w1).sum() + (reg_ab * w2).sum()
    if distill_ns:
        wd = torch.randn(reg_dist.shape, generator=g).to(dev)
        L = L + (reg_dist * wd).sum()
    L.backward()
    torch.cuda.synchronize()
    assert [tuple(f.shape[2:]) for f in feats] == [(size // s, size // s) for s in om.CONFIGS[name]["strides"]]

    # ---- forward vs the oracle (bf16-storage train-mode network, float64 arithmetic)
    if fuse_ab:
        sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
        with torch.no_grad(), om.train_mode(), om.bf16_storage():
            ocls, oreg, _, ocls_ab, oreg_ab = om.forward(sd64, om.CONFIGS[name], x.double(), train_outputs=True, fuse_ab=True)
        e1 = float((cls_ab.detach().cpu().double() - ocls_ab).pow(2).mean().sqrt())
        e2 = _rel(reg_ab.detach().cpu(), oreg_ab)
        print(f"{name} fuse_ab: forward vs oracle: cls_ab rms {e1:.2e}, reg_ab rel L2 {e2:.2e}")
        assert cls_ab.shape == ocls_ab.shape and reg_ab.shape == oreg_ab.shape and e1 < 2e-2 and e2 < 5e-2
    elif distill_ns:
        sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
        with torch.no_grad(), om.train_mode(), om.bf16_storage():
            ocls, oreg, _, odist = om.forward(sd64, dict(om.CONFIGS[name], use_dfl=True, reg_max=16), x.double(), train_outputs=True, distill_ns=True)
        e3 = _rel(reg_dist.detach().cpu(), odist)
        print(f"{name} distill_ns: forward vs oracle: reg_dist rel L2 {e3:.2e}")
        assert reg_dist.shape == odist.shape and e3 < 5e-2
    else:
        ocls, oreg = oracle_forward(name, sd, x)
    # (rounding differences between fp32 and float64 accumulation are amplified layer by layer by the
    # batch-statistics BatchNorm, so this end-to-end bar is an RMS one; each op is checked tightly below)
    e_cls = float((cls.detach().cpu().double() - ocls).pow(2).mean().sqrt())
    e_reg = _rel(reg.detach().cpu(), oreg)
    m_cls = float((cls.detach().cpu().double() - ocls).abs().max())
    print(f"{name}: forward vs oracle: cls rms {e_cls:.2e} (max {m_cls:.2e}), reg rel L2 {e_reg:.2e}")
    assert e_cls < 2e-2 and e_reg < 5e-2

    # ---- backward, op by op
    P = dict(m.named_parameters())
    gr = m.graph
    ref_g = [torch.zeros(t.shape, dtype=torch.float64, device=dev) for t in eng.bufs]
    worst = dict(fwd=0.0, dparam=0.0)
    nparam = 0

    def check_param(pname, ref, tol=1e-2):
        nonlocal nparam
        got = P[pname].grad
        assert got is not None, f"no gradient for {pname}"
        if float(ref.norm()) < 1e-9:
            return
        e = _rel(got.reshape(ref.shape), ref)
        worst["dparam"] = max(worst["dparam"], e)
        nparam += 1
        assert e < tol, f"{pname}: gradient rel err {e:.3e}"

    def sl(bufs, t, c=None):
        return bufs[t.buf][..., t.c_off:t.c_off + (c if c is not None else t.c)]

    for i, op in enumerate(gr.ops):
        ctx, dbg = eng.ctx[i], eng.dbg.get(i)
        if op.kind == "pool":                                   # SPPF / SimSPPF max-pool chain (common.py:104-112)
            c = op.cin
            buf = eng.bufs[op.dst.buf]
            y0 = _nchw(buf[..., :c]).requires_grad_(True)
            ys = [y0]
            for _ in range(3):
                ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
                ys[-1].retain_grad()
            gd = _nchw(dbg["gdst"])
            for j in range(1, 4):
                assert torch.equal(_nchw(buf[..., j * c:(j + 1) * c]), ys[j].detach()), f"{op.name}: pool {j}"
            (torch.cat(ys, 1) * gd).sum().backward()
            for j in range(3):                                   # chain contribution = total - what the consumers sent
                ref_g[op.dst.buf][..., j * c:(j + 1) * c] += (ys[j].grad - gd[:, j * c:(j + 1) * c]).permute(0, 2, 3, 1)
            continue
        src = None
        if op.kind != "stem":
            src = _nchw(sl(eng.bufs, op.src, op.cin)).requires_grad_(True)
        if op.kind == "pred" and op.head[0].endswith("_ab"):    # effidehead_fuseab.py:108-121: (b, na, h, w, .) rows, box transform
            which, lvl = op.head
            na = 3
            w = _nchw(ctx["w"]).requires_grad_(True)
            b = P[op.name + ".bias"].detach().double().requires_grad_(True)
            y = F.conv2d(src, w, b)
            B_, _, h_, w_ = y.shape
            lo, hi = na * eng.offs[lvl], na * eng.offs[lvl + 1]
            if which == "cls_ab":
                yy = torch.sigmoid(y).reshape(B_, na, -1, h_, w_).permute(0, 1, 3, 4, 2).flatten(1, 3)
                out, wt = eng.cls_ab, w1
            else:
                r = y.reshape(B_, na, -1, h_, w_).permute(0, 1, 3, 4, 2)
                anc = (torch.tensor(gr.anchors_init[lvl], dtype=torch.float64, device=dev) / gr.strides[lvl]).reshape(1, na, 1, 1, 2)
                yy = torch.cat([r[..., :2], ((r[..., 2:4].sigmoid() * 2) ** 2) * anc], -1).flatten(1, 3)
                out, wt = eng.reg_ab, w2
            worst["fwd"] = max(worst["fwd"], _rel(out[:, lo:hi], yy.detach()))
            assert _rel(out[:, lo:hi], yy.detach()) < 1e-3, op.name
            (yy * wt[:, lo:hi].double()).sum().backward()
            check_param(op.name + ".weight", w.grad)
            check_param(op.name + ".bias", b.grad)
        elif op.kind == "pred":                                 # effidehead.py:79-92 (train branch)
            which, lvl = op.head
            w = _nchw(ctx["w"]).requires_grad_(True)
            b = P[op.name + ".bias"].detach().double().requires_grad_(True)
            y = F.conv2d(src, w, b)
            y = torch.sigmoid(y) if which == "cls" else y
            out, wt = {"cls": (eng.cls, wc), "reg": (eng.reg, wr)}[which] if which != "reg_dist" else (eng.reg_dist, wd)
            lo, hi = eng.offs[lvl], eng.offs[lvl + 1]
            yf = y.flatten(2).permute(0, 2, 1)
            worst["fwd"] = max(worst["fwd"], _rel(out[:, lo:hi], yf.detach()))
            assert _rel(out[:, lo:hi], yf.detach()) < 1e-3, op.name
            (yf * wt[:, lo:hi].double()).sum().backward()
            check_param(op.name + ".weight", w.grad)
            check_param(op.name + ".bias", b.grad)
        elif op.kind == "convT":                                # Transpose, common.py:149-163
            w = P[op.name + ".upsample_transpose.weight"].detach().to(torch.bfloat16).double().requires_grad_(True)
            b = P[op.name + ".upsample_transpose.bias"].detach().double().requires_grad_(True)
            y = F.conv_transpose2d(src, w, b, stride=2)
            e = _rel(_nchw(sl(eng.bufs, op.dst, op.cout)), y.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-2, op.name
            (y * _nchw(dbg["gdst"])).sum().backward()
            check_param(op.name + ".upsample_transpose.weight", w.grad)
            check_param(op.name + ".upsample_transpose.bias", b.grad)
        else:                                                   # ConvModule / RepVGGBlock, common.py:46-49,245-255
            z, leaves = 0, []
            for br in ctx["branches"]:
                if br["k"] == 0:
                    t, pfx = src, br["prefix"]
                else:
                    pfx = br["prefix"] + ".bn"
                    if op.kind == "stem":                       # fp32 weights, fp32 image
                        w = P[br["prefix"] + ".conv.weight"].detach().double().requires_grad_(True)
                        t = F.conv2d(xd.double(), w, stride=2, padding=br["k"] // 2)
                    else:
                        w = _nchw(br["w"]).requires_grad_(True)  # the engine's bf16 KRSC weights
                        t = F.conv2d(src, w, stride=op.s, padding=br["k"] // 2)
                    t = _q(t)
                    assert _rel(_nchw(br["x"]), t.detach()) < 2e-3, f"{br['prefix']}: raw conv"
                    leaves.append((br["prefix"] + ".conv.weight", w))
                gam = P[pfx + ".weight"].detach().double().requires_grad_(True)
                bet = P[pfx + ".bias"].detach().double().requires_grad_(True)
                leaves += [(pfx + ".weight", gam), (pfx + ".bias", bet)]
                z = z + _bn_train(t, gam, bet)
            y = torch.relu(z) if op.act == "relu" else (z * torch.sigmoid(z) if op.act == "silu" else z)
            if op.res is not None:                              # BottleRep shortcut, common.py:600-617
                res = _nchw(sl(eng.bufs, op.res, op.cout)).requires_grad_(True)
                al = P[op.alpha].detach().double().requires_grad_(True)
                y = y + al * res
                leaves.append((op.alpha, al))
            e = _rel(_nchw(sl(eng.bufs, op.dst, op.cout)), y.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-2, f"{op.name}: forward rel err {e:.3e}"
            (y * _nchw(dbg["gdst"])).sum().backward()
            for pname, leaf in leaves:   # per-channel BN sums over few pixels feel single relu-mask flips (z ~ 0 in fp32 vs float64)
                tol = 1e-2 if leaf.dim() == 4 else 3e-2
                if op.kind == "stem" and leaf.dim() == 4:
                    # dW = sum_px dc * x with sum_px dc = 0 (BatchNorm backward) and x = 0.5 +- 0.29: the image mean cancels, what is
                    # left competes with the bf16 rounding of dc (2^-9 each, independent) -- measured 0.6e-2 .. 1.1e-2 on 3 x Cout numbers
                    tol = 2e-2
                check_param(pname, leaf.grad, tol)
            if op.res is not None:
                sl(ref_g, op.res, op.cout).add_(res.grad.permute(0, 2, 3, 1))
        if src is not None:
            sl(ref_g, op.src, op.cin).add_(src.grad.permute(0, 2, 3, 1))
    # input gradients: every tensor's gradient is the sum over its consumers
    worst_g = 0.0
    for bi, (got, ref) in enumerate(zip(eng.gbufs, ref_g)):
        if float(ref.norm()) == 0:
            continue
        e = _rel(got.float(), ref)
        worst_g = max(worst_g, e)
        assert e < 1e-2, f"buffer {bi} ({gr.bufs[bi].name}): input-gradient rel err {e:.3e}"
    print(f"{name}: {len(gr.ops)} ops, {nparam} parameter gradients; worst rel err: forward {worst['fwd']:.2e}, "
          f"d(param) {worst['dparam']:.2e}, d(input) {worst_g:.2e}")
    assert nparam > 300
    # every trainable parameter received a gradient; running statistics follow nn.BatchNorm2d (momentum 0.03)
    missing = [k for k, p in P.items() if p.requires_grad and p.grad is None]
    assert not missing, missing[:5]
    rm = dict(m.named_buffers())["backbone.ERBlock_2.0.rbr_dense.bn.running_mean"].cpu() if name != "yolov6m" and name != "yolov6l6" else None
    if rm is not None:
        assert not torch.allclose(rm, sd["backbone.ERBlock_2.0.rbr_dense.bn.running_mean"])


def _wgrad_tiles(N, Ho, Wo, k, s, taps):
    """The pixel tiling yv6_conv_wgrad chooses (csrc/yv6_conv_wgrad.cu): (BW, BH, tiles_w, tiles_h, pixel tiles)."""
    pt = 64 if (k == 3 and taps != 1) else 128
    best = None
    bw = 1
    while bw <= pt:
        bh = pt // bw
        if bw * s <= 256 and bh * s <= 256:
            t = -(-Wo // bw) * -(-Ho // bh) * N
            if best is None or t < best[0] or (t == best[0] and bw > best[1]):
                best = (t, bw, bh)
        bw <<= 1
    t, bw, bh = best
    return bw, bh, -(-Wo // bw), -(-Ho // bh), t


# N, H, W, Cin, x_c_total, x channel offset, Cout, dy_c_total, k, stride, force_taps, force_ksplit (-1: more splits than work,
# so that some get no tile), probe: "rand", or "x:" / "dy:" + where the operand is non-zero (last_row / last_col / last_img /
# last_split = the pixels of the last split) -- the whole result then depends on that edge
WGRAD_CASES = [
    (2, 20, 20, 64, 64, 0, 64, 64, 3, 1, 0, 0, "rand"), (3, 16, 24, 128, 128, 0, 96, 96, 1, 1, 0, 0, "rand"),
    (2, 32, 32, 32, 32, 0, 64, 64, 3, 2, 0, 0, "rand"), (2, 16, 16, 48, 48, 0, 16, 16, 3, 1, 0, 0, "rand"),
    (1, 40, 40, 256, 256, 0, 512, 512, 3, 1, 0, 0, "rand"), (2, 16, 16, 320, 320, 0, 80, 80, 1, 1, 0, 0, "rand"),
    (2, 17, 23, 16, 48, 16, 4, 16, 1, 1, 0, 0, "rand"),                 # the reg_max = 0 head: Cout 4 of a 16-channel dY
    (2, 13, 19, 48, 96, 32, 68, 80, 3, 1, 0, 0, "dy:last_row"),         # the DFL head's Cout 68; ragged tiles
    (2, 13, 19, 48, 96, 32, 68, 80, 3, 1, 1, 0, "x:last_col"),
    (2, 25, 31, 384, 384, 0, 160, 160, 3, 2, 0, 0, "rand"),             # partial second Cout tile, stride 2
    (2, 25, 31, 384, 384, 0, 160, 160, 3, 2, 1, 0, "x:last_row"),
    (2, 25, 31, 320, 640, 320, 96, 128, 1, 2, 0, 0, "dy:last_row"),     # 1x1 stride 2 on channel slices
    (2, 25, 31, 320, 640, 320, 96, 128, 1, 2, 0, -1, "dy:last_split"),
    (3, 21, 21, 64, 64, 0, 80, 80, 3, 1, 0, 1, "dy:last_img"),
    (3, 21, 21, 64, 64, 0, 80, 80, 3, 1, 0, -1, "dy:last_split"),
    (3, 21, 21, 64, 64, 0, 80, 80, 3, 1, 1, -1, "x:last_col"),
    (2, 9, 11, 16, 16, 0, 512, 512, 3, 1, 1, 0, "dy:last_img"),
    (2, 30, 30, 48, 64, 16, 16, 24, 3, 2, 0, -1, "dy:last_split"),
    (1, 40, 40, 384, 384, 0, 4, 16, 1, 1, 0, 0, "x:last_row"),
    (2, 24, 40, 64, 64, 0, 80, 80, 3, 1, 0, 3, "dy:last_col"),
]


def _wgrad_case(N, H, W, Cin, xct, xoff, Cout, dyct, k, s, taps, ksplit, probe):
    """Worst |error| / bar of yv6_conv_wgrad on one case of WGRAD_CASES, onto a random prior and onto zeros."""
    import ctypes as C
    from yolov6_b200 import _lib
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(N * H * W + Cin + Cout)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    xfull = torch.randn(N, H, W, xct, generator=g).to(torch.bfloat16)
    dyfull = torch.randn(N, Ho, Wo, dyct, generator=g).to(torch.bfloat16)
    x, dy = xfull[..., xoff:xoff + Cin], dyfull[..., :Cout]
    if probe != "rand":
        which, where = probe.split(":")
        t = x if which == "x" else dy
        keep = torch.zeros(t.shape[:3], dtype=torch.bool)
        if where == "last_row":
            keep[:, -1] = True
        elif where == "last_col":
            keep[:, :, -1] = True
        elif where == "last_img":
            keep[-1] = True
        else:                                   # the pixel tiles of the last split (dY pixels)
            bw, bh, tw, th, pt = _wgrad_tiles(N, Ho, Wo, k, s, taps)
            ks = min(pt, ksplit if ksplit > 0 else pt - 1)
            per = -(-pt // ks)
            last = (pt - 1) // per
            for p in range(last * per, pt):
                i, r = p // (tw * th), p % (tw * th)
                h0, w0 = (r // tw) * bh, (r % tw) * bw
                keep[i, h0:h0 + bh, w0:w0 + bw] = True
        t.mul_(keep.unsqueeze(-1).to(t.dtype))
        assert float(t.float().abs().sum()) > 0
    ref = torch.nn.grad.conv2d_weight(_nchw(x), (Cout, Cin, k, k), _nchw(dy), stride=s, padding=k // 2).permute(0, 2, 3, 1)
    R = torch.nn.grad.conv2d_weight(_nchw(x).abs(), (Cout, Cin, k, k), _nchw(dy).abs(), stride=s, padding=k // 2).permute(0, 2, 3, 1)
    xd, dyd = xfull.to(dev), dyfull.to(dev)
    d = _lib.WgradDesc()
    d.x, d.N, d.H, d.W, d.Cin, d.x_c_total = xd.data_ptr() + 2 * xoff, N, H, W, Cin, xct
    d.dy, d.Cout, d.dy_c_total = dyd.data_ptr(), Cout, dyct
    d.kh = d.kw = k
    d.stride, d.pad = s, k // 2
    d.force_taps = taps
    if ksplit:
        d.force_ksplit = ksplit if ksplit > 0 else _wgrad_tiles(N, Ho, Wo, k, s, taps)[4] - 1
    prior = torch.randn(Cout, k, k, Cin, generator=g)
    worst = 0.0
    for pr in (prior, torch.zeros_like(prior)):
        dw = pr.to(dev)
        d.dw = dw.data_ptr()
        _lib.check(_lib.lib().yv6_conv_wgrad(_lib.handle(0), C.byref(d), _lib.stream_ptr()))
        err = (dw.cpu().double() - (pr.double() + ref)).abs()
        bound = 1e-5 * (R + pr.double().abs())
        assert bool((err[bound == 0] == 0).all())
        worst = max(worst, float((err / bound.clamp_min(1e-300))[bound > 0].max()))
    return worst


def test_wgrad_kernel_matches_torch():
    """yv6_conv_wgrad against the float64 weight gradient of F.conv2d on the same bf16 operands, for every case of WGRAD_CASES,
    accumulated onto a random prior and onto zeros.  Channels outside the slices hold random data.  Bar per element: 1e-5 of the
    same sum over absolute values (fp32 split-K accumulation of <= 2^11 products per element)."""
    bad = []
    for case in WGRAD_CASES:
        worst = _wgrad_case(*case)
        print(f"wgrad {case}: worst error / bar {worst:.3f}")
        if not worst <= 1.0:
            bad.append((case, round(worst, 2)))
    assert not bad, f"wgrad cases over the bar (case, error / bar): {bad}"


@pytest.mark.parametrize("nb,act", [(1, "silu"), (1, "relu"), (3, "relu"), (2, "relu")])
def test_bn_forward_backward_kernels_match_torch(nb, act):
    """yv6_bn_stats/finalize/apply_fwd and yv6_bn_bwd against torch autograd on the same bf16 inputs."""
    import ctypes as C
    from yolov6_b200 import _lib
    dev = torch.device("cuda:0")
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    g = torch.Generator().manual_seed(nb)
    N, H, W, Cc = 3, 10, 12, 32
    xs = [(torch.randn(N, H, W, Cc, generator=g) * (1 + b) + 0.3 * b).to(torch.bfloat16) for b in range(nb)]
    gam = [torch.rand(Cc, generator=g) + 0.5 for _ in range(nb)]
    bet = [torch.randn(Cc, generator=g) * 0.1 for _ in range(nb)]
    dy = torch.randn(N, H, W, Cc, generator=g).to(torch.bfloat16)
    # torch reference (float64)
    xr = [x.double().requires_grad_(True) for x in xs]
    gr = [t.double().requires_grad_(True) for t in gam]
    br = [t.double().requires_grad_(True) for t in bet]
    z = 0
    for b in range(nb):
        mu, var = xr[b].mean(dim=(0, 1, 2)), xr[b].var(dim=(0, 1, 2), unbiased=False)
        z = z + (xr[b] - mu) / torch.sqrt(var + 1e-3) * gr[b] + br[b]
    y = torch.relu(z) if act == "relu" else z * torch.sigmoid(z)
    (y * dy.double()).sum().backward()
    # kernels
    xd = [x.to(dev) for x in xs]
    gd_, bd_ = [t.to(dev) for t in gam], [t.to(dev) for t in bet]      # keep alive: raw pointers go to the kernels
    sts = []
    for b in range(nb):
        s = torch.empty(2, Cc, dtype=torch.float64, device=dev)
        _lib.check(lib.yv6_bn_stats(h, xd[b].data_ptr(), N * H * W, Cc, Cc, s[0].data_ptr(), s[1].data_ptr(), sp))
        out = torch.empty(4, Cc, dtype=torch.float32, device=dev)
        _lib.check(lib.yv6_bn_finalize(h, s[0].data_ptr(), s[1].data_ptr(), float(N * H * W), gd_[b].data_ptr(),
                                       bd_[b].data_ptr(), 1e-3, 0.03, 0, 0, out[0].data_ptr(), out[1].data_ptr(),
                                       out[2].data_ptr(), out[3].data_ptr(), Cc, sp))
        sts.append((out, s))
    yk = torch.empty(N, H, W, Cc, dtype=torch.bfloat16, device=dev)
    d = _lib.BnDesc()
    d.nb, d.act, d.C, d.pixels = nb, _lib.ACT_CODES[act], Cc, N * H * W
    dxs = [torch.zeros(N, H, W, Cc, dtype=torch.bfloat16, device=dev) for _ in range(nb)]
    sums = torch.empty(4, Cc, dtype=torch.float64, device=dev)
    dyd = dy.to(dev)
    for b in range(nb):
        d.x[b], d.x_pitch[b] = xd[b].data_ptr(), Cc
        d.mean[b], d.invstd[b], d.scale[b], d.shift[b] = (sts[b][0][i].data_ptr() for i in range(4))
        d.s2[b] = sums[1 + b].data_ptr()
        d.dx[b], d.dx_pitch[b], d.accumulate[b] = dxs[b].data_ptr(), Cc, 0
    d.y, d.y_pitch, d.dy, d.dy_pitch, d.s1 = yk.data_ptr(), Cc, dyd.data_ptr(), Cc, sums[0].data_ptr()
    _lib.check(lib.yv6_bn_apply_fwd(h, C.byref(d), sp))
    _lib.check(lib.yv6_bn_bwd(h, C.byref(d), sp))
    assert float((yk.float().cpu().double() - y.detach()).abs().max() / (1 + y.detach().abs().max())) < 1e-2
    for b in range(nb):
        ref = xr[b].grad
        got = dxs[b].float().cpu().double()
        assert float((got - ref).norm() / ref.norm()) < 1e-2, f"dx[{b}]"
        assert float((sums[1 + b].cpu() - gr[b].grad).norm() / gr[b].grad.norm()) < 1e-2, f"dgamma[{b}]"
        assert float((sums[0].cpu() - br[b].grad).norm() / br[b].grad.norm()) < 1e-2, f"dbeta[{b}]"


@pytest.mark.parametrize("epoch", [0, 5])       # ATSS warm-up epochs, then TAL (loss.py:86-123)
def test_training_steps_follow_the_oracle_trajectory(epoch):
    """The reference's inner loop (core/engine.py:142-176: forward -> ComputeLoss -> backward -> SGD step)
    through the drop-in Model / ComputeLoss on one fixed synthetic batch, against the loss trajectory of the
    float64 oracle doing the same steps with torch autograd on CPU (tests/golden/make_train_traj.py).
    Bars: total loss and its three items within 2e-3 relative for the first three steps; 2e-2 (items 5e-2)
    after, where rounding differences have been amplified by batch-statistics BatchNorm and have moved single
    anchor assignments of the discrete assigners (bf16 kernels vs float64)."""
    import json
    import os
    from oracle.loss import synthetic_targets
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "train_traj.json")))
    traj = gold["trajectories"][str(epoch)]
    dev = torch.device("cuda:0")
    m = build_model(gold["name"], 80, dev)
    sd = fab.fabricate_state_dict(golden_keys(gold["name"]), seed=0)
    for k in list(sd):                            # keep the reference's head initialisation (effidehead.py:49-65)
        if k.startswith("detect.") and ("_preds." in k or "proj" in k):
            sd.pop(k)
    m.load_state_dict(sd, strict=False)
    m.train()
    size, batch = gold["size"], gold["batch"]
    x = fab.synthetic_images(batch, size, size, seed=gold["image_seed"]).to(dev)
    targets = synthetic_targets(batch, seed=gold["target_seed"]).to(dev)
    crit = ComputeLoss(num_classes=80, ori_img_size=size, warmup_epoch=4, use_dfl=False, reg_max=0, iou_type="siou")
    opt = torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=gold["lr"], momentum=0.9, nesterov=True)
    for step, ref in enumerate(traj):
        opt.zero_grad(set_to_none=True)
        preds, _featmaps = m(x)                       # core/engine.py:151
        loss, items = crit(preds, targets, epoch, step, size, size)
        loss.backward()
        assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
        opt.step()
        got = float(loss.detach())
        rel = abs(got - ref["loss"]) / ref["loss"]
        print(f"epoch {epoch} step {step}: loss {got:.4f} (oracle {ref['loss']:.4f}, rel {rel:.1e})  items "
              f"{[round(float(v), 4) for v in items]} (oracle {[round(v, 4) for v in ref['items']]})")
        assert rel < (2e-3 if step < 3 else 2e-2)
        for a, b in zip(items, ref["items"]):
            assert abs(float(a) - b) < (2e-3 if step < 3 else 5e-2) * max(1.0, abs(b))


def test_running_statistics_follow_the_reference_update():
    """After one train-mode forward the BatchNorm running statistics equal what the reference model holds after the
    same forward (momentum 0.03, unbiased variance; torch_utils.py:38-48, golden from tests/golden/make_golden_train.py)."""
    from conftest import golden_npz
    from yolov6_b200.model import build_model
    g = golden_npz("train_yolov6n.npz")
    dev = torch.device("cuda:0")
    sd = fab.fabricate_state_dict(golden_keys("yolov6n"), seed=0)
    for k in sd:
        if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
    m = build_model("yolov6n", 80, dev)
    m.load_state_dict(sd)
    m.train()
    x = fab.synthetic_images(4, 64, 64, seed=7)
    with torch.no_grad():
        (feats, cls, reg), _ = m(x.to(dev))
    bn = str(g["bn_name"])
    bufs = dict(m.named_buffers())
    rm, rv = bufs[bn + ".running_mean"].cpu().double().numpy(), bufs[bn + ".running_var"].cpu().double().numpy()
    old_m, old_v = sd[bn + ".running_mean"].double().numpy(), sd[bn + ".running_var"].double().numpy()
    # compare the UPDATE (new - 0.97 * old = 0.03 * batch statistic), which is what the kernels compute in bf16 / fp32
    upd_m, ref_m = rm - 0.97 * old_m, g["running_mean"] - 0.97 * old_m
    upd_v, ref_v = rv - 0.97 * old_v, g["running_var"] - 0.97 * old_v
    assert np.abs(upd_m - ref_m).max() <= 2e-2 * np.abs(ref_m).max()
    assert np.abs(upd_v - ref_v).max() <= 2e-2 * np.abs(ref_v).max()
    assert int(bufs[bn + ".num_batches_tracked"]) == int(sd[bn + ".num_batches_tracked"]) + 1
    # head outputs of the same forward against the reference's (bf16 kernels vs float64: RMS bar, see the test above)
    assert float(np.sqrt(np.mean((cls.cpu().double().numpy() - g["cls"]) ** 2))) < 2e-2
