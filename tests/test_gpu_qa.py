"""GPU parity of the quantization-aware RepVGG networks (YOLOv6-N / S / M-QA, configs/qarepvgg).

Inference against the reference goldens of tests/golden/make_golden_qa.py (the bars of test_gpu_model_zoo.py); yv6_qa_fwd /
yv6_qa_bwd on their own against float64 torch; training op by op against float64 autograd (the bars and structure of
test_gpu_model_zoo.py::test_train_step_matches_reference_op_by_op) and the CUDA-graph TrainStep against the autograd path.

The 3x3 average pool of the references is a depthwise conv with 1/9 weights (`_avg3`): the same function as
AvgPool2d(3, 1, 1) with count_include_pad, differentiated by the conv's own backward."""
from ctypes import byref

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import golden_npz
from oracle import fabricate as fab
from oracle import loss as oloss
from oracle import qa
from test_gpu_train import _bn_train, _nchw, _q, _rel
from test_model_qa import SIZE, qa_keys, train_sd

pytestmark = pytest.mark.gpu
NAMES = ["yolov6n_qa", "yolov6s_qa", "yolov6m_qa"]


def rel_err(a, b):
    return float((np.abs(a - b) / (1.0 + np.abs(b))).max())


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_eval_matches_reference_golden(name, precision):
    from yolov6_b200.model import build_model
    m = build_model(name, 80, torch.device("cuda:0"))
    m.load_state_dict(fab.fabricate_state_dict(qa_keys(name), seed=0), strict=True)
    m.eval().set_precision(precision)
    x = fab.synthetic_images(2, SIZE, SIZE, seed=0)
    g = golden_npz(f"model_{name}.npz")
    with torch.no_grad():
        out, _ = m(x.cuda())
        cls, reg = m.engine().head_outputs(2, SIZE, SIZE)
    e_out, e_cls, e_reg = rel_err(out.cpu().numpy(), g["eval_out"]), rel_err(cls.cpu().numpy(), g["cls_train"]), rel_err(reg.cpu().numpy(), g["reg_train"])
    print(f"{name} {precision}-mode: out {e_out:.2e} cls {e_cls:.2e} reg {e_reg:.2e}")
    if precision == "fp32":
        assert e_out < 1e-4 and e_cls < 1e-4 and e_reg < 1e-4
    else:
        assert e_out < 6e-2 and e_cls < 6e-2


def _avg3(x):
    """AvgPool2d(3, 1, 1), count_include_pad=True: every window divided by 9."""
    c = x.shape[1]
    return F.conv2d(x, torch.full((c, 1, 3, 3), 1.0 / 9.0, dtype=x.dtype, device=x.device), padding=1, groups=c)


def test_avg3_is_the_reference_average_pool():
    x = torch.randn(2, 5, 7, 9, dtype=torch.float64)
    assert torch.allclose(_avg3(x), F.avg_pool2d(x, 3, 1, 1, count_include_pad=True), atol=1e-14)


# ------------------------------------------------------------------------------------------------------ the kernels alone
def _slice(N, H, W, C, pitch, off, gen, dev):
    buf = torch.randn(N, H, W, pitch, generator=gen).to(torch.bfloat16).to(dev)
    return buf, buf[..., off:off + C]


@pytest.mark.parametrize("C,x_pitch,x_off,identity,avg,accumulate", [
    (64, 64, 0, True, True, False),      # stride 1, QARepVGGBlockV2
    (64, 64, 0, True, False, True),      # v1: identity, no avg
    (48, 48, 0, False, False, False),    # stride 2 / stem: no identity
    (21, 21, 0, True, True, True),       # odd channel count: scalar path
    (40, 96, 32, True, True, False),     # a slice of a wider concat buffer
    (24, 61, 5, True, True, True),       # unaligned slice of an odd pitch
])
def test_qa_kernels_match_float64(C, x_pitch, x_off, identity, avg, accumulate):
    from yolov6_b200 import _lib
    dev = torch.device("cuda:0")
    lib, h = _lib.lib(), _lib.handle(0)
    gen = torch.Generator().manual_seed(C + x_pitch)
    N, H, W = 2, 13, 37
    u = torch.randn(N, H, W, C, generator=gen).to(torch.bfloat16).to(dev)
    v = torch.randn(N, H, W, C, generator=gen).to(torch.bfloat16).to(dev)
    _, x = _slice(N, H, W, C, x_pitch, x_off, gen, dev)
    sc, sh = (torch.randn(C, generator=gen) * 0.5 + 1).to(dev), torch.randn(C, generator=gen).to(dev)
    gam, bet = (torch.rand(C, generator=gen) + 0.5).to(dev), torch.randn(C, generator=gen).to(dev)
    rm, rv = torch.randn(C, generator=gen).to(dev), (torch.rand(C, generator=gen) + 0.5).to(dev)
    rm0, rv0 = rm.clone(), rv.clone()
    t = torch.zeros(N, H, W, C, dtype=torch.bfloat16, device=dev)
    sums = torch.zeros(2, C, dtype=torch.float64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    stats = torch.zeros(4, C, dtype=torch.float32, device=dev)
    d = _lib.QaDesc()
    d.N, d.H, d.W, d.C = N, H, W, C
    d.u, d.u_pitch, d.v, d.v_pitch = u.data_ptr(), C, v.data_ptr(), C
    d.scale_d, d.shift_d = sc.data_ptr(), sh.data_ptr()
    if identity:
        d.x, d.x_pitch = x.data_ptr(), x_pitch
    d.avg = int(avg)
    d.t, d.t_pitch = t.data_ptr(), C
    d.sums, d.counter, d.zeroed, d.eps, d.momentum = sums.data_ptr(), cnt.data_ptr(), 1, 1e-3, 0.03
    d.gamma, d.beta, d.running_mean, d.running_var, d.stats = gam.data_ptr(), bet.data_ptr(), rm.data_ptr(), rv.data_ptr(), stats.data_ptr()
    _lib.check(lib.yv6_qa_fwd(h, byref(d), _lib.stream_ptr()))
    torch.cuda.synchronize()

    x64 = _nchw(x).contiguous()
    ref = _nchw(u) * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1) + _nchw(v)
    if identity:
        ref = ref + x64 + (_avg3(x64) if avg else 0)
    got = _nchw(t)
    assert float((got - ref).abs().max()) <= 1e-2 * (1 + float(ref.abs().max()))
    assert _rel(got, ref) < 5e-3
    # the statistics are those of the stored (rounded) t
    M = N * H * W
    mean, var = got.mean(dim=(0, 2, 3)), got.var(dim=(0, 2, 3), unbiased=False)
    np.testing.assert_allclose(sums[0].cpu().numpy(), got.sum(dim=(0, 2, 3)).cpu().numpy(), rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(sums[1].cpu().numpy(), (got * got).sum(dim=(0, 2, 3)).cpu().numpy(), rtol=1e-5, atol=1e-3)
    inv = 1 / torch.sqrt(var + 1e-3)
    want = torch.stack([mean, inv, gam.double() * inv, bet.double() - mean * gam.double() * inv]).float()
    np.testing.assert_allclose(stats.cpu().numpy(), want.cpu().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(rm.cpu().numpy(), (0.97 * rm0.double() + 0.03 * mean).cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(rv.cpu().numpy(), (0.97 * rv0.double() + 0.03 * var * M / (M - 1)).cpu().numpy(), rtol=1e-5, atol=1e-6)
    if not identity:
        return

    _, dt = _slice(N, H, W, C, x_pitch, x_off, gen, dev)
    gbuf = torch.randn(N, H, W, x_pitch + 3, generator=gen).to(torch.bfloat16).to(dev)
    g0 = gbuf.clone()
    b = _lib.QaDesc()
    b.N, b.H, b.W, b.C, b.avg, b.accumulate = N, H, W, C, int(avg), int(accumulate)
    b.dt, b.dt_pitch = dt.data_ptr(), x_pitch
    b.dx, b.dx_pitch = gbuf[..., x_off:].data_ptr(), x_pitch + 3
    _lib.check(lib.yv6_qa_bwd(h, byref(b), _lib.stream_ptr()))
    torch.cuda.synchronize()
    xr = torch.zeros_like(x64).requires_grad_(True)
    ((xr + (_avg3(xr) if avg else 0)) * _nchw(dt).contiguous()).sum().backward()
    want = xr.grad + (_nchw(g0[..., x_off:x_off + C]) if accumulate else 0)
    e = _rel(_nchw(gbuf[..., x_off:x_off + C]), want)
    assert e < 5e-3, e
    outside = torch.ones(x_pitch + 3, dtype=torch.bool)
    outside[x_off:x_off + C] = False
    assert torch.equal(gbuf[..., outside], g0[..., outside]), "channels outside the slice were written"


# ------------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("name,size,batch", [("yolov6n_qa", 96, 2), ("yolov6m_qa", 64, 2)])
def test_train_step_matches_reference_op_by_op(name, size, batch):
    """The forward against the oracle's bf16-storage train-mode network, then every op of the engine's backward against torch
    autograd in float64 on the engine's own forward tensors (u, v, t, both BatchNorms' statistics) and incoming gradients.
    Bars: 1e-2 relative L2, 3e-2 for the per-channel BatchNorm sums."""
    from yolov6_b200.model import build_model
    dev = torch.device("cuda:0")
    sd = train_sd(name)
    m = build_model(name, 80, dev)
    m.load_state_dict(sd)
    m.train()
    eng = m.train_engine()
    eng.debug = True
    x = fab.synthetic_images(batch, size, size, seed=11)
    xd = x.to(dev)
    g = torch.Generator().manual_seed(5)
    (feats, cls, reg), _ = m(xd)
    wc, wr = torch.randn(cls.shape, generator=g).to(dev), torch.randn(reg.shape, generator=g).to(dev)
    ((cls * wc).sum() + (reg * wr).sum()).backward()
    torch.cuda.synchronize()

    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad(), qa.om.train_mode(), qa.om.bf16_storage():
        ocls, oreg, _ = qa.forward(sd64, qa.CONFIGS[name], x.double(), train_outputs=True)
    e_cls = float((cls.detach().cpu().double() - ocls).pow(2).mean().sqrt())
    e_reg = _rel(reg.detach().cpu(), oreg)
    print(f"{name}: forward vs oracle: cls rms {e_cls:.2e}, reg rel L2 {e_reg:.2e}")
    assert e_cls < 2e-2 and e_reg < 5e-2

    P = dict(m.named_parameters())
    gr = m.graph
    ref_g = [torch.zeros(t.shape, dtype=torch.float64, device=dev) for t in eng.bufs]
    worst = dict(fwd=0.0, dparam=0.0)
    counts = dict(param=0, qa=0, alpha=0, avg=0)
    checked = set()

    def check_param(pname, ref, tol=1e-2):
        got = P[pname].grad
        assert got is not None, f"no gradient for {pname}"
        checked.add(pname)
        if float(ref.norm()) < 1e-9:
            return
        e = _rel(got.reshape(ref.shape), ref)
        worst["dparam"] = max(worst["dparam"], e)
        counts["param"] += 1
        assert e < tol, f"{pname}: gradient rel err {e:.3e}"

    def sl(bufs, t, c=None):
        return bufs[t.buf][..., t.c_off:t.c_off + (c if c is not None else t.c)]

    def leaf(t):
        return _nchw(t).contiguous().requires_grad_(True)

    for i, op in enumerate(gr.ops):
        ctx, dbg = eng.ctx[i], eng.dbg.get(i)
        if op.kind == "pool":
            c = op.cin
            buf = eng.bufs[op.dst.buf]
            ys = [leaf(buf[..., :c])]
            for _ in range(3):
                ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
                ys[-1].retain_grad()
            gd = _nchw(dbg["gdst"])
            (torch.cat(ys, 1) * gd).sum().backward()
            for j in range(3):
                ref_g[op.dst.buf][..., j * c:(j + 1) * c] += (ys[j].grad - gd[:, j * c:(j + 1) * c]).permute(0, 2, 3, 1)
            continue
        src = None if op.kind == "stem" else leaf(sl(eng.bufs, op.src, op.cin))
        if op.kind == "pred":
            which, lvl = op.head
            w = leaf(ctx["w"])
            b = P[op.name + ".bias"].detach().double().requires_grad_(True)
            y = F.conv2d(src, w, b)
            y = torch.sigmoid(y) if which == "cls" else y
            wt = {"cls": wc, "reg": wr}[which]
            lo, hi = eng.offs[lvl], eng.offs[lvl + 1]
            (y.flatten(2).permute(0, 2, 1) * wt[:, lo:hi].double()).sum().backward()
            check_param(op.name + ".weight", w.grad)
            check_param(op.name + ".bias", b.grad)
        elif op.kind == "convT":
            w = P[op.name + ".upsample_transpose.weight"].detach().to(torch.bfloat16).double().requires_grad_(True)
            b = P[op.name + ".upsample_transpose.bias"].detach().double().requires_grad_(True)
            y = F.conv_transpose2d(src, w, b, stride=2)
            (y * _nchw(dbg["gdst"])).sum().backward()
            check_param(op.name + ".upsample_transpose.weight", w.grad)
            check_param(op.name + ".upsample_transpose.bias", b.grad)
        else:
            leaves, raws = [], []
            for br in ctx["branches"]:
                wname = br["prefix"] + (".weight" if op.layout == "qa" and br["k"] == 1 else ".conv.weight")
                if op.kind == "stem":
                    w = P[wname].detach().double().requires_grad_(True)
                    t = F.conv2d(xd.double(), w, stride=2, padding=br["k"] // 2)
                else:
                    w = leaf(br["w"])
                    t = F.conv2d(src, w, stride=op.s, padding=br["k"] // 2)
                t = _q(t)
                assert _rel(_nchw(br["x"]), t.detach()) < 2e-3, f"{br['prefix']}: raw conv"
                leaves.append((wname, w))
                raws.append((br["prefix"], t))
            if op.layout == "qa":
                counts["qa"] += 1
                pd, pp = op.name + ".rbr_dense.bn", op.name + ".bn"
                gd_, bd_, gp_, bp_ = (P[p + s].detach().double().clone().requires_grad_(True) for p in (pd, pp) for s in (".weight", ".bias"))
                leaves += [(pd + ".weight", gd_), (pd + ".bias", bd_), (pp + ".weight", gp_), (pp + ".bias", bp_)]
                u, v = raws[0][1], raws[1][1]
                mu_d = u.detach().mean(dim=(0, 2, 3))
                assert float((ctx["stats_d"][0].double() - mu_d).abs().max()) < 1e-3 * (1 + float(mu_d.abs().max())), f"{op.name}: BN_d mean"
                tt = _bn_train(u, gd_, bd_) + v
                if op.identity:
                    tt = tt + src
                    if op.avg:
                        counts["avg"] += 1
                        tt = tt + _avg3(src)
                e = _rel(_nchw(ctx["t"]), tt.detach())
                assert e < 1e-2, f"{op.name}: t rel err {e:.3e}"
                mu_p = _nchw(ctx["t"]).mean(dim=(0, 2, 3))      # the post-sum statistics are those of the stored t
                assert float((ctx["stats_p"][0].double() - mu_p).abs().max()) < 1e-3 * (1 + float(mu_p.abs().max())), f"{op.name}: BN_p mean"
                z = _bn_train(_q(tt), gp_, bp_)
            else:
                z = 0
                for prefix, t in raws:
                    gam = P[prefix + ".bn.weight"].detach().double().clone().requires_grad_(True)
                    bet = P[prefix + ".bn.bias"].detach().double().clone().requires_grad_(True)
                    leaves += [(prefix + ".bn.weight", gam), (prefix + ".bn.bias", bet)]
                    z = z + _bn_train(t, gam, bet)
            y = torch.relu(z) if op.act == "relu" else (z * torch.sigmoid(z) if op.act == "silu" else z)
            if op.res is not None:
                res = leaf(sl(eng.bufs, op.res, op.cout))
                al = P[op.alpha].detach().double().requires_grad_(True)
                y = y + al * res
                leaves.append((op.alpha, al))
                counts["alpha"] += 1
            e = _rel(_nchw(sl(eng.bufs, op.dst, op.cout)), y.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-2, f"{op.name}: forward rel err {e:.3e}"
            (y * _nchw(dbg["gdst"])).sum().backward()
            for pname, lf in leaves:
                tol = 1e-2 if lf.dim() == 4 else 3e-2
                if op.kind == "stem" and lf.dim() == 4:
                    tol = 2e-2      # see test_gpu_train.py: the image mean cancels in the stem's weight gradient
                check_param(pname, lf.grad, tol)
            if op.res is not None:
                sl(ref_g, op.res, op.cout).add_(res.grad.permute(0, 2, 3, 1))
        if src is not None:
            sl(ref_g, op.src, op.cin).add_(src.grad.permute(0, 2, 3, 1))
    worst_g = 0.0
    for bi, (got, ref) in enumerate(zip(eng.gbufs, ref_g)):
        if float(ref.norm()) == 0:
            continue
        e = _rel(got.float(), ref)
        worst_g = max(worst_g, e)
        assert e < 1e-2, f"buffer {bi} ({gr.bufs[bi].name}): input-gradient rel err {e:.3e}"
    print(f"{name}: {len(gr.ops)} ops, {counts}; worst rel err: forward {worst['fwd']:.2e}, d(param) {worst['dparam']:.2e}, "
          f"d(input) {worst_g:.2e}")
    assert counts["qa"] > 20 and counts["avg"] > 10
    if name == "yolov6m_qa":
        assert counts["alpha"] > 5
    trainable = {k for k, p in P.items() if p.requires_grad}
    assert not (trainable - checked), sorted(trainable - checked)[:5]


def test_train_step_matches_autograd_path():
    """The CUDA-graph TrainStep of YOLOv6-S-QA against the module's autograd path (test_gpu_step.py)."""
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.step import TrainStep
    name = "yolov6s_qa"
    hd = qa.CONFIGS[name]
    B, S = 2, 128
    x = fab.synthetic_images(B, S, S, seed=3).cuda()
    targets = oloss.synthetic_targets(B, seed=4).cuda()

    def make():
        m = build_model(name, 80, torch.device("cuda:0"))
        m.load_state_dict(train_sd(name))
        loss = ComputeLoss(fpn_strides=hd["strides"], num_classes=80, ori_img_size=S, warmup_epoch=hd["atss_warmup_epoch"],
                           use_dfl=hd["use_dfl"], reg_max=hd["reg_max"], iou_type=hd["iou_type"])
        return m.train(), loss

    (m1, c1), (m2, c2) = make(), make()
    preds, _ = m1(x)
    loss, items = c1(preds, targets, 1, 0, S, S)
    loss.backward()
    ref = {n: p.grad.clone() for n, p in m1.named_parameters() if p.grad is not None}
    step = TrainStep(m2, c2, B, S, S, in_dtype=torch.float32, max_gt=64, graph=True)
    step.load(x, targets)
    out = step.run(epoch_num=1).clone()
    torch.cuda.synchronize()
    assert not step.overflowed()
    assert abs(float(out[0]) - float(loss)) <= 1e-4 * abs(float(loss)), (float(out[0]), float(loss))
    np.testing.assert_allclose(out[1:4].cpu().numpy(), items.cpu().numpy(), rtol=1e-4, atol=1e-7)
    fl = step.eng.flat
    worst = 0.0
    for n, g in ref.items():
        if float(g.norm()) < 1e-12:
            continue
        e = float((fl.grad_view(n).double() - g.double()).norm() / (g.double().norm() + 1e-30))
        worst = max(worst, e)
        assert e < 5e-3, f"{n}: {e:.3e}"
    assert any(n.endswith(".rbr_1x1.weight") for n in ref) and any(n.endswith(".rbr_dense.bn.weight") for n in ref)
    print(f"{name}: loss {float(loss):.5f}, worst gradient rel err vs autograd path {worst:.2e}")
