"""GPU parity of the rest of the reference's released detectors: YOLOv6-L, -N6, -S6, -M6 and the MBLA models.

Inference against the reference goldens of tests/golden/make_golden_zoo.py (the bars of test_gpu_model.py and
test_gpu_configs.py); training of YOLOv6-N6 (EfficientRep6 / RepBiFPANNeck6) and YOLOv6-S-MBLA (MBLABlock, BottleRep3
shortcuts, cv1 run as row slices of one parameter) op by op against float64 autograd, with the bars of
test_gpu_train.py::test_train_step_matches_reference_op_by_op, and the CUDA-graph TrainStep against the autograd path."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import golden_npz
from oracle import fabricate as fab
from oracle import loss as oloss
from oracle import zoo
from test_gpu_train import _bn_train, _nchw, _q, _rel
from test_model_zoo import zoo_keys

pytestmark = pytest.mark.gpu
MODELS = {"yolov6l": 64, "yolov6n6": 128, "yolov6s6": 128, "yolov6m6": 128,
          "yolov6s_mbla": 64, "yolov6m_mbla": 64, "yolov6l_mbla": 64, "yolov6x_mbla": 64}
NATIVE = {"yolov6n6": (1, 1280, 32), "yolov6s_mbla": (4, 640, 32)}


def rel_err(a, b):
    return float((np.abs(a - b) / (1.0 + np.abs(b))).max())


def load(name, precision):
    from yolov6_b200.model import build_model
    m = build_model(name, 80, torch.device("cuda:0"))
    m.load_state_dict(fab.fabricate_state_dict(zoo_keys(name), seed=0), strict=True)
    return m.eval().set_precision(precision)


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_eval_matches_reference_golden(name, precision):
    m = load(name, precision)
    size = MODELS[name]
    x = fab.synthetic_images(2, size, size, seed=0)
    g = golden_npz(f"model_{name}.npz")
    with torch.no_grad():
        out, feats = m(x.cuda())
        cls, reg = m.engine().head_outputs(2, size, size)
    e_out, e_cls, e_reg = rel_err(out.cpu().numpy(), g["eval_out"]), rel_err(cls.cpu().numpy(), g["cls_train"]), rel_err(reg.cpu().numpy(), g["reg_train"])
    print(f"{name} {precision}-mode: out {e_out:.2e} cls {e_cls:.2e} reg {e_reg:.2e}")
    if precision == "fp32":
        assert e_out < 1e-4 and e_cls < 1e-4 and e_reg < 1e-4
    else:
        assert e_out < 6e-2 and e_cls < 6e-2
    assert len(feats) == len(zoo.CONFIGS[name]["strides"]) and feats[0].shape[2] == size // 8


@pytest.mark.parametrize("name", list(NATIVE))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_forward_at_native_size_matches_reference(name, precision):
    B, size, step = NATIVE[name]
    g = golden_npz("configs_zoo.npz")
    x = fab.synthetic_images(B, size, size, seed=40)
    assert abs(fab.checksum(x) - float(g[f"{name}_x_checksum"])) <= 1e-9 * abs(float(g[f"{name}_x_checksum"])), "RNG drift"
    m = load(name, precision)
    with torch.no_grad():
        out = m(x.cuda())[0].cpu().double().numpy()
    A = out.shape[1]
    e_rows = rel_err(out[:, ::step], g[f"{name}_rows"].astype(np.float64))
    e_sum = float((np.abs(out.sum(1) - g[f"{name}_colsum"]) / (A + g[f"{name}_abs_colsum"])).max())
    print(f"{name}@{size} {precision}: sampled rows {e_rows:.2e}, column sums {e_sum:.2e}")
    tol = 1e-4 if precision == "fp32" else 6e-2
    assert e_rows < tol and e_sum < tol


def _train_sd(name):
    sd = fab.fabricate_state_dict(zoo_keys(name), seed=0)
    for k in sd:      # batch-stat BN makes the features unit-variance; keep the head logits O(1)
        if (".cls_preds" in k or ".reg_preds" in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
        if k.endswith(".alpha"):
            sd[k] = sd[k] * 0.75
    return sd


@pytest.mark.parametrize("name,size,batch", [("yolov6n6", 128, 2), ("yolov6s_mbla", 96, 2)])
def test_train_step_matches_reference_op_by_op(name, size, batch):
    """The forward against the oracle's bf16-storage train-mode network (RMS bars), then every op of the engine's backward
    against torch autograd in float64 on the engine's own forward tensors and incoming gradients: parameter gradients --
    for a row-sliced op (MBLABlock.cv1), its rows of the parameter's gradient --, BottleRep3's dalpha, the forward value, and
    every activation gradient summed over its consumers.  Bars: 1e-2 relative L2, 3e-2 for the per-channel BatchNorm sums."""
    from yolov6_b200.model import build_model
    dev = torch.device("cuda:0")
    sd = _train_sd(name)
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
    assert [tuple(f.shape[2:]) for f in feats] == [(size // s, size // s) for s in zoo.CONFIGS[name]["strides"]]

    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad(), zoo.om.train_mode(), zoo.om.bf16_storage():
        ocls, oreg, _ = zoo.forward(sd64, zoo.CONFIGS[name], x.double(), train_outputs=True)
    e_cls = float((cls.detach().cpu().double() - ocls).pow(2).mean().sqrt())
    e_reg = _rel(reg.detach().cpu(), oreg)
    print(f"{name}: forward vs oracle: cls rms {e_cls:.2e}, reg rel L2 {e_reg:.2e}")
    assert e_cls < 2e-2 and e_reg < 5e-2

    P = dict(m.named_parameters())
    gr = m.graph
    ref_g = [torch.zeros(t.shape, dtype=torch.float64, device=dev) for t in eng.bufs]
    worst = dict(fwd=0.0, dparam=0.0)
    counts = dict(param=0, alpha=0, row_sliced=0)

    def check_param(pname, ref, rows=None, tol=1e-2):
        got = P[pname].grad
        assert got is not None, f"no gradient for {pname}"
        if rows is not None:
            got = got[rows]
        if float(ref.norm()) < 1e-9:
            return
        e = _rel(got.reshape(ref.shape), ref)
        worst["dparam"] = max(worst["dparam"], e)
        counts["param"] += 1
        assert e < tol, f"{pname}[{rows}]: gradient rel err {e:.3e}"

    def sl(bufs, t, c=None):
        return bufs[t.buf][..., t.c_off:t.c_off + (c if c is not None else t.c)]

    for i, op in enumerate(gr.ops):
        ctx, dbg = eng.ctx[i], eng.dbg.get(i)
        if op.kind == "pool":
            c = op.cin
            buf = eng.bufs[op.dst.buf]
            ys = [_nchw(buf[..., :c]).requires_grad_(True)]
            for _ in range(3):
                ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
                ys[-1].retain_grad()
            gd = _nchw(dbg["gdst"])
            for j in range(1, 4):
                assert torch.equal(_nchw(buf[..., j * c:(j + 1) * c]), ys[j].detach()), f"{op.name}: pool {j}"
            (torch.cat(ys, 1) * gd).sum().backward()
            for j in range(3):
                ref_g[op.dst.buf][..., j * c:(j + 1) * c] += (ys[j].grad - gd[:, j * c:(j + 1) * c]).permute(0, 2, 3, 1)
            continue
        src = None
        if op.kind != "stem":
            src = _nchw(sl(eng.bufs, op.src, op.cin)).requires_grad_(True)
        if op.kind == "pred":
            which, lvl = op.head
            w = _nchw(ctx["w"]).requires_grad_(True)
            b = P[op.name + ".bias"].detach().double().requires_grad_(True)
            y = F.conv2d(src, w, b)
            y = torch.sigmoid(y) if which == "cls" else y
            out, wt = {"cls": (eng.cls, wc), "reg": (eng.reg, wr)}[which]
            lo, hi = eng.offs[lvl], eng.offs[lvl + 1]
            yf = y.flatten(2).permute(0, 2, 1)
            e = _rel(out[:, lo:hi], yf.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-3, op.name
            (yf * wt[:, lo:hi].double()).sum().backward()
            check_param(op.name + ".weight", w.grad)
            check_param(op.name + ".bias", b.grad)
        elif op.kind == "convT":
            w = P[op.name + ".upsample_transpose.weight"].detach().to(torch.bfloat16).double().requires_grad_(True)
            b = P[op.name + ".upsample_transpose.bias"].detach().double().requires_grad_(True)
            y = F.conv_transpose2d(src, w, b, stride=2)
            e = _rel(_nchw(sl(eng.bufs, op.dst, op.cout)), y.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-2, op.name
            (y * _nchw(dbg["gdst"])).sum().backward()
            check_param(op.name + ".upsample_transpose.weight", w.grad)
            check_param(op.name + ".upsample_transpose.bias", b.grad)
        else:
            rows = slice(op.w_row0, op.w_row0 + op.cout) if op.w_rows else None
            counts["row_sliced"] += rows is not None and op.cout < op.w_rows
            z, leaves = 0, []
            for br in ctx["branches"]:
                if br["k"] == 0:
                    t, pfx = src, br["prefix"]
                else:
                    pfx = br["prefix"] + ".bn"
                    if op.kind == "stem":
                        w = P[br["prefix"] + ".conv.weight"].detach().double().requires_grad_(True)
                        t = F.conv2d(xd.double(), w, stride=2, padding=br["k"] // 2)
                    else:
                        w = _nchw(br["w"]).requires_grad_(True)
                        t = F.conv2d(src, w, stride=op.s, padding=br["k"] // 2)
                    t = _q(t)
                    assert _rel(_nchw(br["x"]), t.detach()) < 2e-3, f"{br['prefix']}: raw conv"
                    leaves.append((br["prefix"] + ".conv.weight", w))
                gp, bp = P[pfx + ".weight"].detach().double(), P[pfx + ".bias"].detach().double()
                gam = (gp[rows] if rows is not None else gp).clone().requires_grad_(True)
                bet = (bp[rows] if rows is not None else bp).clone().requires_grad_(True)
                leaves += [(pfx + ".weight", gam), (pfx + ".bias", bet)]
                z = z + _bn_train(t, gam, bet)
            y = torch.relu(z) if op.act == "relu" else (z * torch.sigmoid(z) if op.act == "silu" else z)
            if op.res is not None:                              # BottleRep / BottleRep3 shortcut, common.py:600-631
                res = _nchw(sl(eng.bufs, op.res, op.cout)).requires_grad_(True)
                al = P[op.alpha].detach().double().requires_grad_(True)
                y = y + al * res
                leaves.append((op.alpha, al))
                counts["alpha"] += 1
            e = _rel(_nchw(sl(eng.bufs, op.dst, op.cout)), y.detach())
            worst["fwd"] = max(worst["fwd"], e)
            assert e < 1e-2, f"{op.name}: forward rel err {e:.3e}"
            (y * _nchw(dbg["gdst"])).sum().backward()
            for pname, leaf in leaves:
                tol = 1e-2 if leaf.dim() == 4 else 3e-2
                if op.kind == "stem" and leaf.dim() == 4:
                    tol = 2e-2      # see test_gpu_train.py: the image mean cancels in the stem's weight gradient
                check_param(pname, leaf.grad, rows if pname != op.alpha else None, tol)
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
    assert counts["param"] > 300
    if name.endswith("_mbla"):
        assert counts["alpha"] > 10 and counts["row_sliced"] > 0
    missing = [k for k, p in P.items() if p.requires_grad and p.grad is None]
    assert not missing, missing[:5]


@pytest.mark.parametrize("name,epoch", [("yolov6s_mbla", 1), ("yolov6n6", 0)])
def test_train_step_matches_autograd_path(name, epoch):
    """The CUDA-graph TrainStep against the module's autograd path (test_gpu_step.py).  YOLOv6-N6 runs an ATSS epoch
    (atss_warmup_epoch = 4, configs/yolov6n6.py), YOLOv6-S-MBLA a TAL one."""
    from yolov6_b200.loss import ComputeLoss
    from yolov6_b200.model import build_model
    from yolov6_b200.step import TrainStep
    hd = zoo.CONFIGS[name]
    B, S = 2, 128
    x = fab.synthetic_images(B, S, S, seed=3).cuda()
    targets = oloss.synthetic_targets(B, seed=4).cuda()

    def make():
        sd = fab.fabricate_state_dict(zoo_keys(name), seed=0)
        for k in sd:
            if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
                sd[k] = sd[k] * 0.1
        m = build_model(name, 80, torch.device("cuda:0"))
        m.load_state_dict(sd)
        loss = ComputeLoss(fpn_strides=hd["strides"], num_classes=80, ori_img_size=S, warmup_epoch=hd["atss_warmup_epoch"],
                           use_dfl=hd["use_dfl"], reg_max=hd["reg_max"], iou_type=hd["iou_type"])
        return m.train(), loss

    (m1, c1), (m2, c2) = make(), make()
    preds, _ = m1(x)
    loss, items = c1(preds, targets, epoch, 0, S, S)
    loss.backward()
    ref = {n: p.grad.clone() for n, p in m1.named_parameters() if p.grad is not None}
    step = TrainStep(m2, c2, B, S, S, in_dtype=torch.float32, max_gt=64, graph=True)
    step.load(x, targets)
    out = step.run(epoch_num=epoch).clone()
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
    print(f"{name} epoch {epoch}: loss {float(loss):.5f}, worst gradient rel err vs autograd path {worst:.2e}")
