"""Every launch of ComputeLoss.forward_backward (and of the fuse_ab loss) run alone through the C ABI at the training shapes,
B = 32 images and G = 64 padded gt rows (TrainStep's max_gt), on the cases of test_loss_launch_cases.py, checked against
float64 references of the same operation.

Before each launch every output holds a sentinel (2^100 in float tensors, 0x7eadbeef / 0xab in integer ones) and the
workspace holds 0xff bytes (NaN as float32 and float64, -1 as integers), so a kernel that leaves an element unwritten or
relies on scratch the caller zeroed is caught.  Configurations: YOLOv6-N (plain ltrb, SIoU, TAL), S (plain, GIoU), M (DFL
reg_max 16, GIoU), L6 (four levels, A = 8500, DFL, ATSS warm-up and TAL), N fuse_ab (A = 25200, TAL top-k 26, division
by target_scores_sum whenever it is > 0), N at 640 x 384, and G = 1 and G = 0.

References and bars (per element unless said otherwise):
  targets_pad: gt and gt_count bit for bit against a restatement of loss.py:184-192 that keeps each image's rows in input
    order and drops the rows past G; pad rows [-1, 0, 0, 0, 0].
  box_decode: plain ltrb bit for bit against an fp32 torch restatement; DFL: the float64 softmax expectation d, within
    1e-5 d + 2^-22 (|c| + d) of it in stride units (c the anchor centre), times the stride.
  tal_assign / atss_assign: gt_idx and fg exact against oracle.assign with ties="index" (the kernels' stated lower-index
    rule); norm to rtol 1e-9 (pow may differ by an ulp).  TAL at top-k 13 and 26.
  assign_expand: labels, boxes, the nonzero pattern of the scores and fg exact, score values rtol 1e-9.
  det_loss, class term: the VFL value and gradient of loss.py:205-211 in float64 with the f32 clamps of
    F.binary_cross_entropy restated (log clamped at -100, (1 - p) p clamped at 1e-12, the target score rounded to f32 in
    the BCE).  The kernel evaluates logf, log1pf, p^2, the BCE and its quotient in f32 (each within an ulp or two) and
    rounds the gradient to f32: 2^-20 of the same terms on absolute values, (|dbce w| + |bce dw|) |scale|.
  det_loss, box term, plain ltrb: float64 autograd of oracle.loss.iou_loss on the kernel's f32 box corners (restated bit
    for bit); the kernel differentiates in float64 dual numbers: 1e-9 of the largest gradient of the row plus the f32
    rounding of the output, 2^-24 |ref|.
  det_loss, box term, DFL: float64 autograd of iou_loss on the softmax-expectation boxes plus the DFL cross-entropy terms;
    the kernel's expectation and softmax are f32: 1e-5 of the terms on absolute values, |g_side| p_i (i + d) +
    |c_dfl| (p_i (wl + wr) + [i = tl] wl + [i = tr] wr), plus twice the change of the IoU gradient when the box corners are
    rounded to f32 (a near-degenerate box amplifies that rounding), plus 2^-100 of the coefficients (f32 underflow of p_i).
  background rows of grad_distri exactly 0; out[0..5] against float64 sums: 1e-6 of the sum of |terms| (f32 terms, f64
    accumulation), num_pos exact.
  ab_boxes / ab_boxes_bwd: float64 restatement of loss_fuseab.py:71-76 and of its derivative; four f32 roundings of the
    operands, 2^-21 (|a| + |xo| + |w|) (times the stride for the pixel boxes), and 2^-24 (|g_l| + |g_r|) for the derivative.
A lost row, a wrong class column, a dropped focal-weight gradient, a wrong tie rule or a lost grid-stride iteration moves a
value by O(its size), far above every bar.  The float64 references run in torch on the GPU; assignment oracles on the CPU.

ComputeLossNS's second det_loss call (the IoU term of the lrtb branch against the first call's assignment: weights
(0, 2.5, 0), reg_ch = 4, division by target_scores_sum whenever it is > 0) runs on the assignment of a DFL first call at the
same shapes: the box term under the bars above, out[2] and out[3] exactly 0, and the class gradient it writes all zero.

Then, on whole forward_backward calls: padding G from the largest per-image count up to 64 changes no output bit; two runs
are bit-identical; the lrtb call with reuse= leaves the first call's outputs bit for bit; with an image of 70 boxes gt_count reports the overflow TrainStep.overflowed reads, and that image's
assignment is the oracle's on its first 64 rows in input order.
"""
import ctypes as C
import types

import pytest
import torch

import test_loss_launch_cases as cases
from oracle import assign as oassign
from oracle import loss as oloss

pytestmark = pytest.mark.gpu

B, G = 32, cases.MAX_GT
NC = cases.NC
F32, F64 = torch.float32, torch.float64
SENT = 2.0 ** 100
SENT_I32, SENT_U8 = 0x7EADBEEF, 0xAB
IOU = {"giou": 0, "siou": 1, "ciou": 2, "diou": 3}
W_CLS, W_IOU, W_DFL = 1.0, 2.5, 0.5

# name -> strides, box channels, H, W, assigner, top-k, fuse_ab
CONFIGS = {
    "n": dict(strides=cases.P5, R=4, H=640, W=640, assign="tal", topk=13),
    "s": dict(strides=cases.P5, R=4, H=640, W=640, assign="tal", topk=13),
    "m": dict(strides=cases.P5, R=68, H=640, W=640, assign="tal", topk=13),
    "l6_atss": dict(strides=cases.P6, R=68, H=640, W=640, assign="atss", topk=9),
    "l6_tal": dict(strides=cases.P6, R=68, H=640, W=640, assign="tal", topk=13),
    "n_ab": dict(strides=cases.P5, R=4, H=640, W=640, assign="tal", topk=26, ab=True),
    "n_rect": dict(strides=cases.P5, R=4, H=384, W=640, assign="tal", topk=13),
}
# det_loss variants: config -> [(iou type, norm_gt_zero, grad_scale)]
LOSS_VARIANTS = {
    "n": [("siou", 0, 1.0), ("ciou", 1, 0.37)],
    "s": [("giou", 0, 1.0), ("siou", 0, 2.5), ("ciou", 0, 2.5), ("diou", 1, 2.5)],
    "m": [("giou", 0, 1.0), ("siou", 1, 0.37), ("ciou", 0, 0.37), ("diou", 0, 1.0)],
    "l6_atss": [("giou", 0, 1.0)],
    "l6_tal": [("giou", 0, 0.37)],
    "n_ab": [("giou", 1, 1.0)],
    "n_rect": [("siou", 0, 1.0)],
}


def lib():
    from yolov6_b200 import _lib
    return _lib.lib(), _lib.handle(0), _lib.stream_ptr(), _lib.check


def _p(t):
    return C.c_void_p(t.data_ptr())


def sentinel(shape, dtype):
    v = SENT if dtype.is_floating_point else SENT_I32 if dtype == torch.int32 else SENT_U8
    return torch.full(shape, v, dtype=dtype, device="cuda")


def nan_workspace(nbytes):
    return torch.full((int(nbytes),), 0xFF, dtype=torch.uint8, device="cuda")


def assert_within(got, ref, bar, what):
    got, ref, bar = got.double(), ref.double(), bar.double()
    bad = ~((got - ref).abs() <= bar)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements off, first at {i}: got {got[tuple(i)].item()!r} "
                             f"ref {ref[tuple(i)].item()!r} bar {bar[tuple(i)].item()!r}")


# ------------------------------------------------------------------------------------------------------------- set-up
def anchors_for(cfg):
    from yolov6_b200.assigners import generate_anchors_train
    from yolov6_b200.loss_fuseab import generate_anchors_ab
    sizes = cases.sizes_of(cfg["H"], cfg["W"], cfg["strides"])
    boxes, pts, n_list, st = generate_anchors_train(sizes, cfg["strides"], torch.device("cuda"))
    if cfg.get("ab"):
        pts, st = generate_anchors_ab(sizes, cfg["strides"], torch.device("cuda"))
    return sizes, boxes, pts, n_list, st.reshape(-1).contiguous()


_CASES = {}


def case(name):
    """Inputs of one configuration (cached): targets in TrainStep's layout, head outputs, anchors."""
    if name in _CASES:
        return _CASES[name]
    cfg = CONFIGS[name]
    H, W = cfg["H"], cfg["W"]
    seed = 12 if H != W else 11
    t = cases.coco_like_targets(B, H, W, seed)
    sizes, boxes, pts, n_list, st = anchors_for(cfg)
    ps, pd = cases.adversarial_head(B, sizes, NC, cfg["R"], seed, t, H, W, cfg["strides"])
    if cfg.get("ab"):                         # three anchors per cell: the head's rows repeated per anchor, (level, anchor, pixel)
        ps = torch.cat([ps[:, o:o + n].repeat(1, 3, 1) for o, n in zip(_offsets(sizes), [h * w for h, w in sizes])], 1)
        pd = torch.cat([pd[:, o:o + n].repeat(1, 3, 1) for o, n in zip(_offsets(sizes), [h * w for h, w in sizes])], 1)
    c = types.SimpleNamespace(name=name, cfg=cfg, H=H, W=W, targets=t, rows=cases.trainstep_rows(t, B), sizes=sizes,
                              boxes=boxes, pts=pts, n_list=n_list, st=st, ps=ps.cuda().contiguous(), pd=pd.cuda().contiguous())
    _CASES[name] = c
    return c


def _offsets(sizes):
    o, out = 0, []
    for h, w in sizes:
        out.append(o)
        o += h * w
    return out


# ------------------------------------------------------------------------------------------------------------- launches
def run_targets_pad(rows, Gp, H, W):
    l, h, sp, check = lib()
    tg = rows.cuda().contiguous()
    gt = sentinel((B, max(Gp, 1), 5), F64)              # G = 0 writes no row; the pointer must still be valid
    cnt = sentinel((B,), torch.int32)
    check(l.yv6_targets_pad(h, _p(tg), tg.shape[0], B, Gp, float(W), float(H), _p(gt), _p(cnt), sp))
    if Gp == 0:
        assert (gt == SENT).all(), "targets_pad wrote a row with G = 0"
    return gt[:, :Gp], cnt


def run_decode(c):
    l, h, sp, check = lib()
    A = c.pts.shape[0]
    out = sentinel((B, A, 4), F32)
    check(l.yv6_box_decode(h, _p(c.pd), _p(c.pts), _p(c.st), B, A, c.cfg["R"], 1, _p(out), sp))
    return out


def run_ab_boxes(c):
    l, h, sp, check = lib()
    A = c.pts.shape[0]
    ltrb, px = sentinel((B, A, 4), F32), sentinel((B, A, 4), F32)
    check(l.yv6_ab_boxes(h, _p(c.pd), _p(c.pts), _p(c.st), B, A, _p(ltrb), _p(px), sp))
    return ltrb, px


def run_assign(c, gt, pboxes, topk, kind):
    l, h, sp, check = lib()
    A, Gp = c.pts.shape[0], gt.shape[1]
    mask = (gt[:, :, 1:].sum(-1) > 0).to(torch.uint8).contiguous() if Gp else torch.zeros(B, 1, dtype=torch.uint8, device="cuda")
    gi, fg, norm = sentinel((B, A), torch.int32), sentinel((B, A), torch.uint8), sentinel((B, A), F64)
    ws = nan_workspace(l.yv6_assign_workspace_bytes(B, A, Gp))
    gtp = gt if Gp else torch.zeros(B, 1, 5, dtype=F64, device="cuda")
    if kind == "tal":
        check(l.yv6_tal_assign(h, _p(c.ps), _p(pboxes), _p(c.pts), _p(gtp), _p(mask), B, A, Gp, NC, int(topk), 1.0, 6.0, 1e-9,
                               _p(gi), _p(fg), _p(norm), _p(ws), ws.numel(), sp))
    else:
        lv = (C.c_int32 * len(c.n_list))(*c.n_list)
        check(l.yv6_atss_assign(h, _p(c.boxes), lv, len(c.n_list), _p(gtp), _p(mask), _p(pboxes), B, A, Gp, NC, int(topk),
                                _p(gi), _p(fg), _p(norm), _p(ws), ws.numel(), sp))
    return gi, fg, norm, mask


def run_det_loss(c, distri, gt, gi, fg, norm, iou, ngz, gscale, weights=(W_CLS, W_IOU, W_DFL)):
    from yolov6_b200 import _lib
    l, h, sp, check = lib()
    A, R = distri.shape[1], distri.shape[2]
    gs, gd, out = sentinel(c.ps.shape, F32), sentinel(distri.shape, F32), sentinel((8,), F64)
    ws = nan_workspace(l.yv6_det_loss_workspace_bytes(B, A))
    d = _lib.LossDesc()
    d.pred_scores, d.pred_distri, d.anc_points, d.strides = c.ps.data_ptr(), distri.data_ptr(), c.pts.data_ptr(), c.st.data_ptr()
    d.gt = gt.data_ptr() if gt.shape[1] else 0
    d.gt_idx, d.fg, d.norm = gi.data_ptr(), fg.data_ptr(), norm.data_ptr()
    d.B, d.A, d.G, d.nc, d.reg_ch, d.iou_type = B, A, gt.shape[1], NC, R, IOU[iou]
    d.w_cls, d.w_iou, d.w_dfl = weights
    d.grad_scale = gscale
    d.grad_scores, d.grad_distri, d.out = gs.data_ptr(), gd.data_ptr(), out.data_ptr()
    d.workspace, d.workspace_bytes, d.norm_gt_zero = ws.data_ptr(), ws.numel(), ngz
    check(l.yv6_det_loss(h, C.byref(d), sp))
    torch.cuda.synchronize()
    return gs, gd, out


# ------------------------------------------------------------------------------------------------------------- references
def decode_ref(c):
    """(boxes in pixels as float64 for DFL / exact float32 for plain, DFL bar or None)."""
    pts, st = c.pts.cpu(), c.st.cpu()[:, None]
    ctr = pts / st                                                     # f32 division, as __fdiv_rn
    pd = c.pd.cpu()
    if c.cfg["R"] == 4:
        box = torch.cat([ctr - pd[..., :2], ctr + pd[..., 2:]], -1) * st
        return box, None
    nb = c.cfg["R"] // 4
    d = (torch.softmax(pd.double().view(B, -1, 4, nb), -1) * torch.arange(nb, dtype=F64)).sum(-1)
    c64 = ctr.double()
    box = torch.cat([c64 - d[..., :2], c64 + d[..., 2:]], -1) * st.double()
    cc = torch.cat([c64, c64], -1).abs()
    bar = (1e-5 * d + 2.0 ** -22 * (cc + d)) * st.double()
    return box, bar


def elementwise_iou(g, p, eps=1e-9):
    """oracle.assign.pair_iou on matching rows: g [..., 4] float64, p [..., 4] float32."""
    wh = (torch.minimum(g[..., 2:], p[..., 2:].double()) - torch.maximum(g[..., :2], p[..., :2].double())).clip(0)
    inter = wh[..., 0] * wh[..., 1]
    a1 = (g[..., 2:] - g[..., :2]).clip(0).prod(-1)
    a2 = (p[..., 2:] - p[..., :2]).clip(0).prod(-1).double()
    return inter / (a1 + a2 - inter + eps)


def assign_ref(c, gt, pboxes, topk, kind):
    """(gt_idx, fg, norm, dense oracle outputs) from oracle.assign with the lower-index tie rule, on the CPU."""
    gtc, pb = gt.cpu(), pboxes.cpu()
    mask = (gtc[..., 1:].sum(-1, keepdim=True) > 0).float()
    if kind == "tal":
        r = oassign.tal_assign(c.ps.cpu(), pb, c.pts.cpu(), gtc[..., :1], gtc[..., 1:], mask, topk=topk, num_classes=NC,
                               ties="index")
        norm = torch.where(r[3], r[2].sum(-1), torch.zeros((), dtype=F64))
    else:
        r = oassign.atss_assign(c.boxes.cpu(), c.n_list, gtc[..., :1], gtc[..., 1:], mask, pb, topk=topk, num_classes=NC,
                                ties="index")
        g = torch.gather(gtc[..., 1:], 1, r[4][..., None].expand(-1, -1, 4))
        norm = torch.where(r[3], elementwise_iou(g, pb), torch.zeros((), dtype=F64))
    return r[4], r[3], norm, r


def loss_refs(c, distri, gt, gi, fg, norm, iou, ngz, gscale, weights=(W_CLS, W_IOU, W_DFL)):
    """float64 references of det_loss on the values in memory: (grad_scores, bar), (grad_distri, bar), out[0..5], out bars."""
    W_CLS, W_IOU, W_DFL = weights
    dev = norm.device
    fgb = fg.bool()
    tss = norm[fgb].sum()
    denom = tss if float(tss) > (0.0 if ngz else 1.0) else torch.ones((), dtype=F64, device=dev)
    # class term
    p = c.ps.double()
    lab = torch.full((B, p.shape[1]), -1, dtype=torch.long, device=dev)
    if gt.shape[1]:
        lab_all = torch.gather(gt[..., 0], 1, gi.long().clamp(0, gt.shape[1] - 1)).long()
        lab = torch.where(fgb, lab_all, lab)
    pos = torch.arange(NC, device=dev)[None, None] == lab[..., None]
    q64 = torch.where(pos, norm[..., None], torch.zeros((), dtype=F64, device=dev))
    qf = q64.float().double()
    lp, l1p = torch.log(p).clamp(min=-100), torch.log1p(-p).clamp(min=-100)
    bce = -(qf * lp + (1 - qf) * l1p)
    w = torch.where(pos, q64, 0.75 * p * p)
    dbce = (p - qf) / torch.clamp((1 - p) * p, min=float(torch.tensor(1e-12, dtype=F32)))
    dw = torch.where(pos, torch.zeros((), dtype=F64, device=dev), 1.5 * p)
    gsc = W_CLS * gscale / denom
    g_cls = (dbce * w + bce * dw) * gsc
    bar_cls = 2.0 ** -20 * ((dbce * w).abs() + (bce * dw).abs()) * abs(float(gsc))
    cls_sum, cls_abs = (bce * w).sum(), (bce * w).abs().sum()
    del p, pos, q64, qf, lp, l1p, bce, w, dbce, dw
    # box term on the positive rows
    R = distri.shape[2]
    g_box = torch.zeros(distri.shape, dtype=F64, device=dev)
    bar_box = torch.zeros(distri.shape, dtype=F64, device=dev)
    iou_sum = dfl_sum = iou_abs = dfl_abs = torch.zeros((), dtype=F64, device=dev)
    rows = fgb.nonzero()
    if rows.shape[0]:
        bi, ai = rows[:, 0], rows[:, 1]
        s = c.st[ai]
        ctr = (c.pts[ai].cpu() / s.cpu()[:, None]).to(dev)       # f32 division, as __fdiv_rn
        t = gt[bi, gi[bi, ai].long(), 1:] / s.double()[:, None]
        bw = norm[bi, ai]
        ci = W_IOU * gscale * bw / denom
        reg = distri[bi, ai]
        if R == 4:
            pbx = torch.cat([ctr - reg[:, :2], ctr + reg[:, 2:]], -1).double().requires_grad_(True)   # exact f32 corners
            li = oloss.iou_loss(pbx, t, iou)[:, 0]
            (gc,) = torch.autograd.grad((li * ci).sum(), pbx)
            gl = torch.cat([-gc[:, :2], gc[:, 2:]], -1)
            g_box[bi, ai] = gl
            bar_box[bi, ai] = 2.0 ** -24 * gl.abs() + 1e-9 * gl.abs().amax(-1, keepdim=True)
            iou_sum, iou_abs = (li.detach() * bw).sum(), (li.detach() * bw).abs().sum()
        else:
            nb = R // 4
            reg_max = nb - 1
            lg = reg.double().view(-1, 4, nb).requires_grad_(True)
            sm = torch.softmax(lg, -1)
            d = (sm * torch.arange(nb, dtype=F64, device=dev)).sum(-1)
            d.retain_grad()
            c64 = ctr.double()
            pbx = torch.cat([c64 - d[:, :2], c64 + d[:, 2:]], -1)
            li = oloss.iou_loss(pbx, t, iou)[:, 0]
            tv = torch.cat([c64 - t[:, :2], t[:, 2:] - c64], -1).clamp(0, reg_max - 0.01)
            tl = tv.long()
            wl = (tl + 1).float().double() - tv
            wr = 1 - wl
            lse = torch.logsumexp(lg, -1)
            ce_l = lse - lg.gather(-1, tl[..., None])[..., 0]
            ce_r = lse - lg.gather(-1, (tl + 1)[..., None])[..., 0]
            dfl = (ce_l * wl + ce_r * wr).sum(-1) * 0.25 * bw
            cd = W_DFL * gscale * bw / denom * 0.25
            ((li * ci).sum() + (dfl * (W_DFL * gscale / denom)).sum()).backward()
            g_box[bi, ai] = lg.grad.reshape(-1, R)
            # bar: the terms on absolute values, and the IoU gradient's change when the corners are rounded to f32
            with torch.no_grad():
                ar = torch.arange(nb, dtype=F64, device=dev)
                gl = d.grad                                                           # dL / d(distance), [P, 4]
                pbx32 = torch.cat([ctr - d[:, :2].float(), ctr + d[:, 2:].float()], -1).double()
            pbx32.requires_grad_(True)
            (gc32,) = torch.autograd.grad((oloss.iou_loss(pbx32, t, iou)[:, 0] * ci).sum(), pbx32)
            with torch.no_grad():
                gl32 = torch.cat([-gc32[:, :2], gc32[:, 2:]], -1)
                smd = sm.detach()
                onel = torch.nn.functional.one_hot(tl, nb).double() * wl[..., None]
                oner = torch.nn.functional.one_hot(tl + 1, nb).double() * wr[..., None]
                terms = gl.abs()[..., None] * smd * (ar + d.detach()[..., None]) + \
                    cd.abs()[:, None, None] * (smd * (wl + wr)[..., None] + onel + oner)
                shift = 2 * (gl32 - gl).abs()[..., None] * (smd * (ar - d.detach()[..., None]).abs())
                floor = 2.0 ** -100 * (gl.abs()[..., None] * reg_max + cd.abs()[:, None, None])
                bar_box[bi, ai] = (1e-5 * terms + shift + floor).reshape(-1, R)
            iou_sum, iou_abs = (li.detach() * bw).sum(), (li.detach() * bw).abs().sum()
            dfl_sum, dfl_abs = dfl.detach().sum(), dfl.detach().abs().sum()
    ref_out = torch.stack([W_CLS * cls_sum / denom + W_IOU * iou_sum / denom + (W_DFL * dfl_sum / denom if R > 4 else 0 * dfl_sum),
                           W_IOU * iou_sum / denom, (W_DFL * dfl_sum / denom if R > 4 else 0 * dfl_sum), W_CLS * cls_sum / denom,
                           tss, fgb.sum().double()])
    out_bar = 1e-6 * torch.stack([(W_CLS * cls_abs + W_IOU * iou_abs + W_DFL * dfl_abs) / denom, W_IOU * iou_abs / denom,
                                  W_DFL * dfl_abs / denom, W_CLS * cls_abs / denom, norm[fgb].abs().sum(),
                                  torch.zeros((), dtype=F64, device=dev)])
    return (g_cls, bar_cls), (g_box, bar_box), ref_out, out_bar


# ------------------------------------------------------------------------------------------------------------- the tests
_ASSIGN = {}


def checked_assignment(name, topk=None):
    """targets_pad -> box_decode / ab_boxes -> assignment of one configuration, each launch checked; cached for the loss
    tests (which take the kernels' assignment as their input)."""
    key = (name, topk)
    if key in _ASSIGN:
        return _ASSIGN[key]
    c = case(name)
    cfg = c.cfg
    gt, cnt = run_targets_pad(c.rows, G, c.H, c.W)
    ref_gt, ref_cnt = cases.padded_gt(c.targets, B, G, c.H, c.W)
    assert torch.equal(gt.cpu(), ref_gt), "targets_pad: padded gt"
    assert torch.equal(cnt.cpu(), ref_cnt), "targets_pad: gt_count"
    distri = c.pd
    if cfg.get("ab"):
        ltrb, pboxes = run_ab_boxes(c)
        check_ab_boxes(c, ltrb, pboxes)
        distri = ltrb
    else:
        pboxes = run_decode(c)
        ref, bar = decode_ref(c)
        if bar is None:
            assert torch.equal(pboxes.cpu(), ref), "box_decode (plain ltrb)"
        else:
            assert_within(pboxes.cpu(), ref, bar, "box_decode (DFL)")
    k = topk or cfg["topk"]
    gi, fg, norm, mask = run_assign(c, gt, pboxes, k, cfg["assign"])
    r_gi, r_fg, r_norm, dense = assign_ref(c, gt, pboxes, k, cfg["assign"])
    fg_c = fg.cpu()
    assert torch.equal(fg_c.bool(), r_fg.bool()) and int(fg_c.max()) <= 1, f"{cfg['assign']}: fg"
    assert torch.equal(gi.cpu().long(), r_gi), f"{cfg['assign']}: gt_idx"
    torch.testing.assert_close(norm.cpu(), r_norm, rtol=1e-9, atol=0)
    _ASSIGN[key] = (c, gt, distri, pboxes, gi, fg, norm, dense)
    return _ASSIGN[key]


def check_ab_boxes(c, ltrb, px):
    st = c.st.cpu().double()[:, None]
    a = (c.pts.cpu() / c.st.cpu()[:, None]).double()                   # anchor_points / stride_tensor (f32), loss_fuseab.py:71
    r = c.pd.cpu().double()
    cxy = r[..., :2] + a
    x1y1 = cxy - r[..., 2:] * 0.5
    x2y2 = x1y1 + r[..., 2:]
    mag = a.abs() + r[..., :2].abs() + r[..., 2:].abs()
    bar = 2.0 ** -21 * torch.cat([mag, mag], -1)
    assert_within(px.cpu(), torch.cat([x1y1, x2y2], -1) * st, bar * st, "ab_boxes: boxes in pixels")
    assert_within(ltrb.cpu(), torch.cat([a - x1y1, x2y2 - a], -1), bar, "ab_boxes: ltrb")


@pytest.mark.parametrize("name", list(CONFIGS))
def test_pad_decode_and_assign_launches(name):
    checked_assignment(name)
    if CONFIGS[name]["assign"] == "tal" and CONFIGS[name]["topk"] == 13 and name == "n":
        checked_assignment(name, 26)


@pytest.mark.parametrize("name", ["n", "l6_atss"])
def test_assign_expand_launch(name):
    c, gt, _, _, gi, fg, norm, dense = checked_assignment(name)
    l, h, sp, check = lib()
    A = c.pts.shape[0]
    bg = -1 if c.cfg["assign"] == "tal" else NC
    labels, boxes = sentinel((B, A), torch.int64), sentinel((B, A, 4), F64)
    scores, fgo = sentinel((B, A, NC), F64), sentinel((B, A), torch.bool)
    check(l.yv6_assign_expand(h, _p(gt), _p(gi), _p(fg), _p(norm), B, A, G, NC, bg, _p(labels), _p(boxes), _p(scores),
                              _p(fgo), sp))
    r_labels, r_boxes, _, r_fg, _ = dense
    assert torch.equal(labels.cpu(), r_labels.long()), "assign_expand: labels"
    assert torch.equal(boxes.cpu(), r_boxes), "assign_expand: boxes"
    assert torch.equal(fgo.cpu(), r_fg.bool()), "assign_expand: fg"
    col = r_labels.clamp(0, NC - 1)
    ref = torch.zeros(B, A, NC, dtype=F64).scatter_(2, col[..., None], torch.where(r_fg, norm.cpu(), 0.0)[..., None])
    if bg >= 0:
        ref[~r_fg] = 0
    sc = scores.cpu()
    assert torch.equal(sc != 0, ref != 0), "assign_expand: nonzero pattern of the scores"
    torch.testing.assert_close(sc, ref, rtol=1e-9, atol=0)


LOSS_CASES = [(n, *v) for n, vs in LOSS_VARIANTS.items() for v in vs]


@pytest.mark.parametrize("name,iou,ngz,gscale", LOSS_CASES, ids=[f"{n}-{i}-ngz{z}-gs{g}" for n, i, z, g in LOSS_CASES])
def test_det_loss_launch(name, iou, ngz, gscale):
    c, gt, distri, _, gi, fg, norm, _ = checked_assignment(name)
    gs, gd, out = run_det_loss(c, distri, gt, gi, fg, norm, iou, ngz, gscale)
    (rc, bc), (rb, bb), ro, ob = loss_refs(c, distri, gt, gi, fg, norm, iou, ngz, gscale)
    assert_within(gs, rc, bc, "det_loss: grad_scores")
    assert (gd[~fg.bool()] == 0).all(), "det_loss: background rows of grad_distri"
    assert_within(gd, rb, bb, "det_loss: grad_distri")
    assert_within(out[:6], ro, ob, "det_loss: out[0..5]")
    assert out[5].item() == fg.sum().item()
    if c.cfg.get("ab"):
        l, h, sp, check = lib()
        g_reg = sentinel(gd.shape, F32)
        check(l.yv6_ab_boxes_bwd(h, _p(gd), B * gd.shape[1], _p(g_reg), sp))
        g = gd.double()
        ref = torch.stack([g[..., 2] - g[..., 0], g[..., 3] - g[..., 1], 0.5 * (g[..., 0] + g[..., 2]), 0.5 * (g[..., 1] + g[..., 3])], -1)
        mag = torch.stack([g[..., 0].abs() + g[..., 2].abs(), g[..., 1].abs() + g[..., 3].abs()] * 2, -1)
        assert_within(g_reg, ref, 2.0 ** -24 * mag, "ab_boxes_bwd")


@pytest.mark.parametrize("Gp", [1, 0])
def test_launches_with_one_and_no_gt_rows(Gp):
    c = case("n")
    gt, cnt = run_targets_pad(c.rows, Gp, c.H, c.W)
    ref_gt, ref_cnt = cases.padded_gt(c.targets, B, Gp, c.H, c.W)
    assert torch.equal(gt.cpu(), ref_gt) and torch.equal(cnt.cpu(), ref_cnt)
    pboxes = run_decode(c)
    for kind, k in (("tal", 13), ("atss", 9)):
        gi, fg, norm, _ = run_assign(c, gt, pboxes, k, kind)
        if Gp == 0:
            assert not fg.any() and not gi.any() and not norm.any()
        else:
            r_gi, r_fg, r_norm, _ = assign_ref(c, gt, pboxes, k, kind)
            assert torch.equal(fg.cpu().bool(), r_fg.bool()) and torch.equal(gi.cpu().long(), r_gi)
            torch.testing.assert_close(norm.cpu(), r_norm, rtol=1e-9, atol=0)
        gs, gd, out = run_det_loss(c, c.pd, gt, gi, fg, norm, "siou", 0, 1.0)
        (rc, bc), (rb, bb), ro, ob = loss_refs(c, c.pd, gt, gi, fg, norm, "siou", 0, 1.0)
        assert_within(gs, rc, bc, f"G={Gp} {kind}: grad_scores")
        assert_within(gd, rb, bb, f"G={Gp} {kind}: grad_distri")
        assert_within(out[:6], ro, ob, f"G={Gp} {kind}: out")


def _forward_backward(name, targets, max_gt, epoch=10):
    from yolov6_b200.loss import ComputeLoss
    c = case(name)
    cfg = c.cfg
    cl = ComputeLoss(fpn_strides=cfg["strides"], num_classes=NC, ori_img_size=c.W, warmup_epoch=4, use_dfl=cfg["R"] > 4,
                     reg_max=cfg["R"] // 4 - 1 if cfg["R"] > 4 else 0, iou_type="giou")
    st = cl.forward_backward(c.ps, c.pd, c.sizes, targets.cuda(), epoch, c.H, c.W, max_gt=max_gt)
    torch.cuda.synchronize()
    a = st["assignment"]
    return st, [a.gt_idx.clone(), a.fg.clone(), a.norm.clone(), st["out"].clone(), st["grad_scores"].clone(),
                st["grad_distri"].clone()]


@pytest.mark.parametrize("name,epoch", [("n", 10), ("m", 10), ("l6_atss", 0)])
def test_padding_to_max_gt_changes_nothing_and_runs_repeat(name, epoch):
    c = case(name)
    t = c.targets[c.targets[:, 0] >= 2]                     # no overflow: the largest image has fewer than 64 rows
    largest = int(torch.bincount(t[:, 0].long()).max())
    assert largest < G
    _, small = _forward_backward(name, t, None, epoch)
    st, padded = _forward_backward(name, cases.trainstep_rows(t, B), G, epoch)
    assert st["G"] == G
    for a, b in zip(small, padded):
        assert torch.equal(a, b), "padding the gt rows to max_gt changed an output"
    _, again = _forward_backward(name, cases.trainstep_rows(t, B), G, epoch)
    for a, b in zip(padded, again):
        assert torch.equal(a, b), "two runs differ"


def test_overflowing_image_is_reported_and_truncated_in_input_order():
    from yolov6_b200.step import TrainStep
    c = case("n")
    st, res = _forward_backward("n", c.rows, G)
    assert int(st["gt_count"][0]) == 70
    assert TrainStep.overflowed(types.SimpleNamespace(state=st, max_gt=G))
    first = c.targets[c.targets[:, 0] == 0][:G]             # image 0's first 64 rows, in input order
    gt0 = oloss.preprocess_targets(first, 1, torch.tensor([c.W, c.H, c.W, c.H], dtype=F32))
    assert gt0.shape[1] == G
    pb = run_decode(c)[:1].cpu()
    mask = (gt0[..., 1:].sum(-1, keepdim=True) > 0).float()
    r = oassign.tal_assign(c.ps[:1].cpu(), pb, c.pts.cpu(), gt0[..., :1], gt0[..., 1:], mask, num_classes=NC, ties="index")
    assert torch.equal(res[1][0].cpu().bool(), r[3][0]) and torch.equal(res[0][0].cpu().long(), r[4][0])


def test_det_loss_lrtb_second_call_launch():
    """ComputeLossNS's second yv6_det_loss launch: the lrtb distances scored against the assignment of the DFL first call
    (config m: YOLOv6 P5 anchors at 640, the n / s shapes, DFL reg_max 16), weights (0, 2.5, 0), reg_ch = 4, norm_gt_zero = 1."""
    c, gt, _, _, gi, fg, norm, _ = checked_assignment("m")
    lrtb = case("n").pd                          # plain (l, t, r, b) distances of the same anchors
    assert lrtb.shape[:2] == c.pd.shape[:2] and lrtb.shape[2] == 4
    w = (0.0, W_IOU, 0.0)
    gs, gd, out = run_det_loss(c, lrtb, gt, gi, fg, norm, "giou", 1, 1.0, weights=w)
    (_, _), (rb, bb), ro, ob = loss_refs(c, lrtb, gt, gi, fg, norm, "giou", 1, 1.0, weights=w)
    assert not bool(gs.any()), "lrtb call: the class gradient of a zero class weight"
    assert out[2].item() == 0.0 and out[3].item() == 0.0, "lrtb call: dfl and class terms"
    assert (gd[~fg.bool()] == 0).all(), "lrtb call: background rows of grad_distri"
    assert_within(gd, rb, bb, "lrtb call: grad_distri")
    assert_within(out[:6], ro, ob, "lrtb call: out[0..5]")
    assert out[1].item() > 0 and out[5].item() == fg.sum().item()


def test_lrtb_second_call_leaves_the_first_calls_outputs():
    """Whole calls as ComputeLossNS makes them: the DFL call, then the lrtb call with reuse=; the first call's gradients,
    outputs and assignment are bit for bit what they were, and the second call's class gradient is all zero."""
    from yolov6_b200.loss_distill import ComputeLossNS
    cm, cn = case("m"), case("n")
    cl = ComputeLossNS(num_classes=NC, ori_img_size=cm.W, use_dfl=True, reg_max=16)
    st = cl.forward_backward(cm.ps, cm.pd, cm.sizes, cm.rows.cuda(), 10, cm.H, cm.W, max_gt=G)
    torch.cuda.synchronize()
    a = st["assignment"]
    before = [t.clone() for t in (st["grad_scores"], st["grad_distri"], st["out"], a.gt_idx, a.fg, a.norm, st["gt"])]
    st2 = cl.forward_backward(cm.ps, cn.pd, cm.sizes, None, 10, cm.H, cm.W, reuse=st, weights=(0.0, W_IOU, 0.0))
    torch.cuda.synchronize()
    after = (st["grad_scores"], st["grad_distri"], st["out"], a.gt_idx, a.fg, a.norm, st["gt"])
    for x, y in zip(before, after):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), "the lrtb call changed an output of the first call"
    assert st2["grad_scores"].data_ptr() != st["grad_scores"].data_ptr() and not bool(st2["grad_scores"].any())
    assert st2["out"][2].item() == 0.0 and st2["out"][3].item() == 0.0
