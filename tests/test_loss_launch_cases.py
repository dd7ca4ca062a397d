"""Seeded targets and head outputs at the training shapes that reach the edges of label assignment and of the detection loss,
and proof that they do.  tests/test_gpu_loss_launches.py runs every launch of ComputeLoss.forward_backward on these cases.

`coco_like_targets(B, H, W, seed)` gives [n, 6] rows (img, cls, cx, cy, w, h; x normalised by W, y by H) in a seeded
shuffled order, so that rows of one image are interleaved with the others':
  * counts: image 0 has 70 rows (more than MAX_GT = 64, the TrainStep default), image 1 exactly 64, image 2 none;
  * small boxes (about 40 % under 32^2 px), among them 2-6 px boxes between the stride-8 anchor centres and boxes that hold
    exactly 1 .. 12 stride-8 centres;
  * crowds: identical duplicate rows with the same and with another class, nested boxes;
  * degenerate rows: zero width, zero height, boxes that cross the image edge;
  * ties: images 3 and 4 hold integer-pixel boxes centred on anchor-grid vertices of every stride, all coordinates exact in
    float32 after normalisation, on head outputs that are constant over the image (a letterbox border) -- the top-k
    metric comes in exactly tied groups there;
  * labels 0 and nc - 1.
`adversarial_head(...)` gives head outputs with scores exactly 0 and 1 (also at the label column of every anchor inside some
boxes), constant images, plain-ltrb distances below 0 and DFL logits whose expectation sits near 0 and near reg_max.
"""
import numpy as np
import pytest
import torch

from oracle import assign as oassign
from oracle import loss as oloss

MAX_GT = 64
NC = 80
P5 = [8, 16, 32]
P6 = [8, 16, 32, 64]
CONST_IMAGES = (3, 4)
TIE_SIDES = (30, 60, 120, 150, 240)      # px; exact in float32 after division by 640 and by 384


def _exact(v, L):
    return float(np.float32(v / L)) * L == v


def _tie_boxes(H, W, img):
    """Integer-pixel boxes centred on a vertex of the stride-64 grid (image 4, one box) or of the stride-32 grid (image 3)."""
    if img == 4:
        return [(W // 2, H // 2, 240, 240)]
    xs = [c for c in range(32, W, 32) if _exact(c, W)]
    ys = [c for c in range(32, H, 32) if _exact(c, H)]
    xs = [xs[len(xs) // 4], xs[(3 * len(xs)) // 4]] if len(xs) >= 2 else xs
    ys = [ys[len(ys) // 4], ys[(3 * len(ys)) // 4]] if len(ys) >= 2 else ys
    out, k = [], 0
    for cy in ys:
        for cx in xs:
            out.append((cx, cy, TIE_SIDES[k % 4], TIE_SIDES[(k + 1) % 4]))
            k += 1
    return out


def coco_like_targets(B, H, W, seed, nc=NC):
    """See the module docstring.  float32 [n, 6]."""
    g = np.random.default_rng(seed)
    rows = []                     # (img, cls, x1, y1, w, h) in pixels

    def box(img, cls, cx, cy, w, h):
        rows.append((img, cls, cx, cy, w, h))

    def random_box(img):
        r = g.random()
        if r < 0.40:              # small: up to 31 px a side
            w, h = g.uniform(2, 31, 2)
        elif r < 0.85:
            w, h = g.uniform(32, 0.6 * W), g.uniform(32, 0.6 * H)
        else:                     # large: DFL targets clip at reg_max - 0.01
            w, h = g.uniform(0.6 * W, W), g.uniform(0.6 * H, H)
        cx, cy = g.uniform(w / 2, W - w / 2), g.uniform(h / 2, H - h / 2)
        box(img, int(g.integers(0, nc)), cx, cy, w, h)

    for img in range(B):
        if img == 2:
            continue
        if img in CONST_IMAGES:
            for cx, cy, w, h in _tie_boxes(H, W, img):
                box(img, int(g.integers(0, nc)), cx, cy, w, h)
            continue
        want = 70 if img == 0 else 64 if img == 1 else int(g.integers(4, 40))
        start = len(rows)
        # 2-6 px boxes strictly between stride-8 anchor centres (centres at 8 i + 4): none inside
        cx0, cy0 = 8.0 * g.integers(2, W // 8 - 2), 8.0 * g.integers(2, H // 8 - 2)
        box(img, 0, cx0, cy0, float(g.uniform(2, 6)), float(g.uniform(2, 6)))
        # k stride-8 centres in one row, k = 1 .. 12 over the images
        k = 1 + img % 12
        ax, ay = 8 * int(g.integers(2, W // 8 - 14)) + 4, 8 * int(g.integers(2, H // 8 - 2)) + 4
        box(img, nc - 1, ax + 4.0 * (k - 1), ay, 8.0 * (k - 1) + 4.0, 4.0)
        # crowd: an exact duplicate, the same box with another class, a box nested inside it
        cls = int(g.integers(0, nc))
        cx, cy, w, h = g.uniform(0.3 * W, 0.7 * W), g.uniform(0.3 * H, 0.7 * H), g.uniform(40, 120), g.uniform(40, 120)
        box(img, cls, cx, cy, w, h)
        box(img, cls, cx, cy, w, h)
        box(img, (cls + 1) % nc, cx, cy, w, h)
        box(img, cls, cx + 0.1 * w, cy - 0.1 * h, 0.5 * w, 0.5 * h)
        # degenerate: zero width, zero height, across the left / bottom edge
        box(img, cls, g.uniform(50, W - 50), g.uniform(50, H - 50), 0.0, g.uniform(10, 40))
        box(img, cls, g.uniform(50, W - 50), g.uniform(50, H - 50), g.uniform(10, 40), 0.0)
        box(img, cls, g.uniform(0, 10), g.uniform(50, H - 50), g.uniform(40, 80), g.uniform(40, 80))
        box(img, cls, g.uniform(50, W - 50), H - g.uniform(0, 10), g.uniform(40, 80), g.uniform(40, 80))
        # a box with edges on stride-8 anchor centres: integer DFL targets
        ex, ey = 8 * int(g.integers(4, W // 8 - 20)) + 4, 8 * int(g.integers(4, H // 8 - 20)) + 4
        box(img, cls, ex + 64.0, ey + 64.0, 128.0, 128.0)
        while len(rows) - start < want:
            random_box(img)
    t = np.array([(i, c, cx / W, cy / H, w / W, h / H) for i, c, cx, cy, w, h in rows], dtype=np.float64)
    t = t[g.permutation(len(t))]
    return torch.from_numpy(t).float()


def trainstep_rows(targets, B, max_gt=MAX_GT):
    """The layout TrainStep.load leaves in its static target buffer: B * max_gt rows, unused rows all -1."""
    out = torch.full((B * max_gt, 6), -1.0)
    out[:targets.shape[0]] = targets
    return out


def sizes_of(H, W, strides):
    return [(H // s, W // s) for s in strides]


def adversarial_head(B, sizes, nc, R, seed, targets, H, W, strides):
    """(scores [B, A, nc] post-sigmoid f32, distri [B, A, R] f32); see the module docstring."""
    g = torch.Generator().manual_seed(7000 + seed)
    A = sum(h * w for h, w in sizes)
    ps = torch.sigmoid(torch.randn(B, A, nc, generator=g) * 1.5 - 2.0)
    u = torch.rand(B, A, nc, generator=g)
    ps[u < 0.003] = 0.0
    ps[u > 0.997] = 1.0
    if R == 4:
        pd = torch.rand(B, A, 4, generator=g) * 4 + 0.5
        neg = torch.rand(B, A, 4, generator=g) < 0.03
        pd[neg] = -torch.rand(int(neg.sum()), generator=g) * 1.5
    else:
        reg_max = R // 4 - 1
        pd = torch.randn(B, A, R, generator=g) * 0.8
        v = pd.view(B, A, 4, reg_max + 1)
        pick = torch.rand(B, A, 4, generator=g)
        lo, hi = pick < 0.02, pick > 0.98
        v[lo] = 0.0
        v[lo, 0] = 16.0               # expectation ~ 1e-5: the box edge on the anchor centre
        v[hi] = 0.0
        v[hi, reg_max] = 16.0         # expectation ~ reg_max - 1e-5
    _, pts, _, _ = oassign.train_anchors(sizes, strides)
    t = oloss.preprocess_targets(targets[targets[:, 0] >= 0], B, torch.tensor([W, H, W, H], dtype=torch.float32))
    for b in (5, 6):                  # label column exactly 1 (image 5) / 0 (image 6) at every anchor inside the first boxes
        if b >= B:
            continue
        for j in range(min(3, t.shape[1])):
            if t[b, j, 0] < 0:
                continue
            inside = oassign.centres_in_gts(pts.double(), t[b, j:j + 1, 1:])[0].bool()
            ps[b, inside, int(t[b, j, 0])] = 1.0 if b == 5 else 0.0
    for b in CONST_IMAGES:
        if b < B:
            ps[b] = 0.5
            pd[b] = 2.0 if R == 4 else 0.0
    return ps.float().contiguous(), pd.float().contiguous()


def padded_gt(targets, B, G, H, W):
    """Restatement of ComputeLoss.preprocess (loss.py:184-192) at a fixed G: rows of each image in input order, rows past
    G dropped, pad rows [-1, 0, 0, 0, 0]; float64.  Also the per-image row counts."""
    gt = torch.zeros(B, G, 5, dtype=torch.float64)
    gt[:, :, 0] = -1.0
    count = torch.zeros(B, dtype=torch.int32)
    sw, sh = float(np.float32(W)), float(np.float32(H))
    for r in targets.tolist():
        b = int(r[0])
        if b < 0 or b >= B:
            continue
        k = int(count[b])
        count[b] += 1
        if k >= G:
            continue
        cx, cy, w, h = r[2] * sw, r[3] * sh, r[4] * sw, r[5] * sh
        x1, y1 = cx - w * 0.5, cy - h * 0.5
        gt[b, k] = torch.tensor([r[1], x1, y1, x1 + w, y1 + h], dtype=torch.float64)
    return gt, count


def plain_boxes(pd, sizes, strides):
    """Predicted boxes in pixels for the assigner, float32 like box_decode (plain ltrb)."""
    _, pts, _, st = oassign.train_anchors(sizes, strides)
    c = pts / st
    return torch.cat([c - pd[..., :2], c + pd[..., 2:]], -1) * st


def tal_topk_sets(ps, pb, pts, gt, ties, topk=13):
    """Per (image, valid gt): the in-gt anchors of its top-k, under one tie rule."""
    out = {}
    for b in range(gt.shape[0]):
        for j in range(gt.shape[1]):
            if gt[b, j, 1:].sum() <= 0:
                continue
            gb = gt[b, j:j + 1, 1:]
            ov = oassign.pair_iou(gb, pb[b])
            lab = int(gt[b, j, 0])
            al = ps[b, :, lab][None].pow(1.0) * ov.pow(6.0)
            ing = oassign.centres_in_gts(pts, gb)
            m = al * ing
            idx = oassign._lowest_k(-m, topk) if ties == "index" else torch.topk(m, topk, dim=-1)[1]
            out[(b, j)] = frozenset(i for i in idx[0].tolist() if ing[0, i] > 0)
    return out


def atss_candidate_sets(anchors, n_list, gt, ties, topk=9):
    acx = (anchors[:, 0] + anchors[:, 2]) / 2.0
    acy = (anchors[:, 1] + anchors[:, 3]) / 2.0
    ac = torch.stack([acx, acy], 1)
    out = {}
    for b in range(gt.shape[0]):
        for j in range(gt.shape[1]):
            if gt[b, j, 1:].sum() <= 0:
                continue
            gb = gt[b, j, 1:]
            gc = torch.stack([(gb[0] + gb[2]) / 2.0, (gb[1] + gb[3]) / 2.0])
            dist = (gc[None] - ac).pow(2).sum(-1).sqrt()
            sel, start = [], 0
            for n in n_list:
                d = dist[start:start + n][None]
                k = min(topk, n)
                idx = oassign._lowest_k(d, k) if ties == "index" else d.topk(k, dim=-1, largest=False)[1]
                sel += (idx[0] + start).tolist()
                start += n
            out[(b, j)] = frozenset(sel)
    return out


CASES = {"square": dict(B=32, H=640, W=640, seed=11), "rect": dict(B=32, H=384, W=640, seed=12)}


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    c = dict(CASES[request.param], name=request.param)
    c["targets"] = coco_like_targets(c["B"], c["H"], c["W"], c["seed"])
    c["gt"], c["count"] = padded_gt(c["targets"], c["B"], MAX_GT, c["H"], c["W"])
    return c


def test_counts_and_trainstep_layout(case):
    t, B = case["targets"], case["B"]
    count = torch.bincount(t[:, 0].long(), minlength=B)
    assert count[0] == 70 and count[1] == 64 and count[2] == 0
    assert int(count[3:].max()) < MAX_GT
    assert torch.equal(case["count"], count.int())
    assert case["gt"][0, :, 0].ge(0).all() and case["gt"][2, :, 0].eq(-1).all()
    # rows of image 0 are interleaved with other images' rows, so "the first 64" is an order in the input
    first = (t[:, 0] == 0).nonzero().flatten()
    assert (t[first[0]:first[-1], 0] != 0).any()
    rows = trainstep_rows(t, B)
    assert rows.shape == (B * MAX_GT, 6) and rows[t.shape[0]:].eq(-1).all() and torch.equal(rows[:t.shape[0]], t)


def test_small_boxes_and_anchor_centres(case):
    gt, H, W = case["gt"], case["H"], case["W"]
    valid = gt[..., 1:].sum(-1) > 0
    b = gt[valid][:, 1:]
    w, h = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
    small = (w * h < 32 * 32).double().mean()
    assert 0.3 < small < 0.55, small
    _, pts, _, _ = oassign.train_anchors(sizes_of(H, W, [8]), [8])
    inside = oassign.centres_in_gts(pts.double(), b).sum(-1)
    tiny = (w >= 2) & (w <= 6) & (h >= 2) & (h <= 6)
    assert (tiny & (inside == 0)).any()
    assert set(range(1, 13)) <= set(inside[(h - 4).abs() < 1e-3].long().tolist())


def test_crowds_and_degenerate_boxes(case):
    gt, W, H = case["gt"], case["W"], case["H"]
    same = diff = nested = 0
    for b in range(gt.shape[0]):
        r = gt[b][gt[b, :, 1:].sum(-1) > 0]
        eq_box = (r[:, None, 1:] == r[None, :, 1:]).all(-1) & ~torch.eye(len(r), dtype=torch.bool)
        eq_cls = r[:, None, 0] == r[None, :, 0]
        same += int((eq_box & eq_cls).sum())
        diff += int((eq_box & ~eq_cls).sum())
        inner = (r[:, None, 1] > r[None, :, 1]) & (r[:, None, 2] > r[None, :, 2]) & (r[:, None, 3] < r[None, :, 3]) & \
                (r[:, None, 4] < r[None, :, 4])
        nested += int(inner.sum())
    assert same > 0 and diff > 0 and nested > 0
    v = gt[gt[..., 1:].sum(-1) > 0]
    assert ((v[:, 3] == v[:, 1]) & (v[:, 4] > v[:, 2])).any()
    assert ((v[:, 4] == v[:, 2]) & (v[:, 3] > v[:, 1])).any()
    assert (v[:, 1] < 0).any() and (v[:, 4] > H).any()
    assert (v[:, 0] == 0).any() and (v[:, 0] == NC - 1).any()
    assert (v[:, 3] <= W).all()


def test_anchors_claimed_by_several_gts(case):
    B, H, W = case["B"], case["H"], case["W"]
    sizes = sizes_of(H, W, P5)
    ps, pd = adversarial_head(B, sizes, NC, 4, case["seed"], case["targets"], H, W, P5)
    pb = plain_boxes(pd, sizes, P5)
    _, pts, _, _ = oassign.train_anchors(sizes, P5)
    claims = torch.zeros(B, pts.shape[0], dtype=torch.int64)
    for (b, j), s in tal_topk_sets(ps, pb, pts, case["gt"], "index").items():
        claims[b, list(s)] += 1
    assert int((claims > 1).sum()) > 100


def test_tie_boxes_make_the_tie_rules_disagree(case):
    gt, B, H, W = case["gt"], case["B"], case["H"], case["W"]
    for b in CONST_IMAGES:
        r = gt[b][gt[b, :, 1:].sum(-1) > 0][:, 1:]
        assert len(r) > 0 and torch.equal(r, r.round()), "tie boxes are integer-pixel"
        c = (r[:, :2] + r[:, 2:]) / 2
        assert (c % 32 == 0).all(), "centred on a vertex of the stride-8, 16 and 32 grids"
    assert ((gt[4, 0, 1:3] + gt[4, 0, 3:5]) / 2 % 64 == 0).all(), "and of the stride-64 grid"
    for strides in (P5, P6):
        sizes = sizes_of(H, W, strides)
        ps, pd = adversarial_head(B, sizes, NC, 4, case["seed"], case["targets"], H, W, strides)
        pb = plain_boxes(pd, sizes, strides)
        anchors, pts, n_list, _ = oassign.train_anchors(sizes, strides)
        sub = gt[list(CONST_IMAGES)]
        for k in (13, 26):
            a = tal_topk_sets(ps[list(CONST_IMAGES)], pb[list(CONST_IMAGES)], pts, sub, "index", k)
            o = tal_topk_sets(ps[list(CONST_IMAGES)], pb[list(CONST_IMAGES)], pts, sub, "topk", k)
            assert any(a[key] != o[key] for key in a), f"TAL topk {k}: the tie rules agree on every gt"
        a, o = atss_candidate_sets(anchors, n_list, sub, "index"), atss_candidate_sets(anchors, n_list, sub, "topk")
        assert any(a[key] != o[key] for key in a), "ATSS: the tie rules agree on every gt"


def test_head_outputs_reach_the_clamps(case):
    B, H, W, t = case["B"], case["H"], case["W"], case["targets"]
    sizes = sizes_of(H, W, P5)
    ps, pd = adversarial_head(B, sizes, NC, 4, case["seed"], t, H, W, P5)
    assert (ps == 0).any() and (ps == 1).any() and (pd < 0).any()
    for b in CONST_IMAGES:
        assert (ps[b] == 0.5).all() and (pd[b] == 2.0).all()
    pb = plain_boxes(pd, sizes, P5)
    _, pts, _, _ = oassign.train_anchors(sizes, P5)
    gt = case["gt"]
    mask = (gt[..., 1:].sum(-1, keepdim=True) > 0).float()
    labels, _, _, fg, gi = oassign.tal_assign(ps, pb, pts, gt[..., :1], gt[..., 1:], mask, num_classes=NC, ties="index")
    pos_score = ps.gather(2, labels[..., None].clamp(min=0))[..., 0][fg]
    assert (pos_score == 1).any(), "a positive anchor with score exactly 1 at its label"
    # DFL: expectations near 0 and reg_max, targets on an integer bin and clipped at reg_max - 0.01
    reg_max = 16
    _, pdd = adversarial_head(B, sizes, NC, 4 * (reg_max + 1), case["seed"], t, H, W, P5)
    e = (torch.softmax(pdd.view(B, -1, 4, reg_max + 1).double(), -1) * torch.arange(reg_max + 1).double()).sum(-1)
    assert (e < 0.01).any() and (e > reg_max - 0.01).any()
    _, _, _, st = oassign.train_anchors(sizes, P5)
    pbd = oloss.decode_pred(pdd, pts / st, True, reg_max) * st
    _, tb, _, fgd, _ = oassign.tal_assign(ps, pbd, pts, gt[..., :1], gt[..., 1:], mask, num_classes=NC, ties="index")
    aps = (pts / st).double()[None].expand(B, -1, -1)
    tbs = tb / st.double()
    ltrb = torch.cat([aps - tbs[..., :2], tbs[..., 2:] - aps], -1)[fgd]
    assert (ltrb >= reg_max - 0.01).any(), "DFL targets clipped at reg_max - 0.01"
    assert ((ltrb == ltrb.round()) & (ltrb > 0) & (ltrb < reg_max - 0.01)).any(), "DFL targets on an integer bin"


def test_rect_case_scales_x_and_y_apart():
    c = CASES["rect"]
    t = coco_like_targets(c["B"], c["H"], c["W"], c["seed"])
    gt, _ = padded_gt(t, c["B"], MAX_GT, c["H"], c["W"])
    v = gt[gt[..., 1:].sum(-1) > 0]
    assert c["H"] != c["W"] and float(v[:, 4].max()) > c["H"] - 20 and float(v[:, 3].max()) > c["H"] + 100
    swapped, _ = padded_gt(t, c["B"], MAX_GT, c["W"], c["H"])
    assert not torch.equal(swapped, gt)


def test_tie_rule_option_matches_topk_away_from_ties():
    """On inputs without exact ties the two rules are the same assignment (the default still is what the goldens pin)."""
    sizes = sizes_of(160, 160, P5)
    g = torch.Generator().manual_seed(5)
    A = sum(h * w for h, w in sizes)
    ps = torch.rand(2, A, 5, generator=g) * 0.9 + 0.05
    pd = torch.rand(2, A, 4, generator=g) * 3 + 0.5
    t = oloss.synthetic_targets(2, seed=6, num_classes=5)
    gt = oloss.preprocess_targets(t, 2, torch.tensor([160.0] * 4))
    mask = (gt[..., 1:].sum(-1, keepdim=True) > 0).float()
    anchors, pts, n_list, _ = oassign.train_anchors(sizes, P5)
    pb = plain_boxes(pd, sizes, P5)
    for k in (13, 26):
        a = oassign.tal_assign(ps, pb, pts, gt[..., :1], gt[..., 1:], mask, topk=k, num_classes=5)
        b = oassign.tal_assign(ps, pb, pts, gt[..., :1], gt[..., 1:], mask, topk=k, num_classes=5, ties="index")
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    a = oassign.atss_assign(anchors, n_list, gt[..., :1], gt[..., 1:], mask, pb, num_classes=5)
    b = oassign.atss_assign(anchors, n_list, gt[..., :1], gt[..., 1:], mask, pb, num_classes=5, ties="index")
    assert torch.equal(a[3], b[3]) and torch.equal(a[4], b[4]) and torch.equal(a[0], b[0])
    with pytest.raises(ValueError):
        oassign.tal_assign(ps, pb, pts, gt[..., :1], gt[..., 1:], mask, ties="random")
