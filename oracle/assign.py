"""oracle/assign.py -- CPU restatement of the label assigners (TEST INFRASTRUCTURE ONLY).

Re-states, one image at a time with dense [G, A] tensors, what the reference computes in
  * TaskAlignedAssigner.forward   yolov6/assigners/tal_assigner.py:22-173
  * ATSSAssigner.forward          yolov6/assigners/atss_assigner.py:18-161
  * the helpers in                yolov6/assigners/assigner_utils.py:4-89 and
                                  yolov6/assigners/iou2d_calculator.py:201-243 (bbox_overlaps)
  * generate_anchors (train)      yolov6/assigners/anchor_generator.py:34-63
Everything derived from the ground truth is float64, as in the reference (its targets come from
numpy float64, SURVEY.md F5).  `torch.topk` is used for the top-k steps because its tie order is
part of what the reference observes on CPU.  Pinned against the live reference by
tests/golden/make_golden.py.

`ties="index"` replaces `torch.topk`, whose order among equal values is unspecified, by the rule the
CUDA assigners state (yv6_assign.cu): a stable sort on (-metric, anchor index) for TAL and on
(distance, anchor index) for ATSS, so ties go to the lower anchor index.  In that mode ATSS also
forms the mean and the standard deviation of the candidate IoUs as the kernel does (sequential
float64 sums over the candidates in level, then rank order), so an IoU equal to the threshold falls
on the same side.  Duplicate top-k indices are counted with `scatter_add` there, which keeps the
memory at [G, A] per image.
"""
import torch
import torch.nn.functional as F

TIE_RULES = ("topk", "index")


def _lowest_k(keys, k):
    """Indices of the k smallest keys along the last dim, equal keys in index order."""
    return torch.sort(keys, dim=-1, stable=True)[1][..., :k]


def _count(idx, n):
    """[G, k] indices -> [G, n] number of times each index occurs in its row."""
    return torch.zeros(idx.shape[0], n, dtype=torch.int64).scatter_add_(1, idx, torch.ones_like(idx))


def _seq_sum(x):
    """Sum over the last dim, left to right, keepdim."""
    s = torch.zeros_like(x[..., :1])
    for j in range(x.shape[-1]):
        s = s + x[..., j:j + 1]
    return s


def train_anchors(sizes, strides, cell_size=5.0, cell_offset=0.5, dtype=torch.float32):
    """anchor boxes [A,4], centres in pixels [A,2], per-level counts, stride column [A,1]."""
    boxes, pts, counts, strs = [], [], [], []
    for (h, w), s in zip(sizes, strides):
        half = cell_size * s * 0.5
        sx = (torch.arange(w, dtype=dtype) + cell_offset) * s
        sy = (torch.arange(h, dtype=dtype) + cell_offset) * s
        yy, xx = torch.meshgrid(sy, sx, indexing="ij")
        boxes.append(torch.stack([xx - half, yy - half, xx + half, yy + half], -1).reshape(-1, 4))
        pts.append(torch.stack([xx, yy], -1).reshape(-1, 2))
        counts.append(h * w)
        strs.append(torch.full((h * w, 1), float(s), dtype=dtype))
    return torch.cat(boxes), torch.cat(pts), counts, torch.cat(strs)


def pair_iou(gt, pd, eps=1e-9):
    """iou_calculator, assigner_utils.py:69-89: gt [G,4], pd [A,4] -> [G,A]."""
    g, p = gt[:, None, :], pd[None, :, :]
    wh = (torch.minimum(g[..., 2:], p[..., 2:]) - torch.maximum(g[..., :2], p[..., :2])).clip(0)
    inter = wh[..., 0] * wh[..., 1]
    a1 = (g[..., 2:] - g[..., :2]).clip(0).prod(-1)
    a2 = (p[..., 2:] - p[..., :2]).clip(0).prod(-1)
    return inter / (a1 + a2 - inter + eps)


def centres_in_gts(pts, gt, eps=1e-9):
    """select_candidates_in_gts, assigner_utils.py:25-44 -> [G,A] in gt dtype."""
    lt = pts[None, :, :] - gt[:, None, :2]
    rb = gt[:, None, 2:] - pts[None, :, :]
    return (torch.cat([lt, rb], -1).min(-1)[0] > eps).to(gt.dtype)


def resolve_conflicts(mask_pos, overlaps):
    """select_highest_overlaps, assigner_utils.py:46-67 (per image)."""
    fg = mask_pos.sum(0)
    if fg.max() > 1:
        multi = fg[None, :] > 1
        best = F.one_hot(overlaps.argmax(0), overlaps.shape[0]).T.to(overlaps.dtype)
        mask_pos = torch.where(multi, best, mask_pos)
        fg = mask_pos.sum(0)
    return mask_pos.argmax(0), fg, mask_pos


def tal_assign(pd_scores, pd_bboxes, anc_points, gt_labels, gt_bboxes, mask_gt, topk=13, num_classes=80,
               alpha=1.0, beta=6.0, eps=1e-9, ties="topk"):
    """pd_scores [B,A,nc] f32, pd_bboxes [B,A,4] f32 (pixels), anc_points [A,2], gt_labels [B,G,1],
    gt_bboxes [B,G,4] f64, mask_gt [B,G,1].  Returns labels i64 [B,A], bboxes [B,A,4], scores
    [B,A,nc], fg bool [B,A], gt_idx i64 [B,A].  `ties`: see the module docstring."""
    if ties not in TIE_RULES:
        raise ValueError(f"ties={ties!r}")
    B, A, _ = pd_scores.shape
    G = gt_bboxes.shape[1]
    if G == 0:  # tal_assigner.py:48-53
        return (torch.full((B, A), num_classes, dtype=pd_scores.dtype), torch.zeros_like(pd_bboxes),
                torch.zeros_like(pd_scores), torch.zeros(B, A, dtype=torch.bool), torch.zeros(B, A, dtype=torch.int64))
    out = [[] for _ in range(5)]
    for b in range(B):
        gl = gt_labels[b, :, 0].long()
        gb = gt_bboxes[b]
        mg = mask_gt[b]                                                  # [G,1]
        ov = pair_iou(gb, pd_bboxes[b])                                  # :129
        sc = pd_scores[b].T[gl]                                          # :123-128 (label -1 -> last class)
        al = sc.pow(alpha) * ov.pow(beta)                                # :131
        ing = centres_in_gts(anc_points, gb)                             # :108
        if ties == "index":
            idx = _lowest_k(-(al * ing), topk)
        else:
            _, idx = torch.topk(al * ing, topk, dim=-1, largest=True)    # :141-142
        idx = torch.where(mg.bool().expand(-1, topk), idx, torch.zeros_like(idx))
        cnt = _count(idx, A) if ties == "index" else F.one_hot(idx, A).sum(-2)
        in_topk = torch.where(cnt > 1, torch.zeros_like(cnt), cnt).to(al.dtype)   # :146-149
        mask_pos = in_topk * ing * mg                                    # :113
        gt_idx, fg, mask_pos = resolve_conflicts(mask_pos, ov)
        labels = gl[gt_idx].clone()
        labels[labels < 0] = 0                                           # :165
        boxes = gb[gt_idx]
        scores = F.one_hot(labels, num_classes)
        scores = torch.where(fg[:, None] > 0, scores, torch.zeros_like(scores))
        al = al * mask_pos                                               # :77-81
        pos_al = al.max(-1, keepdim=True)[0]
        pos_ov = (ov * mask_pos).max(-1, keepdim=True)[0]
        norm = (al * pos_ov / (pos_al + eps)).max(0)[0][:, None]
        scores = scores * norm
        for lst, v in zip(out, (labels, boxes, scores, fg.bool(), gt_idx)):
            lst.append(v)
    return tuple(torch.stack(o) for o in out)


def bbox_overlaps_max_eps(b1, b2, eps=1e-6):
    """iou2d_calculator / bbox_overlaps(mode='iou'), iou2d_calculator.py:201-243: union clamped by eps."""
    a1 = (b1[:, 2] - b1[:, 0]) * (b1[:, 3] - b1[:, 1])
    a2 = (b2[:, 2] - b2[:, 0]) * (b2[:, 3] - b2[:, 1])
    wh = (torch.minimum(b1[:, None, 2:], b2[None, :, 2:]) - torch.maximum(b1[:, None, :2], b2[None, :, :2])).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = torch.max(a1[:, None] + a2[None, :] - inter, torch.tensor([eps], dtype=inter.dtype))
    return inter / union


def atss_assign(anc_bboxes, n_level, gt_labels, gt_bboxes, mask_gt, pd_bboxes, topk=9, num_classes=80, ties="topk"):
    """ATSSAssigner.forward.  Returns labels i64 [B,A] (bg = num_classes), bboxes, scores f32->f64, fg, gt_idx.
    `ties`: see the module docstring."""
    if ties not in TIE_RULES:
        raise ValueError(f"ties={ties!r}")
    B, G = gt_bboxes.shape[:2]
    A = anc_bboxes.shape[0]
    if G == 0:  # atss_assigner.py:45-50
        return (torch.full((B, A), num_classes), torch.zeros(B, A, 4), torch.zeros(B, A, num_classes),
                torch.zeros(B, A), torch.zeros(B, A, dtype=torch.int64))
    acx = (anc_bboxes[:, 0] + anc_bboxes[:, 2]) / 2.0
    acy = (anc_bboxes[:, 1] + anc_bboxes[:, 3]) / 2.0
    ac = torch.stack([acx, acy], 1)
    out = [[] for _ in range(5)]
    for b in range(B):
        gb = gt_bboxes[b]
        mg = mask_gt[b]
        ov = bbox_overlaps_max_eps(gb, anc_bboxes.to(gb.dtype))              # :53
        gc = torch.stack([(gb[:, 0] + gb[:, 2]) / 2.0, (gb[:, 1] + gb[:, 3]) / 2.0], 1)
        dist = (gc[:, None, :] - ac[None, :, :]).pow(2).sum(-1).sqrt()        # assigner_utils.py:21
        cand_mask, cand_idx, start = [], [], 0
        for n in n_level:                                                     # :88-116
            k = min(topk, n)
            if ties == "index":
                idx = _lowest_k(dist[:, start:start + n], k)
            else:
                _, idx = dist[:, start:start + n].topk(k, dim=-1, largest=False)
            cand_idx.append(idx + start)
            idx = torch.where(mg.bool().expand(-1, k), idx, torch.zeros_like(idx))
            cnt = _count(idx, n) if ties == "index" else F.one_hot(idx, n).sum(-2)
            cand_mask.append(torch.where(cnt > 1, torch.zeros_like(cnt), cnt).to(dist.dtype))
            start += n
        is_cand = torch.cat(cand_mask, -1)
        cand_idx = torch.cat(cand_idx, -1)
        cov = torch.where(is_cand > 0, ov, torch.zeros_like(ov))              # :124-125
        sel = torch.gather(cov, 1, cand_idx)
        if ties == "index":
            n_c = sel.shape[-1]
            mean = _seq_sum(sel) / n_c
            thr = mean + (_seq_sum((sel - mean) * (sel - mean)) / (n_c - 1)).sqrt()
        else:
            thr = sel.mean(-1, keepdim=True) + sel.std(-1, keepdim=True)      # :132-134
        is_pos = torch.where(cov > thr, is_cand, torch.zeros_like(is_cand))   # :65-67
        mask_pos = is_pos * centres_in_gts(ac.to(gb.dtype), gb) * mg          # :69-70
        gt_idx, fg, mask_pos = resolve_conflicts(mask_pos, ov)
        labels = gt_labels[b, :, 0][gt_idx]
        labels = torch.where(fg > 0, labels, torch.full_like(labels, num_classes)).long()
        boxes = gb[gt_idx]
        scores = F.one_hot(labels, num_classes + 1).float()[:, :num_classes]
        ious = (pair_iou(gb, pd_bboxes[b]) * mask_pos).max(0)[0][:, None]     # :81-84
        scores = scores.mul_(ious)   # in place: stays float32 like the reference (atss_assigner.py:84)
        for lst, v in zip(out, (labels, boxes, scores, fg.bool(), gt_idx)):
            lst.append(v)
    return tuple(torch.stack(o) for o in out)
