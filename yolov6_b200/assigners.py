"""Drop-in label assigners backed by the sm_90a kernels of csrc/yv6_assign.cu.

`TaskAlignedAssigner` / `ATSSAssigner` keep the constructor and `forward` signatures and the dense
return values of the reference (yolov6/assigners/tal_assigner.py:6-95, atss_assigner.py:7-86):
(target_labels int64 [B,A], target_bboxes [B,A,4], target_scores [B,A,nc], fg_mask bool [B,A]).
The compact form used by the fused loss is available through `assign_compact`.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _pack_gt(gt_labels, gt_bboxes):
    """[B,G,1] labels + [B,G,4] boxes -> [B,G,5] float64 (class, xyxy)."""
    return torch.cat([gt_labels.double().reshape(*gt_bboxes.shape[:2], 1), gt_bboxes.double()], -1).contiguous()


def generate_anchors_train(sizes, strides, device, grid_cell_size=5.0, grid_cell_offset=0.5):
    """Train-mode anchors of reference yolov6/assigners/anchor_generator.py:34-63, built analytically:
    anchor boxes [A,4], centres in pixels [A,2], per-level counts, stride column [A,1]."""
    boxes, pts, counts, strs = [], [], [], []
    for (h, w), s in zip(sizes, strides):
        half = grid_cell_size * s * 0.5
        sx = (torch.arange(w, dtype=torch.float32, device=device) + grid_cell_offset) * s
        sy = (torch.arange(h, dtype=torch.float32, device=device) + grid_cell_offset) * s
        yy, xx = torch.meshgrid(sy, sx, indexing="ij")
        boxes.append(torch.stack([xx - half, yy - half, xx + half, yy + half], -1).reshape(-1, 4))
        pts.append(torch.stack([xx, yy], -1).reshape(-1, 2))
        counts.append(h * w)
        strs.append(torch.full((h * w, 1), float(s), dtype=torch.float32, device=device))
    return torch.cat(boxes).contiguous(), torch.cat(pts).contiguous(), counts, torch.cat(strs).contiguous()


class _Compact:
    """gt [B,G,5] f64, gt_idx [B,A] i32, fg [B,A] u8, norm [B,A] f64."""
    __slots__ = ("gt", "gt_idx", "fg", "norm", "B", "A", "G", "nc")


def _workspace(dev, nbytes):
    return torch.empty(int(nbytes), dtype=torch.uint8, device=dev)


def tal_compact(pd_scores, pd_bboxes, anc_points, gt, mask_gt, topk=13, alpha=1.0, beta=6.0, eps=1e-9, stream=None):
    B, A, nc = pd_scores.shape
    if A < topk:      # the reference's torch.topk over the anchors raises here (tal_assigner.py:141); the kernel would pad with -1
        raise ValueError(f"TAL: top-{topk} candidates of a map with {A} anchors: the map needs at least {topk} anchors")
    _lib.require_cuda(pd_scores, "yolov6_b200 assigners run")
    dev = pd_scores.device
    G = gt.shape[1]
    out = _Compact()
    out.gt, out.B, out.A, out.G, out.nc = gt, B, A, G, nc
    out.gt_idx = torch.empty(B, A, dtype=torch.int32, device=dev)
    out.fg = torch.empty(B, A, dtype=torch.uint8, device=dev)
    out.norm = torch.empty(B, A, dtype=torch.float64, device=dev)
    lib = _lib.lib()
    ws = _workspace(dev, lib.yv6_assign_workspace_bytes(B, A, G))
    _lib.check(lib.yv6_tal_assign(_lib.handle(dev.index or 0), _p(pd_scores.float().contiguous()),
                                  _p(pd_bboxes.float().contiguous()), _p(anc_points.float().contiguous()), _p(gt),
                                  _p(mask_gt), B, A, G, nc, int(topk), float(alpha), float(beta), float(eps),
                                  _p(out.gt_idx), _p(out.fg), _p(out.norm), _p(ws), ws.numel(), _lib.stream_ptr(stream)))
    return out


def atss_compact(anc_bboxes, n_level_bboxes, gt, mask_gt, pd_bboxes, nc, topk=9, stream=None):
    _lib.require_cuda(anc_bboxes, "yolov6_b200 assigners run")
    dev = anc_bboxes.device
    B, G = gt.shape[:2]
    A = anc_bboxes.shape[0]
    out = _Compact()
    out.gt, out.B, out.A, out.G, out.nc = gt, B, A, G, nc
    out.gt_idx = torch.empty(B, A, dtype=torch.int32, device=dev)
    out.fg = torch.empty(B, A, dtype=torch.uint8, device=dev)
    out.norm = torch.empty(B, A, dtype=torch.float64, device=dev)
    lib = _lib.lib()
    ws = _workspace(dev, lib.yv6_assign_workspace_bytes(B, A, G))
    lv = (C.c_int32 * len(n_level_bboxes))(*[int(n) for n in n_level_bboxes])
    _lib.check(lib.yv6_atss_assign(_lib.handle(dev.index or 0), _p(anc_bboxes.float().contiguous()), lv,
                                   len(n_level_bboxes), _p(gt), _p(mask_gt),
                                   _p(pd_bboxes.float().contiguous()) if pd_bboxes is not None else C.c_void_p(0),
                                   B, A, G, nc, int(topk), _p(out.gt_idx), _p(out.fg), _p(out.norm), _p(ws),
                                   ws.numel(), _lib.stream_ptr(stream)))
    return out


def expand(c, bg_label, stream=None):
    """Compact assignment -> the reference's dense tensors."""
    dev = c.gt.device
    labels = torch.empty(c.B, c.A, dtype=torch.int64, device=dev)
    bboxes = torch.empty(c.B, c.A, 4, dtype=torch.float64, device=dev)
    scores = torch.empty(c.B, c.A, c.nc, dtype=torch.float64, device=dev)
    fg = torch.empty(c.B, c.A, dtype=torch.bool, device=dev)
    _lib.check(_lib.lib().yv6_assign_expand(_lib.handle(dev.index or 0), _p(c.gt), _p(c.gt_idx), _p(c.fg), _p(c.norm),
                                            c.B, c.A, c.G, c.nc, int(bg_label), _p(labels), _p(bboxes), _p(scores),
                                            _p(fg), _lib.stream_ptr(stream)))
    return labels, bboxes, scores, fg


class TaskAlignedAssigner(nn.Module):
    def __init__(self, topk=13, num_classes=80, alpha=1.0, beta=6.0, eps=1e-9):
        super().__init__()
        self.topk, self.num_classes, self.bg_idx = topk, num_classes, num_classes
        self.alpha, self.beta, self.eps = alpha, beta, eps

    @torch.no_grad()
    def forward(self, pd_scores, pd_bboxes, anc_points, gt_labels, gt_bboxes, mask_gt):
        self.bs, self.n_max_boxes = pd_scores.size(0), gt_bboxes.size(1)
        if self.n_max_boxes == 0:       # tal_assigner.py:48-53
            return (torch.full_like(pd_scores[..., 0], self.bg_idx), torch.zeros_like(pd_bboxes),
                    torch.zeros_like(pd_scores), torch.zeros_like(pd_scores[..., 0]))
        gt = _pack_gt(gt_labels, gt_bboxes)
        mask = (mask_gt.reshape(self.bs, self.n_max_boxes) > 0).to(torch.uint8).contiguous()
        c = tal_compact(pd_scores, pd_bboxes, anc_points, gt, mask, self.topk, self.alpha, self.beta, self.eps)
        return expand(c, -1)


class ATSSAssigner(nn.Module):
    def __init__(self, topk=9, num_classes=80):
        super().__init__()
        self.topk, self.num_classes, self.bg_idx = topk, num_classes, num_classes

    @torch.no_grad()
    def forward(self, anc_bboxes, n_level_bboxes, gt_labels, gt_bboxes, mask_gt, pd_bboxes):
        self.n_anchors, self.bs, self.n_max_boxes = anc_bboxes.size(0), gt_bboxes.size(0), gt_bboxes.size(1)
        if self.n_max_boxes == 0:       # atss_assigner.py:45-50
            dev = gt_bboxes.device
            return (torch.full([self.bs, self.n_anchors], self.bg_idx).to(dev), torch.zeros([self.bs, self.n_anchors, 4]).to(dev),
                    torch.zeros([self.bs, self.n_anchors, self.num_classes]).to(dev), torch.zeros([self.bs, self.n_anchors]).to(dev))
        gt = _pack_gt(gt_labels, gt_bboxes)
        mask = (mask_gt.reshape(self.bs, self.n_max_boxes) > 0).to(torch.uint8).contiguous()
        c = atss_compact(anc_bboxes, n_level_bboxes, gt, mask, pd_bboxes, self.num_classes, self.topk)
        return expand(c, self.bg_idx)
