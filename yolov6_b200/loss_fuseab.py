"""Drop-in `ComputeLoss` of the anchor-aided (fuse_ab) branch, backed by the sm_90a assignment + loss kernels.

Same constructor and call signature as the reference's yolov6/models/losses/loss_fuseab.py:14-148, which the Trainer
uses next to the anchor-free loss when `--fuse_ab` is given (core/engine.py:161-166, 298-309):

    preds, _ = model(images)                                     # (feats, cls_ab, reg_ab, cls_af, reg_af)
    loss, items = compute_loss((preds[0], preds[3], preds[4]), targets, ...)
    loss_ab, items_ab = compute_loss_ab(preds[:3], targets, ...)

What differs from the anchor-free loss (loss.py): anchors in mode 'ab' (every cell centre three times, rows ordered
(level, anchor, pixel), anchor_generator.py:53-55), boxes built from (x_off, y_off, w, h) around the cell centre
(loss_fuseab.py:71-76), TaskAlignedAssigner with topk = 26 at every epoch (:40, no ATSS warm-up), no DFL term, and the
sums are divided by `target_scores_sum` whenever it is > 0 (:139, BboxLoss :203-206) instead of > 1.

Implementation: `yv6_ab_boxes` turns the head's (x_off, y_off, w, h) into pixel boxes for the assigner and into the
equivalent (l, t, r, b) distances around the cell centre, so that `yv6_tal_assign` and `yv6_det_loss` (value + gradients in
one launch) are reused unchanged; `yv6_ab_boxes_bwd` maps the gradient back.  Everything runs on the device without host
synchronisation (except the per-image target count when `max_gt` is not given, as in loss.py).
"""
import torch

from . import _lib
from .assigners import _p, generate_anchors_train, tal_compact
from .loss import ComputeLoss as _DetLoss

AB_TOPK = 26        # loss_fuseab.py:40


def generate_anchors_ab(sizes, strides, device, grid_cell_offset=0.5, num_anchors=3):
    """anchor_generator.py:36-63 with mode='ab': the train-mode cell centres in pixels and strides, each level's block repeated
    `num_anchors` times ((anchor, pixel) order inside a level)."""
    levels = [generate_anchors_train([hw], [s], device, 0.0, grid_cell_offset) for hw, s in zip(sizes, strides)]
    pts = torch.cat([pt.repeat(num_anchors, 1) for _, pt, _, _ in levels])
    strs = torch.cat([st.repeat(num_anchors, 1) for _, _, _, st in levels])
    return pts.contiguous(), strs.contiguous()


class ComputeLoss(_DetLoss):
    _norm_gt_zero = 1       # loss_fuseab.py:139, 203-206

    def __init__(self, fpn_strides=[8, 16, 32], grid_cell_size=5.0, grid_cell_offset=0.5, num_classes=80,
                 ori_img_size=640, warmup_epoch=0, use_dfl=True, reg_max=16, iou_type='giou',
                 loss_weight={'class': 1.0, 'iou': 2.5, 'dfl': 0.5}):     # use_dfl: the ab head has no DFL term either way
        super().__init__(fpn_strides, grid_cell_size, grid_cell_offset, num_classes, ori_img_size, warmup_epoch, use_dfl, reg_max,
                         iou_type, loss_weight)

    def _build_anchors(self, sizes, device):
        return generate_anchors_ab(sizes, self.fpn_strides, device, self.grid_cell_offset)

    def forward_backward(self, pred_scores, pred_distri, sizes, targets, epoch_num, batch_height, batch_width, max_gt=None,
                         grad_scores=None, grad_distri=None, grad_scale=1.0):
        """Loss value and its gradients w.r.t. (cls_ab, reg_ab) in one pass; same contract as loss.ComputeLoss.forward_backward."""
        _lib.require_cuda(pred_scores, "yolov6_b200.loss_fuseab.ComputeLoss runs")
        dev = pred_scores.device
        anchor_points, stride_t = self._get_anchors(sizes, dev)
        B, A, nc = pred_scores.shape
        if pred_distri.shape[2] != 4 or anchor_points.shape[0] != A:
            raise RuntimeError(f"fuse_ab loss: expected [B, {anchor_points.shape[0]}, 4] box predictions, got {tuple(pred_distri.shape)}")
        lib, h, sp = _lib.lib(), _lib.handle(dev.index or 0), _lib.stream_ptr()
        ps, pd = (t.detach().float().contiguous() for t in (pred_scores, pred_distri))
        strides = stride_t.reshape(-1).contiguous()
        st, tg = self._pad_targets(targets, B, max_gt, batch_height, batch_width, dev)
        ltrb = torch.empty(B, A, 4, dtype=torch.float32, device=dev)
        pboxes = torch.empty(B, A, 4, dtype=torch.float32, device=dev)
        _lib.check(lib.yv6_ab_boxes(h, _p(pd), _p(anchor_points), _p(strides), B, A, _p(ltrb), _p(pboxes), sp))
        # formal_assigner, every epoch (:78-86)
        st["assignment"] = self.last_assignment = tal_compact(ps, pboxes, anchor_points, st["gt"], st["mask"], AB_TOPK, 1.0, 6.0)
        grad_distri = torch.empty_like(pd) if grad_distri is None else grad_distri
        grad_ltrb = torch.empty_like(pd)
        ws = self._det_loss(st, ps, ltrb, anchor_points, strides, grad_scores, grad_ltrb, grad_scale)
        _lib.check(lib.yv6_ab_boxes_bwd(h, _p(grad_ltrb), B * A, _p(grad_distri), sp))
        st["grad_distri"], st["keep"] = grad_distri, (ps, pd, st["gt"], st["mask"], pboxes, ltrb, grad_ltrb, ws, tg)
        return st
