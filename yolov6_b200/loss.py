"""Drop-in `ComputeLoss` backed by the sm_90a assignment + fused loss kernels.

Same constructor and call signature as the reference (yolov6/models/losses/loss.py:14-182):
    ComputeLoss(fpn_strides, grid_cell_size, grid_cell_offset, num_classes, ori_img_size, warmup_epoch,
                use_dfl, reg_max, iou_type, loss_weight)
    loss, loss_items = compute_loss(outputs, targets, epoch_num, step_num, batch_height, batch_width)
`loss` is a float64 scalar that is differentiable w.r.t. pred_scores / pred_distri (the gradients are
produced by the same kernel launch as the forward values); `loss_items` = [iou, dfl, cls] weighted and
detached (loss.py:179-182).  The whole path (target padding, box decode, TAL or ATSS, VFL + IoU + DFL,
normalisation) runs on the device with no host synchronisation; failures surface as RuntimeError.
The anchor-aided (loss_fuseab.py) and self-distillation (loss_distill.py) losses subclass it.
"""
import ctypes as C

import torch

from . import _lib
from .assigners import _p, atss_compact, generate_anchors_train, tal_compact

IOU_TYPES = {"giou": 0, "siou": 1, "ciou": 2, "diou": 3}


class LossFn(torch.autograd.Function):
    """Scalar loss whose gradients w.r.t. its tensor inputs were produced by the kernels already: forward returns state['out'][0],
    backward hands out `grads` (one per tensor) scaled by the incoming gradient, in each tensor's dtype."""

    @staticmethod
    def forward(ctx, state, grads, *tensors):
        ctx.save_for_backward(*grads)
        ctx.dtypes = [t.dtype for t in tensors]
        return state["out"][0].clone()

    @staticmethod
    def backward(ctx, grad_out):
        return (None, None, *[(g * grad_out).to(dt) for g, dt in zip(ctx.saved_tensors, ctx.dtypes)])


class ComputeLoss:
    _norm_gt_zero = 0       # subclasses: 1 = divide by target_scores_sum whenever it is > 0 (loss_distill.py:190-191, 318-323)

    def __init__(self, fpn_strides=[8, 16, 32], grid_cell_size=5.0, grid_cell_offset=0.5, num_classes=80,
                 ori_img_size=640, warmup_epoch=4, use_dfl=True, reg_max=16, iou_type='giou',
                 loss_weight={'class': 1.0, 'iou': 2.5, 'dfl': 0.5}):
        self.fpn_strides = list(fpn_strides)
        self.grid_cell_size, self.grid_cell_offset = grid_cell_size, grid_cell_offset
        self.num_classes, self.ori_img_size = num_classes, ori_img_size
        self.warmup_epoch = warmup_epoch
        self.use_dfl, self.reg_max = use_dfl, reg_max
        self.iou_type = iou_type.lower()
        if self.iou_type not in IOU_TYPES:
            raise ValueError(f"unknown iou_type {iou_type}")
        self.loss_weight = loss_weight
        self._anchor_key, self._anchors = None, None
        self.last_assignment = None

    def _build_anchors(self, sizes, device):
        return generate_anchors_train(sizes, self.fpn_strides, device, self.grid_cell_size, self.grid_cell_offset)

    def _get_anchors(self, sizes, device):
        key = (tuple(sizes), str(device))
        if key != self._anchor_key:       # cached like loss.py:63-69
            self._anchors, self._anchor_key = self._build_anchors(sizes, device), key
        return self._anchors

    def __call__(self, outputs, targets, epoch_num, step_num, batch_height, batch_width):
        feats, pred_scores, pred_distri = outputs
        sizes = [tuple(f.shape[2:]) for f in feats]
        state = self.forward_backward(pred_scores, pred_distri, sizes, targets, epoch_num, batch_height, batch_width)
        return LossFn.apply(state, [state["grad_scores"], state["grad_distri"]], pred_scores, pred_distri), state["out"][1:4].detach().clone()

    def forward_backward(self, pred_scores, pred_distri, sizes, targets, epoch_num, batch_height, batch_width, max_gt=None,
                         grad_scores=None, grad_distri=None, grad_scale=1.0, reuse=None, weights=None):
        """Loss value and its gradients w.r.t. the head outputs in one pass (no autograd): returns
        {"out": float64[8] (loss, iou, dfl, cls, target_scores_sum, num_pos), "grad_scores", "grad_distri", "gt_count"}.
        `max_gt` fixes the padded target count G (static shapes for CUDA-graph capture; images with more boxes are
        reported through gt_count > G); otherwise G is the largest per-image count, as in loss.py:184-192 (one small
        host read when `targets` lives on the device).  `grad_*` let the caller provide the output buffers.
        `reuse` = the state of an earlier call: its padded targets and label assignment are used as they are (a second box
        branch scored against the same assignment, loss_distill_ns.py:93,150-160); `weights` overrides the (class, iou, dfl) weights."""
        _lib.require_cuda(pred_scores, "yolov6_b200.ComputeLoss runs")
        dev = pred_scores.device
        anchors, anchor_points, n_list, stride_t = self._get_anchors(sizes, dev)
        B, A, nc = pred_scores.shape
        ps, pd = (t.detach().float().contiguous() for t in (pred_scores, pred_distri))
        strides = stride_t.reshape(-1).contiguous()
        if reuse is not None:       # second box branch against the first call's padded targets and assignment
            st, tg, pboxes = {k: reuse[k] for k in ("gt", "gt_count", "G", "mask", "assignment")}, None, None
        else:
            st, tg = self._pad_targets(targets, B, max_gt, batch_height, batch_width, dev)
            pboxes = torch.empty(B, A, 4, dtype=torch.float32, device=dev)      # in pixels, for the assigner (loss.py:82-83, 94/100)
            _lib.check(_lib.lib().yv6_box_decode(_lib.handle(dev.index or 0), _p(pd), _p(anchor_points), _p(strides), B, A,
                                                 pd.shape[2], 1, _p(pboxes), _lib.stream_ptr()))
            if epoch_num < self.warmup_epoch:
                c = atss_compact(anchors, n_list, st["gt"], st["mask"], pboxes, nc, 9)
            else:
                c = tal_compact(ps, pboxes, anchor_points, st["gt"], st["mask"], 13, 1.0, 6.0)
            st["assignment"] = self.last_assignment = c
        ws = self._det_loss(st, ps, pd, anchor_points, strides, grad_scores, grad_distri, grad_scale, weights)
        st["keep"] = (ps, pd, st["gt"], st["mask"], pboxes, ws, tg)
        return st

    def _pad_targets(self, targets, B, max_gt, batch_height, batch_width, dev):
        """yv6_targets_pad of the [n, 6] (image, class, cx, cy, w, h) rows into a state {"gt": [B, G, 5] float64 (class, xyxy
        in pixels), "gt_count", "G", "mask": uint8 [B, G] of the real rows (loss.py:79)}; also returns the float32 rows read."""
        n = targets.shape[0]
        if max_gt is not None:
            G = max(int(max_gt), 1)
        elif n == 0:
            G = 1
        else:   # loss.py:184-192 pads to the largest per-image count
            img = targets[:, 0].detach()
            valid = img[(img >= 0) & (img < B)].long()
            G = max(int(torch.bincount(valid, minlength=1).max()), 1) if valid.numel() else 1
        tg = targets.detach().float().contiguous().to(dev)
        gt = torch.empty(B, G, 5, dtype=torch.float64, device=dev)
        gt_count = torch.empty(B, dtype=torch.int32, device=dev)
        _lib.check(_lib.lib().yv6_targets_pad(_lib.handle(dev.index or 0), _p(tg), n, B, G, float(batch_width), float(batch_height),
                                              _p(gt), _p(gt_count), _lib.stream_ptr()))
        mask = (gt[:, :, 1:].sum(-1) > 0).to(torch.uint8).contiguous()
        return {"gt": gt, "gt_count": gt_count, "G": G, "mask": mask}, tg

    def _det_loss(self, st, ps, pd, anchor_points, strides, grad_scores=None, grad_distri=None, grad_scale=1.0, weights=None):
        """yv6_det_loss of scores `ps` and box predictions `pd` (reg_ch = pd.shape[2]) against the state's targets and assignment:
        adds "out" and the gradient buffers "grad_scores" / "grad_distri" (new unless given) to the state; returns the workspace."""
        B, A, nc = ps.shape
        dev, lib, c = ps.device, _lib.lib(), st["assignment"]
        grad_scores = torch.empty_like(ps) if grad_scores is None else grad_scores
        grad_distri = torch.empty_like(pd) if grad_distri is None else grad_distri
        out = torch.zeros(8, dtype=torch.float64, device=dev)
        ws = torch.empty(int(lib.yv6_det_loss_workspace_bytes(B, A)), dtype=torch.uint8, device=dev)
        w = [float(v) for v in (weights if weights is not None else [self.loss_weight[k] for k in ("class", "iou", "dfl")])]
        d = _lib.LossDesc(pred_scores=ps.data_ptr(), pred_distri=pd.data_ptr(), anc_points=anchor_points.data_ptr(), strides=strides.data_ptr(),
                          gt=st["gt"].data_ptr(), gt_idx=c.gt_idx.data_ptr(), fg=c.fg.data_ptr(), norm=c.norm.data_ptr(),
                          B=B, A=A, G=st["G"], nc=nc, reg_ch=pd.shape[2], iou_type=IOU_TYPES[self.iou_type],
                          w_cls=w[0], w_iou=w[1], w_dfl=w[2], grad_scale=float(grad_scale),
                          grad_scores=grad_scores.data_ptr(), grad_distri=grad_distri.data_ptr(), out=out.data_ptr(),
                          workspace=ws.data_ptr(), workspace_bytes=ws.numel(), norm_gt_zero=self._norm_gt_zero)
        _lib.check(lib.yv6_det_loss(_lib.handle(dev.index or 0), C.byref(d), _lib.stream_ptr()))
        st.update(out=out, grad_scores=grad_scores, grad_distri=grad_distri)
        return ws
