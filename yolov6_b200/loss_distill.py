"""Drop-in `ComputeLoss` of the self-distillation recipe for the M / L models (SURVEY.md 8f N3, second half).

Same constructor and call signature as yolov6/models/losses/loss_distill.py:14-211, which the Trainer uses with
`--distill` (core/engine.py:153-159, 311-322):

    preds, s_featmaps = model(images)
    with torch.no_grad():
        t_preds, t_featmaps = teacher_model(images)
    loss, items = compute_loss_distill(preds, t_preds, s_featmaps, t_featmaps, targets, epoch_num, max_epoch, temperature,
                                       step_num, batch_height, batch_width)

= the anchor-free detection loss (with the "> 0" normalisation rule of :190-191, 318-323)
  + distill_weight['class'] * decay * T^2 KL(softmax(t_scores / T) || softmax(s_scores / T))        summed over all anchors (:213-222)
  + distill_weight['dfl']   * decay * T^2 mean KL over the 4 x 17-bin side distributions of the positives (:351-361),
    multiplied by sum(bbox_weight) / target_scores_sum (= 1, or 0 when no target score is positive; :318-323)
with decay = ((1 - cos(epoch * pi / max_epoch)) / 2) * (0.01 - 1) + 1 (:196).  The detection part is `yv6_det_loss` (value +
gradients in one launch); the two KL terms are `yv6_kl_rows`, which adds its gradients to the same buffers.  The channel-wise
feature-map term (`distill_feat=True`, :223-245) is the same kernel over (image, channel) rows of H*W positions; it needs the real,
differentiable neck outputs: set `model.return_featmaps = True` on the student and the teacher.  `ComputeLossNS` below is the N / S variant (loss_distill_ns.py, for the
student head of effidehead_distill_ns.py).
"""
import math

import torch

from . import _lib
from .assigners import _p
from .loss import ComputeLoss as _DetLoss, LossFn


class ComputeLoss(_DetLoss):
    _norm_gt_zero = 1

    def __init__(self, fpn_strides=[8, 16, 32], grid_cell_size=5.0, grid_cell_offset=0.5, num_classes=80, ori_img_size=640,
                 warmup_epoch=0, use_dfl=True, reg_max=16, iou_type='giou',
                 loss_weight={'class': 1.0, 'iou': 2.5, 'dfl': 0.5, 'cwd': 10.0},
                 distill_feat=False, distill_weight={'class': 1.0, 'dfl': 1.0}):
        super().__init__(fpn_strides, grid_cell_size, grid_cell_offset, num_classes, ori_img_size, warmup_epoch, use_dfl, reg_max,
                         iou_type, loss_weight)
        self.distill_feat = bool(distill_feat)       # needs `model.return_featmaps = True` on student and teacher (real neck outputs)
        self.distill_weight = distill_weight

    def _cw_term(self, s_featmaps, t_featmaps, decay, terms):
        """distill_loss_cw (:223-245), temperature 1: per level KL over the H*W positions of every (image, channel) row, / (N*C).
        Returns the gradients w.r.t. the student's feature maps; adds the weighted term to terms[2]."""
        if len(s_featmaps) < 3 or any(f.dim() != 4 or f.shape[1] <= 1 for f in s_featmaps[:3]):
            raise RuntimeError("distill_feat needs the real neck outputs: set model.return_featmaps = True on the student and the teacher")
        lib = _lib.lib()
        grads = []
        for sf, tf in zip(s_featmaps[:3], t_featmaps[:3]):      # the reference sums levels 0..2
            N, C, H, W = sf.shape
            s32, t32 = sf.detach().float().contiguous(), tf.detach().float().contiguous()
            if t32.shape != s32.shape:
                raise RuntimeError(f"teacher feature map {tuple(t32.shape)} vs student {tuple(s32.shape)}")
            g = torch.zeros_like(s32)
            scale = float(self.loss_weight['cwd']) * decay / float(N * C)
            _lib.check(lib.yv6_kl_rows(_lib.handle(sf.device.index or 0), _p(s32), _p(t32), N * C, H * W, 1.0, 0, 1, scale, 0, 0,
                                       terms.data_ptr() + 16, _p(g), _lib.stream_ptr()))
            grads.append(g)
        return grads

    def distill_forward_backward(self, pred_scores, pred_distri, t_pred_scores, t_pred_distri, sizes, targets, epoch_num, max_epoch,
                                 temperature, batch_height, batch_width, s_featmaps=(), t_featmaps=(), max_gt=None, grad_scores=None,
                                 grad_distri=None):
        """The whole loss and its gradients on the device (no autograd, no host read), as `forward_backward` is for the detection
        loss: returns its state with "out" = float64[8] (loss, iou, dfl, cls, target_scores_sum, num_pos, cwd, 0) -- iou / dfl / cls
        include the distillation terms as in loss_items -- and "feat_grads", the NCHW fp32 gradients w.r.t. s_featmaps[:3]
        (distill_feat).  `max_gt` and `grad_*` as in forward_backward: step.TrainStep passes its engine's buffers."""
        state = self.forward_backward(pred_scores, pred_distri, sizes, targets, epoch_num, batch_height, batch_width, max_gt=max_gt,
                                      grad_scores=grad_scores, grad_distri=grad_distri)
        dev = pred_scores.device
        lib, h, sp = _lib.lib(), _lib.handle(dev.index or 0), _lib.stream_ptr()
        B, A, nc = pred_scores.shape
        ps, pd = state["keep"][0], state["keep"][1]
        ts = t_pred_scores.detach().float().contiguous()
        td = t_pred_distri.detach().float().contiguous()
        if ts.shape != ps.shape or td.shape != pd.shape:
            raise RuntimeError(f"teacher outputs {tuple(ts.shape)}, {tuple(td.shape)} do not match the student's {tuple(ps.shape)}, {tuple(pd.shape)}")
        decay = ((1 - math.cos(epoch_num * math.pi / max_epoch)) / 2) * (0.01 - 1) + 1          # :196
        T = float(temperature)
        w_cls, w_dfl = float(self.loss_weight['class']), float(self.loss_weight['dfl'])
        terms = torch.zeros(3, dtype=torch.float64, device=dev)                 # weighted d_loss_cls, d_loss_dfl, d_loss_cw
        out = state["out"]
        s_cls = w_cls * float(self.distill_weight['class']) * decay * T * T
        _lib.check(lib.yv6_kl_rows(h, _p(ps), _p(ts), B * A, nc, T, 0, 1, s_cls, 0, 0, terms.data_ptr(), _p(state["grad_scores"]), sp))
        if self.use_dfl:
            R = self.reg_max + 1
            s_dfl = w_dfl * float(self.distill_weight['dfl']) * decay * T * T
            fg = self.last_assignment.fg
            # rows = (anchor, side); active = positives; mean over 4 * num_pos rows (out[5]); zero unless target_scores_sum (out[4]) > 0
            _lib.check(lib.yv6_kl_rows(h, _p(pd), _p(td), B * A * 4, R, T, _p(fg), 4, s_dfl, out.data_ptr() + 5 * 8, out.data_ptr() + 4 * 8,
                                       terms.data_ptr() + 8, _p(state["grad_distri"]), sp))
        feat_grads = self._cw_term(s_featmaps, t_featmaps, decay, terms) if self.distill_feat else []
        total = out.clone()
        total[0] = out[0] + terms[0] + terms[1] + terms[2]
        total[2] = out[2] + terms[1]               # loss_weight['dfl'] * loss_dfl_all
        total[3] = out[3] + terms[0]               # loss_weight['class'] * loss_cls_all
        total[6] = terms[2]
        state["out"] = total
        state["keep_distill"] = (ts, td, terms)
        state["feat_grads"] = feat_grads
        return state

    def __call__(self, outputs, t_outputs, s_featmaps, t_featmaps, targets, epoch_num, max_epoch, temperature, step_num,
                 batch_height, batch_width):
        feats, pred_scores, pred_distri = outputs
        t_pred_scores, t_pred_distri = t_outputs[-2], t_outputs[-1]            # loss_distill.py:76 (a fuse_ab teacher returns five)
        sizes = [tuple(f.shape[2:]) for f in feats]
        state = self.distill_forward_backward(pred_scores, pred_distri, t_pred_scores, t_pred_distri, sizes, targets, epoch_num, max_epoch,
                                              temperature, batch_height, batch_width, s_featmaps, t_featmaps)
        loss = LossFn.apply(state, [state["grad_scores"], state["grad_distri"]] + state["feat_grads"], pred_scores, pred_distri,
                            *list(s_featmaps[:3] if self.distill_feat else []))
        return loss, _items(state["out"])


def _items(out):
    """(iou, dfl_all, cls_all, cwd): the reference's loss_items."""
    return torch.cat([out[1:4], out[6:7]]).detach()


class ComputeLossNS(ComputeLoss):
    """yolov6/models/losses/loss_distill_ns.py:14-211 -- the N / S recipe: the student head (heads/effidehead_distill_ns.py) emits
    DFL distributions for the distillation and plain (l, r, t, b) distances for inference; the loss is the M / L one on
    (scores, distributions) -- TaskAlignedAssigner at every epoch (:95-103) -- plus a second IoU term of the lrtb boxes against
    the same assignment (BboxLoss :283-292, `loss_iou + loss_iou_lrtb`)."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.warmup_epoch = 0          # loss_distill_ns.py never calls its warm-up assigner

    def distill_forward_backward(self, pred_scores, pred_distri, t_pred_scores, t_pred_distri, sizes, targets, epoch_num, max_epoch,
                                 temperature, batch_height, batch_width, s_featmaps=(), t_featmaps=(), max_gt=None, grad_scores=None,
                                 grad_distri=None, pred_lrtb=None, grad_lrtb=None):
        """ComputeLoss.distill_forward_backward plus the IoU term of the lrtb branch `pred_lrtb` (its gradient into `grad_lrtb`,
        when given) against the same targets and assignment: no class or DFL term (reg_ch = 4)."""
        state = super().distill_forward_backward(pred_scores, pred_distri, t_pred_scores, t_pred_distri, sizes, targets, epoch_num,
                                                 max_epoch, temperature, batch_height, batch_width, s_featmaps, t_featmaps, max_gt,
                                                 grad_scores, grad_distri)
        st2 = self.forward_backward(pred_scores, pred_lrtb, sizes, targets, epoch_num, batch_height, batch_width, reuse=state,
                                    grad_distri=grad_lrtb, weights=(0.0, float(self.loss_weight['iou']), 0.0))
        total = state["out"].clone()
        total[:2] += st2["out"][:2]
        # (the class-score gradient of the second call is exactly zero: w_cls = 0)
        return dict(state, out=total, keep_lrtb=st2)

    def __call__(self, outputs, t_outputs, s_featmaps, t_featmaps, targets, epoch_num, max_epoch, temperature, step_num,
                 batch_height, batch_width):
        feats, pred_scores, pred_distri, pred_lrtb = outputs
        sizes = [tuple(f.shape[2:]) for f in feats]
        state = self.distill_forward_backward(pred_scores, pred_distri, t_outputs[-2], t_outputs[-1], sizes, targets, epoch_num, max_epoch,
                                              temperature, batch_height, batch_width, s_featmaps, t_featmaps, pred_lrtb=pred_lrtb)
        grads = [state["grad_scores"], state["grad_distri"], state["keep_lrtb"]["grad_distri"]] + state["feat_grads"]
        loss = LossFn.apply(state, grads, pred_scores, pred_distri, pred_lrtb, *list(s_featmaps[:3] if self.distill_feat else []))
        return loss, _items(state["out"])
