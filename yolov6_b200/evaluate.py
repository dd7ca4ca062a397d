"""Validating the training EMA between epochs: the reference Trainer's `after_epoch` evaluation (yolov6/core/engine.py:178-220)
on captured pipelines whose weights are refolded in place.

`is_val_epoch` is the Trainer's schedule (engine.py:184-186).  `EpochEval` is built once, on the rank that evaluates, from an
eval Model of the training config: it keeps one DetectPipeline per distinct ValFeed canvas across epochs (built on first use)
and `run(opt)` loads the FusedSGDEMA's EMA into it with Model.load_weights_ -- one yv6_fold launch per engine, no host copy,
no recapture -- streams every validation batch through the pipelines into the metric and returns (map50, map) with the
metric's full result.  A refold refused because a BottleRep alpha changed (refold.AlphaChanged) rebuilds the pipelines and
sets `rebuilt`.
"""
from .cocoeval import COCOMetric
from .pipeline import DetectPipeline
from .refold import AlphaChanged


def is_val_epoch(epoch, max_epoch, eval_interval, heavy_eval_range, eval_final_only):
    """Trainer.after_epoch's condition (engine.py:184-186): always after the final epoch, every `eval_interval` epochs
    before the last `heavy_eval_range` ones and at least every 3 inside them, only the final one with eval_final_only."""
    remaining = max_epoch - 1 - epoch
    interval = eval_interval if remaining >= heavy_eval_range else min(3, eval_interval)
    return remaining == 0 or ((not eval_final_only) and (epoch + 1) % interval == 0)


class EpochEval:
    """Per-epoch validation of an EMA on captured pipelines.

    model: an eval Model of the training config (its precision is the evaluation's: "fp32" is the reference's Evaler, which
    runs the EMA unfused in fp32; "bf16" the fast choice); feed: the ValFeed of the validation set; frames(indices) ->
    (frames, labels) of those source indices (host frames, CUDA tensors or a device cache, as ValFeed.feed takes them);
    metric: a COCOMetric (updated with image_ids[i], default the source index i) or a PRMetric; nms_kw: the Evaler's NMS
    (conf 0.03, iou 0.65, multi_label)."""

    def __init__(self, model, feed, frames, metric, image_ids=None, conf_thres=0.03, iou_thres=0.65, multi_label=True,
                 max_det=300):
        self.model = model.eval()
        self.feed, self.frames, self.metric = feed, frames, metric
        self.image_ids = image_ids
        self.nms_kw = dict(conf_thres=conf_thres, iou_thres=iou_thres, multi_label=multi_label, max_det=max_det)
        self.pipes = {}           # canvas (H, W) -> DetectPipeline, kept across epochs
        self.rebuilt = False      # the last run rebuilt its pipelines (an alpha changed)

    def pipeline(self, H, W):
        p = self.pipes.get((H, W))
        if p is None:
            p = self.pipes[H, W] = DetectPipeline(self.model, self.feed.batch, H, W, host_input=False, **self.nms_kw)
        return p

    def run(self, src):
        """One validation pass at the weights of `src` (a FusedSGDEMA, a state_dict or (flat, slots): Model.load_weights_).
        Returns ((map50, map), result): COCOMetric -> COCOResult, map = stats[0] and map50 = stats[1]; PRMetric -> PRResult,
        its map50 / map (the Evaler's pr_metric_result, evaler.py:203-205)."""
        self.rebuilt = False
        try:
            self.model.load_weights_(src)
        except AlphaChanged:      # the parameters are loaded; the engine and every pipeline are rebuilt at them
            self.pipes.clear()
            self.rebuilt = True
        m, coco = self.metric, isinstance(self.metric, COCOMetric)
        m.reset()
        for idx in self.feed.batches():
            frames, labels = self.frames(idx)
            canvas, targets, shapes, n = self.feed.feed(idx, frames, labels)
            H, W = canvas.shape[2:]
            p = self.pipeline(H, W)
            p.x_dev.copy_(canvas)              # uint8 -> the fp32 input, still 0..255 (the stem scales)
            p.launch()
            out, count = p.out_dev[:n].contiguous(), p.count_dev[:n].contiguous()
            if coco:
                m.update(out, count, shapes, [int(i) if self.image_ids is None else self.image_ids[int(i)] for i in idx])
            else:
                m.update(out, count, targets, shapes, (H, W))
        res = m.result()
        if coco:
            return (float(res.stats[1]), float(res.stats[0])), res
        return (float(res.map50), float(res.map)), res
