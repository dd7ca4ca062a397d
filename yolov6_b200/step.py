"""One training step as a replayed CUDA graph (SURVEY.md 8f N1).

`Trainer.train_in_steps` (core/engine.py:142-176) is, per batch: H2D copy + `.float()/255` (prepro_data, :407-410),
forward under autocast, ComputeLoss (host-side target padding, :184-192 of loss.py), `loss * world_size`, backward
through autograd with DDP's bucketed all-reduce, GradScaler, SGD step, EMA update -- several thousand kernel launches
and a handful of host synchronisations.  `TrainStep` runs the same arithmetic as

    copy images (uint8 or fp32) and padded targets into static buffers
    -> graph segment 0: clear accumulators, repack weights, forward, assignment + loss + its gradients, backward of
       the ops of gradient bucket 0, unpack bucket 0
    -> [all-reduce bucket 0 on the communication stream]  ||  graph segment 1: backward of bucket 1 ...
    -> wait for the all-reduces -> fused SGD + EMA kernel

with static shapes: batch, image size, at most `max_targets` target rows per batch and `max_gt` boxes per image
(rows beyond that are dropped and reported by `overflowed()`).  Gradients are the SUM over ranks of the per-rank
gradients, which is what the reference's `loss * world_size` + DDP averaging produce (core/engine.py:171-172,464-466);
bf16 storage has fp32's exponent range, so no GradScaler is needed.

Self-distillation (`--distill`, core/engine.py:153-159): with `teacher=` a model and `compute_loss` a
`loss_distill.ComputeLoss[NS]`, segment 0 forks the teacher's forward-only plan (`Model.teacher_engine`: batch statistics,
running statistics untouched, as get_teacher_model's `track_running_stats = False`, core/engine.py:429-441) onto a stream of its
own next to the student's forward -- both read the same input buffer -- joins it, and computes the detection loss, the two
KL terms (and the lrtb IoU term of ComputeLossNS, the channel-wise term with `distill_feat`) into the student's gradient
buffers.  The KL weights decay with the epoch (loss_distill.py:196), so the graphs are captured once per epoch.

Several canvases (`--rect` batches, core/engine.py:151): `shapes=[(H, W), ...]`, each inside the step's height x width, plans
every shape over one set of activation, gradient and head-output buffers sized for the largest (`TrainEngine.plan_shapes`)
and keeps the graphs of every (shape, assigner branch) once captured.  `use_shape` / `load` pick the next batch's shape; the
loss normalises its targets with that H and W.  Weights, the flat gradient buckets, the optimizer and the all-reduce are
shared.  The shared buffers are cleared when the shape changes, so a shape's step computes what a step built for it alone
computes.  Distillation takes one shape only.
"""
import torch
import torch.distributed as dist

from . import _lib, loss_distill
from .dist import GradSync


class TrainStep:
    def __init__(self, model, compute_loss, batch, height, width, in_dtype=torch.float32, max_targets=None, max_gt=64,
                 optimizer=None, n_buckets=None, graph=True, group=None, compute_loss_ab=None, teacher=None, temperature=20.0,
                 max_epoch=None, shapes=None):
        self.fuse_ab = bool(getattr(model, "fuse_ab", False))
        self.distill = isinstance(compute_loss, loss_distill.ComputeLoss)
        if self.distill or teacher is not None:
            _check_distill(model, compute_loss, teacher, max_epoch)
        if self.fuse_ab and compute_loss_ab is None:
            raise ValueError("a fuse_ab model needs compute_loss_ab (yolov6_b200.loss_fuseab.ComputeLoss): core/engine.py:161-166 adds "
                             "the anchor-aided loss to the anchor-free one")
        self.model = model.train()
        self.loss = compute_loss
        self.loss_ab = compute_loss_ab
        self.dev = next(model.parameters()).device
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        if n_buckets is None:
            n_buckets = 3 if self.world > 1 else 1
        self.eng = model.train_engine(n_buckets=n_buckets)
        self.B, self.H, self.W, self.in_dtype = batch, height, width, in_dtype
        self.max_gt = int(max_gt)
        self.max_targets = int(max_targets or batch * max_gt)
        self.targets = torch.full((self.max_targets, 6), -1.0, dtype=torch.float32, device=self.dev)
        if self.distill and self.loss.distill_feat != self.eng.external_feat_grads:
            self.eng.external_feat_grads = self.loss.distill_feat     # the neck outputs' gradients come from the channel-wise term
            self.eng._shape = None
        self.shapes = None
        if shapes is not None:      # several (H, W) canvases (--rect): one arena sized for the largest, graphs per shape
            self.shapes = list(dict.fromkeys([(int(height), int(width))] + [(int(h), int(w)) for h, w in shapes]))
            for h, w in self.shapes:
                if h > height or w > width:
                    raise ValueError(f"shape {h}x{w} does not fit inside the step's {height}x{width}: every rect canvas "
                                     f"(pad 0) fits inside img_size x img_size")
            if teacher is not None and len(self.shapes) > 1:
                raise ValueError(f"distillation over several shapes ({self.shapes}) is not supported: build one TrainStep "
                                 f"per shape")
            self.eng.plan_shapes(batch, self.shapes, in_dtype)
        self.eng._plan(batch, height, width, in_dtype)
        self.images = self.eng.x_static
        self.teacher = teacher
        if teacher is not None:
            self.teng = teacher.teacher_engine()
            self.teng._plan(batch, height, width, in_dtype, x_static=self.images)
            self.t_stream = torch.cuda.Stream(device=self.dev)
            self.temperature, self.max_epoch = float(temperature), max_epoch
        self.opt = optimizer
        self.sync = GradSync(self.eng.flat.gflat, self.eng.bucket_range, group) if self.world > 1 else None
        self.use_graph = bool(graph)
        self.graphs = {}           # (assigner branch (True = ATSS warm-up), epoch when distilling[, (H, W)]) -> list of graph segments
        self.states = {}           # with shapes: the same key -> the loss state its graphs write, and the anchors they read
        self.captures = 0
        self.state = None
        self.accumulate = False
        self.sizes = self.eng.sizes

    # ------------------------------------------------------------------ the step body, in bucket-sized segments
    def _segments(self):
        cuts = self.eng.bucket_call_index()
        return [0] + cuts[:-1], cuts[:-1] + [len(self.eng.bwd_calls)]

    def _segment(self, j, epoch_num):
        eng = self.eng
        firsts, lasts = self._segments()
        if j == 0:
            sp = _lib.stream_ptr()
            eng.begin_step(sp)
            eng.flat.iflat.add_(1)
            if self.distill:
                self._distill_forward_loss(sp, epoch_num)
            else:
                eng.run_forward(sp)
                self.state = self.loss.forward_backward(eng.cls, eng.reg, self.sizes, self.targets, epoch_num, self.H, self.W,
                                                        max_gt=self.max_gt, grad_scores=eng.grad_cls, grad_distri=eng.grad_reg)
            if self.fuse_ab:      # total_loss += total_loss_ab; loss_items += loss_items_ab (core/engine.py:164-166)
                st_ab = self.loss_ab.forward_backward(eng.cls_ab, eng.reg_ab, self.sizes, self.targets, epoch_num, self.H, self.W,
                                                      max_gt=self.max_gt, grad_scores=eng.grad_cls_ab, grad_distri=eng.grad_reg_ab)
                self.state["out_af"], self.state["out_ab"] = self.state["out"], st_ab["out"]
                total = self.state["out"].clone()
                total[:4] += st_ab["out"][:4]
                self.state["out"] = total
                self.state["keep_ab"] = st_ab
        eng.backward(None, None, accumulate=self.accumulate, first=firsts[j], last=lasts[j])

    def _distill_forward_loss(self, sp, epoch_num):
        """Segment 0 of a distillation step after the student's begin_step: teacher forward on its own stream || student forward,
        join, then the distillation loss into the student's gradient buffers."""
        eng, teng = self.eng, self.teng
        main = torch.cuda.current_stream(self.dev)
        fork, join = torch.cuda.Event(), torch.cuda.Event()
        fork.record(main)
        self.t_stream.wait_event(fork)
        with torch.cuda.stream(self.t_stream):
            tsp = _lib.stream_ptr(self.t_stream)
            teng.begin_step(tsp)
            teng.run_forward(tsp)
        join.record(self.t_stream)
        eng.run_forward(sp)
        main.wait_event(join)
        s_feats = t_feats = ()
        if self.loss.distill_feat:
            s_feats, t_feats = eng.neck_outputs(), teng.neck_outputs()
        kw = dict(max_gt=self.max_gt, grad_scores=eng.grad_cls)
        if eng.g.distill_ns:       # DFL logits for the loss and the KL term, lrtb distances for the second IoU term
            kw.update(grad_distri=eng.grad_reg_dist, pred_lrtb=eng.reg, grad_lrtb=eng.grad_reg)
            distri = eng.reg_dist
        else:
            kw.update(grad_distri=eng.grad_reg)
            distri = eng.reg
        self.state = self.loss.distill_forward_backward(eng.cls, distri, teng.cls, teng.reg, self.sizes, self.targets, epoch_num,
                                                        self.max_epoch, self.temperature, self.H, self.W, s_feats, t_feats, **kw)
        if self.loss.distill_feat:
            eng._feat_grads = self.state["feat_grads"]

    def _capture(self, epoch_num):
        nseg = len(self._segments()[0])
        fl = self.eng.flat
        snap = (fl.pflat.clone(), fl.gflat.clone(), fl.iflat.clone())   # warm-up runs must not train: running statistics,
        side = torch.cuda.Stream(device=self.dev)                       # batch counters and accumulated gradients are restored
                                                                        # (a teacher's plan writes none of its model's state)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            for _ in range(2):                      # plans, tensor maps, cudaFuncSetAttribute, allocator warm-up
                for j in range(nseg):
                    self._segment(j, epoch_num)
        torch.cuda.current_stream(self.dev).wait_stream(side)
        fl.pflat.copy_(snap[0])
        fl.gflat.copy_(snap[1])
        fl.iflat.copy_(snap[2])
        del snap
        torch.cuda.synchronize(self.dev)
        graphs = []
        pool = None
        for j in range(nseg):
            gph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gph, pool=pool):
                self._segment(j, epoch_num)
            pool = gph.pool()
            graphs.append(gph)
        self.captures += 1
        return graphs

    def _planned_here(self):
        """With shapes: the engine planned at the current shape, its arena holding that shape's tensors."""
        self.eng._plan(self.B, self.H, self.W, self.in_dtype)
        self.eng.make_live(self.H, self.W)
        self.sizes = self.eng.sizes

    # ------------------------------------------------------------------ public
    def use_shape(self, height, width):
        """A step built with `shapes`: makes (height, width) the shape of the next `load` / `run`; `images` becomes that
        shape's input view (an AugmentFeed writes the batch there)."""
        if self.shapes is None or (int(height), int(width)) not in self.shapes:
            raise ValueError(f"shape {height}x{width} is not one of this step's shapes {self.shapes}")
        self.H, self.W = int(height), int(width)
        self.images = self.eng.x_store[:self.B * 3 * self.H * self.W].view(self.B, 3, self.H, self.W)

    def load(self, images, targets):
        """images: [B,3,H,W] (host or device; pinned host memory makes the copy asynchronous); targets: [n,6] fp32
        (img, cls, cx, cy, w, h normalised), n <= max_targets.  A step built with `shapes` takes any of them."""
        if self.shapes is not None:
            self.use_shape(*images.shape[2:])
        self.images.copy_(images, non_blocking=True)
        n = int(targets.shape[0])
        if n > self.max_targets:
            raise RuntimeError(f"{n} target rows exceed max_targets={self.max_targets}")
        self.targets[:n].copy_(targets, non_blocking=True)
        if n < self.max_targets:
            self.targets[n:].fill_(-1.0)             # rows with image index -1 are ignored by yv6_targets_pad

    def run(self, epoch_num=0, accumulate=False):
        """Forward + loss + backward (+ gradient all-reduce).  Returns the device tensor float64[8] =
        (loss, iou, dfl, cls, target_scores_sum, num_pos, cwd, 0) of this rank -- no host synchronisation.  With a teacher,
        iou / dfl / cls include the distillation terms and cwd is the channel-wise one: out[[1, 2, 3, 6]] are the reference's
        loss_items (iou, dfl, cls, cwd); cwd is 0 otherwise."""
        if self.teacher is not None and not self.teng.flat.valid():
            raise RuntimeError("the teacher's tensors were replaced after the step was built (model.to / .half / a train_engine "
                               "of its own); build the TrainStep again")
        key = (epoch_num < self.loss.warmup_epoch, epoch_num if self.distill else None)
        if self.shapes is not None:   # graphs of every shape are kept; the arena is cleared when the shape changes
            key += ((self.H, self.W),)
            if not self.use_graph or accumulate != self.accumulate or key not in self.graphs:
                if accumulate != self.accumulate:
                    self.graphs, self.states = {}, {}
                self._planned_here()
            else:
                self.eng.make_live(self.H, self.W)
        nseg = len(self._segments()[0])
        if self.use_graph:
            if accumulate != self.accumulate or key not in self.graphs:
                self.accumulate = accumulate
                if self.shapes is None:
                    self.graphs = {key: self._capture(epoch_num)}
                else:
                    self.graphs[key] = self._capture(epoch_num)
                    self.states[key] = (self.state, self.loss._anchors, getattr(self.loss_ab, "_anchors", None))
            if self.shapes is not None:
                self.state = self.states[key][0]
            graphs = self.graphs[key]
        for j in range(nseg):
            if self.use_graph:
                graphs[j].replay()
            else:
                self.accumulate = accumulate
                self._segment(j, epoch_num)
            if self.sync is not None:
                self.sync.bucket_ready(j)
        if self.sync is not None:
            self.sync.finish()
        return self.state["out"]

    def step(self, images=None, targets=None, epoch_num=0):
        """load -> run -> optimizer (when one was given)."""
        if images is not None:
            self.load(images, targets)
        out = self.run(epoch_num)
        if self.opt is not None:
            self.opt.step()
        return out

    def overflowed(self):
        """True when the last batch had an image with more than max_gt boxes (host read)."""
        return bool((self.state["gt_count"] > self.max_gt).any().item())


def _check_distill(student, compute_loss, teacher, max_epoch):
    """The combinations core/engine.py:153-167, 305-322 and 429-441 allow: a distillation loss with a teacher of the same head,
    ComputeLossNS exactly for a distill_ns student, no fuse_ab student."""
    if not isinstance(compute_loss, loss_distill.ComputeLoss) or teacher is None:
        raise ValueError("self-distillation needs both a teacher model and a loss_distill.ComputeLoss / ComputeLossNS")
    if getattr(student, "fuse_ab", False):
        raise ValueError("a fuse_ab student cannot be distilled: --distill and --fuse_ab are exclusive (core/engine.py:153-167)")
    ns = bool(getattr(student, "distill_ns", False))
    if ns != isinstance(compute_loss, loss_distill.ComputeLossNS):
        raise ValueError("a distill_ns student takes loss_distill.ComputeLossNS, any other student loss_distill.ComputeLoss "
                         "(core/engine.py:305-322)")
    if max_epoch is None:
        raise ValueError("distillation needs max_epoch: the KL weights decay over the epochs (loss_distill.py:196)")
    sg, tg = student.graph, teacher.graph
    s_reg = sg.dist_reg_ch if ns else 4 * (sg.reg_max + 1)
    t_reg = 4 * (tg.reg_max + 1)
    if (sg.num_classes, s_reg, list(sg.strides)) != (tg.num_classes, t_reg, list(tg.strides)):
        raise ValueError(f"teacher head (classes {tg.num_classes}, box channels {t_reg}, strides {list(tg.strides)}) differs from the "
                         f"student's (classes {sg.num_classes}, box channels {s_reg}, strides {list(sg.strides)})")
    if compute_loss.distill_feat and [t.c for t in sg.feat[:3]] != [t.c for t in tg.feat[:3]]:
        raise ValueError("distill_feat needs teacher neck outputs with the student's channel counts")
