"""Drop-in model API: `build_model(cfg, num_classes, device)` -> nn.Module with the reference's
surface (yolov6/models/yolo.py:14-47,136-138; yolov6/models/effidehead.py:10-65):

  * `.backbone`, `.neck`, `.detect`, `.stride`; `state_dict()` keys/shapes identical to the reference
    (checkpoints load unchanged; the module stays picklable -- it holds only parameters + the config);
  * `forward(x)` in eval mode returns `[pred [B,A,5+nc], featmaps]` like Model.forward (`pred` alone
    when `export` is set), computed by the sm_90a engine (engine.py) from folded deploy weights;
  * `Detect` keeps nc/no/nl/stride/grid/use_dfl/reg_max/proj/proj_conv/prior_prob, the ModuleLists
    stems/cls_convs/reg_convs/cls_preds/reg_preds and `initialize_biases()`.

Parameters live in a tree of plain containers with real nn.Conv2d / nn.BatchNorm2d /
nn.ConvTranspose2d leaves generated from the layer graph (arch.py); nothing here executes a
PyTorch convolution -- there is no eager fallback.
"""
import math

import torch
import torch.nn as nn

from . import arch, configs
from .engine import InferEngine


class Node(nn.Module):
    """Generic parameter container; numeric children behave like an nn.ModuleList."""

    def __getitem__(self, i):
        return self._modules[str(i)]

    def __len__(self):
        return len(self._modules)

    def __iter__(self):
        return iter(self._modules.values())

    def forward(self, *a, **k):
        raise RuntimeError("yolov6_b200 sub-modules are parameter containers; call the Model (its engine "
                           "runs the whole network as sm_90a kernels)")


def _ensure(root, path, cls=Node):
    node = root
    for part in path:
        if part not in node._modules:
            node.add_module(part, cls())
        node = node._modules[part]
    return node


class Detect(Node):
    """Efficient decoupled head (effidehead.py:10-65) -- attributes and bias initialisation."""
    export = False

    def __init__(self, num_classes=80, num_layers=3, use_dfl=True, reg_max=16):
        super().__init__()
        self.nc = num_classes
        self.no = num_classes + 5
        self.nl = num_layers
        self.grid = [torch.zeros(1)] * num_layers
        self.prior_prob = 1e-2
        self.inplace = True
        self.stride = torch.tensor([8, 16, 32] if num_layers == 3 else [8, 16, 32, 64])
        self.use_dfl = use_dfl
        self.reg_max = reg_max
        self.grid_cell_offset = 0.5
        self.grid_cell_size = 5.0

    def initialize_biases(self):
        """effidehead.py:49-65: cls bias = -log((1-p)/p), reg bias = 1, pred weights = 0, proj = 0..reg_max."""
        for conv in self.cls_preds:
            conv.bias.data.fill_(-math.log((1 - self.prior_prob) / self.prior_prob))
            conv.weight.data.fill_(0.)
        for conv in self.reg_preds:
            conv.bias.data.fill_(1.0)
            conv.weight.data.fill_(0.)
        if "reg_preds_dist" in self._modules:       # effidehead_distill_ns.py:59-66
            for conv in self.reg_preds_dist:
                conv.bias.data.fill_(1.0)
                conv.weight.data.fill_(0.)
        if "cls_preds_ab" in self._modules:         # effidehead_fuseab.py:65-87
            for conv in self.cls_preds_ab:
                conv.bias.data.fill_(-math.log((1 - self.prior_prob) / self.prior_prob))
                conv.weight.data.fill_(0.)
            for conv in self.reg_preds_ab:
                conv.bias.data.fill_(1.0)
                conv.weight.data.fill_(0.)
        self.proj.data.copy_(torch.linspace(0, self.reg_max, self.reg_max + 1))
        self.proj_conv.weight.data.copy_(self.proj.view(1, self.reg_max + 1, 1, 1))


class LiteDetect(Node):
    """The YOLOv6Lite head (effidehead_lite.py:10-56): no DFL, so no use_dfl / reg_max / proj / proj_conv."""
    export = False

    def __init__(self, num_classes=80, num_layers=4):
        super().__init__()
        self.nc = num_classes
        self.no = num_classes + 5
        self.nl = num_layers
        self.grid = [torch.zeros(1)] * num_layers
        self.prior_prob = 1e-2
        self.inplace = True
        self.stride = torch.tensor([8, 16, 32] if num_layers == 3 else [8, 16, 32, 64])
        self.grid_cell_offset = 0.5
        self.grid_cell_size = 5.0

    def initialize_biases(self):
        """effidehead_lite.py:46-56: cls bias = -log((1-p)/p), reg bias = 1, pred weights = 0."""
        for conv in self.cls_preds:
            conv.bias.data.fill_(-math.log((1 - self.prior_prob) / self.prior_prob))
            conv.weight.data.fill_(0.)
        for conv in self.reg_preds:
            conv.bias.data.fill_(1.0)
            conv.weight.data.fill_(0.)


LITE_TRAINING = ("training a YOLOv6Lite model is not supported: yolov6_b200 runs the Lite networks for inference only "
                 "(no backward kernels for the depthwise, squeeze-excite, Hardswish and channel-shuffle layers)")


class Model(nn.Module):
    export = False

    def __init__(self, config, channels=3, num_classes=None, fuse_ab=False, distill_ns=False):
        super().__init__()
        assert channels == 3
        self.fuse_ab = bool(fuse_ab)
        self.distill_ns = bool(distill_ns)
        self.return_featmaps = False      # True: the training forward returns the real, differentiable neck outputs (feature distillation)
        self.cfg = configs.normalize(config)
        self.num_classes = int(num_classes if num_classes is not None else 80)
        g = self.graph
        hd = self.cfg["head"]
        self.backbone, self.neck = Node(), Node()
        if g.lite:
            self.detect = LiteDetect(self.num_classes, hd["num_layers"])
        else:   # build_network passes use_dfl but not reg_max to Detect (yolo.py:130-131)
            self.detect = Detect(self.num_classes, hd["num_layers"], bool(hd["use_dfl"]), arch.DETECT_DEFAULT_REG_MAX)
        for name in (("stems", "cls_convs", "reg_convs", "cls_preds") + (("reg_preds_dist",) if self.distill_ns else ()) + ("reg_preds",) +
                     (("cls_preds_ab", "reg_preds_ab") if self.fuse_ab else ())):
            self.detect.add_module(name, Node())
        if self.fuse_ab:        # effidehead_fuseab.py:20-35
            self.detect.na = arch.AB_ANCHORS
            self.detect.anchors_init = (torch.tensor(g.anchors_init) / self.detect.stride[:, None]).reshape(hd["num_layers"], arch.AB_ANCHORS, 2)
        self._materialize(g)
        self.stride = self.detect.stride
        self.detect.initialize_biases()
        for m in self.modules():                      # initialize_weights, torch_utils.py:38-48
            if isinstance(m, nn.BatchNorm2d):
                m.eps, m.momentum = 1e-3, 0.03
        self.precision = "bf16"
        self._engine = None
        self._engine_key = None
        self._weights_epoch = 0      # bumped by writers that bypass autograd's version counters (fused optimizer kernel)

    # graph is rebuilt on demand so that the pickled module stays small and version-proof
    @property
    def graph(self):
        g = self.__dict__.get("_graph")
        if g is None:
            g = arch.build_graph(self.cfg, self.num_classes, fuse_ab=self.__dict__.get("fuse_ab", False),
                                 distill_ns=self.__dict__.get("distill_ns", False))
            self.__dict__["_graph"] = g
        return g

    def __getstate__(self):
        st = self.__dict__.copy()
        for k in ("_graph", "_engine", "_engine_key", "_train_engine"):
            st.pop(k, None)
        st["_engine"], st["_engine_key"] = None, None
        return st

    def _materialize(self, g):
        for op in g.ops:
            if op.kind in ("pool", "shuffle", "up"):
                continue
            path = op.name.split(".")
            root = getattr(self, path[0])
            if op.alpha:
                holder = _ensure(root, op.alpha.split(".")[1:-1])
                if "alpha" not in holder._parameters:
                    holder.alpha = nn.Parameter(torch.ones(1))
            if op.layout == "rep":
                node = _ensure(root, path[1:])
                if op.cin == op.cout and op.s == 1:
                    node.add_module("rbr_identity", nn.BatchNorm2d(op.cin))
                for br, k in (("rbr_dense", 3), ("rbr_1x1", 1)):
                    b = _ensure(node, [br])
                    b.add_module("conv", nn.Conv2d(op.cin, op.cout, k, op.s, k // 2, bias=False))
                    b.add_module("bn", nn.BatchNorm2d(op.cout))
            elif op.layout == "qa":     # QARepVGGBlock[V2] (common.py:322-477): rbr_dense ConvModule, bare rbr_1x1, post-sum bn
                node = _ensure(root, path[1:])
                b = _ensure(node, ["rbr_dense"])
                b.add_module("conv", nn.Conv2d(op.cin, op.cout, 3, op.s, 1, bias=False))
                b.add_module("bn", nn.BatchNorm2d(op.cout))
                node.add_module("rbr_1x1", nn.Conv2d(op.cin, op.cout, 1, op.s, 0, bias=False))
                node.add_module("bn", nn.BatchNorm2d(op.cout))
            elif op.kind == "se":
                node = _ensure(root, path[1:])
                node.add_module("conv1", nn.Conv2d(op.cin, op.cin // 4, 1))
                node.add_module("conv2", nn.Conv2d(op.cin // 4, op.cin, 1))
            elif op.layout == "cba":
                b = _ensure(root, path[1:] + ["block"])
                b.add_module("conv", nn.Conv2d(op.cin, op.cout, op.k, op.s, op.k // 2, bias=False,
                                               groups=op.cin if op.kind == "dw" else 1))
                b.add_module("bn", nn.BatchNorm2d(op.cout))
            elif op.layout == "dp":
                node = _ensure(root, path[1:-1])
                node.add_module(path[-1], nn.Conv2d(op.cin, op.cout, op.k, op.s, op.k // 2, groups=op.cin if op.kind == "dw" else 1))
                node.add_module(arch.dp_bn(op.name).rsplit(".", 1)[1], nn.BatchNorm2d(op.cout))
            elif op.layout == "cm":
                if op.w_row0 == 0:
                    node = _ensure(root, path[1:])
                    node.add_module("conv", nn.Conv2d(op.cin, op.param_rows, op.k, op.s, op.k // 2, bias=False))
                    node.add_module("bn", nn.BatchNorm2d(op.param_rows))
            elif op.layout == "plain":
                _ensure(root, path[1:-1]).add_module(path[-1], nn.Conv2d(op.cin, op.cout, 1))
            elif op.layout == "convT":
                _ensure(root, path[1:]).add_module("upsample_transpose", nn.ConvTranspose2d(op.cin, op.cout, 2, 2, bias=True))
        if g.lite:
            return
        R = arch.DETECT_DEFAULT_REG_MAX
        self.detect.proj = nn.Parameter(torch.linspace(0, R, R + 1), requires_grad=False)
        self.detect.add_module("proj_conv", nn.Conv2d(R + 1, 1, 1, bias=False))
        self.detect.proj_conv.weight.requires_grad_(False)

    def _apply(self, fn):
        self = super()._apply(fn)
        self.detect.stride = fn(self.detect.stride)           # yolo.py:43-47
        self.detect.grid = list(map(fn, self.detect.grid))
        self._engine = None
        return self

    # ------------------------------------------------------------------ execution
    def set_precision(self, precision):
        """'bf16' (speed: bf16 operands, fp32 accumulate) or 'fp32' (bf16x3 operands, fp32-equivalent)."""
        assert precision in ("bf16", "fp32")
        self.precision = precision
        return self

    def engine(self):
        dev = next(self.parameters()).device
        key = (self.precision, str(dev), sum(p._version for p in self.parameters()) +
               sum(b._version for b in self.buffers()), self.__dict__.get("_weights_epoch", 0))
        if self._engine is None or self._engine_key != key:
            self._engine = InferEngine(self.graph, self.state_dict(), dev, self.precision)
            self._engine_key = key
        return self._engine

    def mark_weights_changed(self):
        """Tell the model that its parameters were rewritten through raw device pointers (yv6_sgd_ema_step): the folded
        inference engine is rebuilt on the next eval forward."""
        self.__dict__["_weights_epoch"] = self.__dict__.get("_weights_epoch", 0) + 1

    def train_engine(self, n_buckets=None, rebuild=False):
        """The training engine of this model (train.py).  `n_buckets` > 1 splits the flat gradient buffer into that many
        contiguous buckets, completed one after the other during the backward pass (overlapped all-reduce, dist.py)."""
        if self.graph.lite:
            raise NotImplementedError(LITE_TRAINING)
        eng = self.__dict__.get("_train_engine")
        stale = eng is not None and (eng.dev != next(self.parameters()).device or not eng.flat.valid() or
                                     (n_buckets is not None and eng.n_buckets != n_buckets))
        if eng is None or stale or rebuild:
            from .train import TrainEngine
            eng = TrainEngine(self, n_buckets or 1)
            self.__dict__["_train_engine"] = eng
        return eng

    def forward(self, x):
        if self.training:
            if self.graph.lite:
                raise NotImplementedError(LITE_TRAINING)
            # train form (batch-stat BatchNorm, three-branch RepVGG) through the sm_90a training engine;
            # returns the reference's train-mode structure [(feats, cls, reg), featmaps] (yolo.py:33-41,
            # effidehead.py:72-92); `feats` carry only the level shapes ComputeLoss needs (loss.py:63-68)
            from .train import train_forward
            eng = self.train_engine()
            want = bool(self.__dict__.get("return_featmaps", False))
            if eng.external_feat_grads != want:       # differentiable neck outputs change the backward plan (train.py)
                eng.external_feat_grads = want
                eng._shape = None
            outs = train_forward(eng, x)
            feats = [torch.empty(x.shape[0], 1, h, w, device=x.device) for h, w in eng.sizes]
            if want:                                  # the real feature maps (yolo.py:37-39), differentiable: feature distillation
                nf = len(self.graph.feat)
                outs, fmaps = outs[:-nf], list(outs[-nf:])
            else:
                fmaps = feats
            if self.fuse_ab:       # effidehead_fuseab.py:140: (x, cls_ab, reg_ab, cls_af, reg_af); engine.py:161-166 slices it
                cls, reg, cls_ab, reg_ab = outs
                return [(feats, cls_ab, reg_ab, cls, reg), fmaps]
            if self.distill_ns:    # effidehead_distill_ns.py:104: (x, cls, reg_distri, reg_lrtb)
                cls, reg, reg_dist = outs
                return [(feats, cls, reg_dist, reg), fmaps]
            cls, reg = outs
            return [(feats, cls, reg), fmaps]
        export_mode = torch.onnx.is_in_onnx_export() or self.export
        eng = self.engine()
        # the engine owns (and reuses) its output buffers; callers of the drop-in API get their own tensors, as with the
        # reference's nn.Module (p1 = model(x1)[0]; p2 = model(x2)[0] must not alias).  DetectPipeline uses the engine directly.
        pred = eng.forward(x).clone()
        if export_mode:
            return pred
        N, _, H, W = x.shape
        return [pred, [f.clone() for f in eng.feature_maps(N, H, W, x.dtype if x.dtype == torch.uint8 else torch.float32)]]


def build_model(cfg, num_classes, device, fuse_ab=False, distill_ns=False):
    """yolov6/models/yolo.py:136-138."""
    return Model(cfg, channels=3, num_classes=num_classes, fuse_ab=fuse_ab, distill_ns=distill_ns).to(device)
