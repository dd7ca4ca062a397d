"""Declarative layer graph of the YOLOv6 networks on the hot path.

The reference builds its models as nested nn.Modules (yolov6/models/yolo.py:55-133 -> efficientrep.py,
reppan.py, effidehead.py, layers/common.py).  Here a network is a flat list of ops over NHWC
activation buffers, emitted once per (config, num_classes):

  * every op names the reference parameter prefix it owns (`backbone.ERBlock_3.1.block.0`, ...), so
    the parameter container (model.py) exposes exactly the reference's `state_dict` keys and released
    checkpoints load unchanged;
  * `torch.cat` never happens: a concat is one buffer and its producers write channel slices
    (reppan.py:228,232, common.py:650,718 -> `dst=T(buf, c_off, c)`);
  * the engine (engine.py) walks the list and issues one kernel per op through the C ABI.

Op kinds: stem | conv (rep / qa / cba / cm / plain / dp parameter layouts) | convT | pool, and for the YOLOv6Lite networks
(build_lite_graph) dw (depthwise conv) | se (squeeze-excite, in place) | shuffle (channel_shuffle of two slices) | up (nearest
2x upsample).
"""
import math
from dataclasses import dataclass, field
from typing import List, Optional


@dataclass(frozen=True)
class T:
    """Channel slice [c_off, c_off + c) of activation buffer `buf`."""
    buf: int
    c_off: int
    c: int


@dataclass
class Buf:
    level: int      # spatial size = input / 2**level
    c_total: int
    name: str = ""


@dataclass
class Op:
    kind: str                 # 'stem' | 'conv' | 'convT' | 'pool' | 'pred' | 'dw' | 'se' | 'shuffle' | 'up'
    name: str                 # reference parameter prefix
    layout: str = ""          # 'rep' | 'qa' (QARepVGGBlock[V2]) | 'cba' | 'cm' (bare ConvModule) | 'plain' | 'convT' | 'dp' (a DPBlock conv: bias, bn_1 / bn_2)
    src: Optional[T] = None
    dst: Optional[T] = None
    cin: int = 0
    cout: int = 0
    k: int = 1
    s: int = 1
    act: Optional[str] = None
    res: Optional[T] = None
    alpha: Optional[str] = None   # parameter name of BottleRep.alpha (common.py:600-603)
    head: Optional[tuple] = None  # ('cls' | 'reg', level index) for the prediction convs
    # an op that computes output rows [w_row0, w_row0 + cout) of a parameter with w_rows output rows (0: the whole parameter);
    # the op with w_row0 == 0 owns the parameter.  BatchNorm is per output channel, so the rows fold and train on their own.
    w_row0: int = 0
    w_rows: int = 0
    src2: Optional[T] = None  # shuffle: the second source (y[2j] = src[j], y[2j+1] = src2[j])
    avg: bool = False         # 'qa': the block has QARepVGGBlockV2's 3x3 average-pool branch (common.py:406-425)

    @property
    def identity(self):
        """A RepVGG-style block ('rep' / 'qa') with an identity branch: Cin == Cout at stride 1, not the stem."""
        return self.layout in ("rep", "qa") and self.kind != "stem" and self.cin == self.cout and self.s == 1

    @property
    def param_rows(self):
        return self.w_rows or self.cout


@dataclass
class Graph:
    name: str
    num_classes: int
    strides: List[int]
    use_dfl: bool
    reg_max: int
    mode: str
    bufs: List[Buf] = field(default_factory=list)
    ops: List[Op] = field(default_factory=list)
    feat: List[T] = field(default_factory=list)   # neck outputs (reference `featmaps`, yolo.py:37-39)
    fuse_ab: bool = False
    lite: bool = False                            # a YOLOv6Lite network (build_lite_graph): no DFL projection in the head
    anchors_init: Optional[list] = None           # fuse_ab: per level [w0, h0, w1, h1, w2, h2] in pixels
    distill_ns: bool = False
    dist_reg_ch: int = 0                          # distill_ns: channels of the DFL (reg_preds_dist) branch

    # -- builders ---------------------------------------------------------------------------
    def buf(self, level, c_total, name=""):
        self.bufs.append(Buf(level, c_total, name))
        return len(self.bufs) - 1

    def new(self, level, c, name=""):
        return T(self.buf(level, c, name), 0, c)

    def level(self, t):
        return self.bufs[t.buf].level

    def conv(self, name, layout, src, cout, k=1, s=1, act="relu", dst=None, res=None, alpha=None, rows=(0, 0)):
        lvl = self.level(src) + (1 if s == 2 else 0)
        if dst is None:
            dst = self.new(lvl, cout, name)
        assert dst.c == cout and self.level(dst) == lvl, (name, dst, cout, lvl)
        self.ops.append(Op("conv", name, layout, src, dst, src.c, cout, k, s, act, res, alpha, w_row0=rows[0], w_rows=rows[1]))
        return dst

    def block(self, name, src, cout, s=1, dst=None, res=None, alpha=None):
        """get_block(training_mode) of common.py:721-737: RepVGGBlock (relu), QARepVGGBlock[V2] (relu) or ConvBNSiLU /
        ConvBNReLU."""
        if self.mode in QA_MODES:
            dst = self.conv(name, "qa", src, cout, 3, s, "relu", dst, res, alpha)
            self.ops[-1].avg = self.mode == "qarepvggv2" and src.c == cout and s == 1
            return dst
        if self.mode == "repvgg":
            return self.conv(name, "rep", src, cout, 3, s, "relu", dst, res, alpha)
        return self.conv(name, "cba", src, cout, 3, s, "silu" if self.mode == "conv_silu" else "relu", dst, res, alpha)

    @property
    def act(self):
        return "silu" if self.mode == "conv_silu" else "relu"


QA_MODES = ("qarepvgg", "qarepvggv2")
# get_block's modes (common.py:721-737) that build a network here; 'hyper_search' (LinearAddBlock) and 'repopt' (RealVGGBlock)
# are not among them
TRAINING_MODES = ("repvgg", "conv_relu", "conv_silu") + QA_MODES
DETECT_DEFAULT_REG_MAX = 16  # effidehead.py:16
AB_ANCHORS = 3                # build_network passes num_anchors = 3 to the fuse_ab head (yolo.py:125)


def make_divisible(x, divisor):
    return math.ceil(x / divisor) * divisor


def _rep_block(g, name, src, cout, n, dst=None):
    """RepBlock with plain basic blocks (common.py:569-588)."""
    for i in range(n):
        last = i == n - 1
        src = g.block(f"{name}.conv1" if i == 0 else f"{name}.block.{i - 1}", src, cout, dst=dst if last else None)
    return src


def _bottle_stage(g, name, src, c, n, dst=None):
    """RepBlock(block=BottleRep, weight=True): n // 2 BottleReps, each conv2(conv1(x)) + alpha * x
    (common.py:579-582, 591-608).  The shortcut is fused into conv2's epilogue."""
    nb = max(n // 2, 1)
    for i in range(nb):
        p = f"{name}.conv1" if i == 0 else f"{name}.block.{i - 1}"
        mid = g.block(p + ".conv1", src, c)
        shortcut = src.c == c
        src = g.block(p + ".conv2", mid, c, dst=dst if i == nb - 1 else None,
                      res=src if shortcut else None, alpha=p + ".alpha")
    return src


def _bepc3(g, name, src, cout, n, e, dst=None):
    """BepC3 (common.py:634-650): cv3(cat(m(cv1 x), cv2 x)); the cat is one buffer with two slices."""
    c_ = int(cout * e)
    lvl = g.level(src)
    cat = g.buf(lvl, 2 * c_, name + ".cat")
    a = g.conv(name + ".cv1", "cba", src, c_, 1, 1, g.act)
    _bottle_stage(g, name + ".m", a, c_, n, dst=T(cat, 0, c_))
    g.conv(name + ".cv2", "cba", src, c_, 1, 1, g.act, dst=T(cat, c_, c_))
    return g.conv(name + ".cv3", "cba", T(cat, 0, 2 * c_), cout, 1, 1, g.act, dst=dst)


def mbla_branches(n):
    """MBLABlock's BottleRep3 chain lengths (common.py:657-668): n // 2 (at least 1) blocks in the longest branch, plus one
    branch of the largest power of two below half of that when there are more than one."""
    n = max(n // 2, 1)
    if n == 1:
        return [0, 1]
    e = 1
    while 2 * e < n:
        e *= 2
    return [0, e, n]


def _mbla(g, name, src, cout, n, e, dst=None):
    """MBLABlock (common.py:653-692): cv2(cat(y0, y1, m0(y1)..., y2, m1(y2)...)) with y = split(cv1(x)), where branch i is
    a chain of BottleRep3 blocks (common.py:611-631), each conv3(conv2(conv1(x))) + alpha * x; every block reads the
    previous block's output.  cv1 / cv2 are bare ConvModules.  The concat is one buffer; the y_i are not adjacent in it
    once there is a third branch, so cv1 runs as one launch per contiguous run of concat slots, each over its rows of
    the parameter."""
    n_list = mbla_branches(n)
    c = int(cout * e)
    ctot = (sum(n_list) + len(n_list)) * c
    cat = g.buf(g.level(src), ctot, name + ".cat")
    slot = [i + sum(n_list[:i]) for i in range(len(n_list))]     # concat slot (in units of c) of y_i
    b0 = 0
    for b in range(1, len(n_list) + 1):
        if b == len(n_list) or slot[b] != slot[b - 1] + 1:
            g.conv(name + ".cv1", "cm", src, (b - b0) * c, 1, 1, g.act, dst=T(cat, slot[b0] * c, (b - b0) * c),
                   rows=(b0 * c, len(n_list) * c))
            b0 = b
    for i, k in enumerate(n_list[1:]):
        x = T(cat, slot[i + 1] * c, c)
        for j in range(k):
            p = f"{name}.m.{i}.{j}"
            t = g.block(p + ".conv2", g.block(p + ".conv1", x, c), c)
            x = g.block(p + ".conv3", t, c, dst=T(cat, x.c_off + c, c), res=x, alpha=p + ".alpha")
    return g.conv(name + ".cv2", "cm", T(cat, 0, ctot), cout, 1, 1, g.act, dst=dst)


STAGE_BLOCKS = ("BepC3", "MBLABlock")


def _stage(g, kind, name, src, cout, n, e, dst=None):
    """The stage block of the backbones and necks: RepBlock (EfficientRep*, RepBiFPANNeck*) or, on the CSP variants, the
    `stage_block_type` of the config (yolo.py:75-96, efficientrep.py:271-274, reppan.py:684-687)."""
    if kind == "RepBlock":
        return _rep_block(g, name, src, cout, n, dst)
    if kind == "BepC3":
        return _bepc3(g, name, src, cout, n, e, dst)
    return _mbla(g, name, src, cout, n, e, dst)


def _sppf(g, name, src, cout, act):
    """SimSPPF / SPPF (common.py:97-133)."""
    p = name + ".sppf"
    c_ = src.c // 2
    lvl = g.level(src)
    cat = g.buf(lvl, 4 * c_, p + ".cat")
    g.conv(p + ".cv1", "cba", src, c_, 1, 1, act, dst=T(cat, 0, c_))
    g.ops.append(Op("pool", p + ".m", src=T(cat, 0, c_), dst=T(cat, 0, 4 * c_), cin=c_, cout=c_))
    return g.conv(p + ".cv2", "cba", T(cat, 0, 4 * c_), cout, 1, 1, act)


def _cspsppf(g, name, src, cout, act):
    """SimCSPSPPF / CSPSPPF (common.py:135-178), e = 0.5."""
    p = name + ".cspsppf"
    c_ = int(cout * 0.5)
    lvl = g.level(src)
    cat4 = g.buf(lvl, 4 * c_, p + ".cat4")
    cat2 = g.buf(lvl, 2 * c_, p + ".cat2")
    a = g.conv(p + ".cv1", "cba", src, c_, 1, 1, act)
    a = g.conv(p + ".cv3", "cba", a, c_, 3, 1, act)
    g.conv(p + ".cv4", "cba", a, c_, 1, 1, act, dst=T(cat4, 0, c_))
    g.conv(p + ".cv2", "cba", src, c_, 1, 1, act, dst=T(cat2, 0, c_))
    g.ops.append(Op("pool", p + ".m", src=T(cat4, 0, c_), dst=T(cat4, 0, 4 * c_), cin=c_, cout=c_))
    b = g.conv(p + ".cv5", "cba", T(cat4, 0, 4 * c_), c_, 1, 1, act)
    g.conv(p + ".cv6", "cba", b, c_, 3, 1, act, dst=T(cat2, c_, c_))
    return g.conv(p + ".cv7", "cba", T(cat2, 0, 2 * c_), cout, 1, 1, act)


def _bifusion(g, name, x0, x1, x2, cout):
    """BiFusion (common.py:695-718), always ReLU: cv3(cat(up2x(x0), cv1(x1), down(cv2(x2))))."""
    lvl = g.level(x1)
    cat = g.buf(lvl, 3 * cout, name + ".cat")
    g.ops.append(Op("convT", name + ".upsample", "convT", x0, T(cat, 0, cout), x0.c, cout, 2, 2, None))
    g.conv(name + ".cv1", "cba", x1, cout, 1, 1, "relu", dst=T(cat, cout, cout))
    t = g.conv(name + ".cv2", "cba", x2, cout, 1, 1, "relu")
    g.conv(name + ".downsample", "cba", t, cout, 3, 2, "relu", dst=T(cat, 2 * cout, cout))
    return g.conv(name + ".cv3", "cba", T(cat, 0, 3 * cout), cout, 1, 1, "relu")


def build_graph(cfg, num_classes=80, name="yolov6", fuse_ab=False, distill_ns=False):
    """The network of a normalised config (configs.normalize): build_lite_graph for the Lite_EffiBackbone ones, else below.

    cfg: dict with the fields of the reference's `config.model` (see configs.py / config_from_reference).
    fuse_ab: add the anchor-aided training branch of effidehead_fuseab.py (two more 1x1 pred convs per level).
    distill_ns: the N / S student head of effidehead_distill_ns.py -- `reg_preds` emits the 4 (l, r, t, b) distances used at
    inference, `reg_preds_dist` the 4 * (reg_max + 1) DFL logits used by the distillation loss (training only)."""
    if is_lite(cfg):
        if fuse_ab or distill_ns:
            raise ValueError("YOLOv6Lite has no fuse_ab or distill_ns head (yolo_lite.py builds only the Lite Detect)")
        return build_lite_graph(cfg, num_classes, name)
    if cfg["training_mode"] not in TRAINING_MODES:
        raise ValueError(f"training_mode {cfg['training_mode']!r} is not one of {TRAINING_MODES} (get_block, common.py:721-737)")
    depth, width = cfg["depth_multiple"], cfg["width_multiple"]
    bb, nk, hd = cfg["backbone"], cfg["neck"], cfg["head"]
    reps = [(max(round(i * depth), 1) if i > 1 else i) for i in bb["num_repeats"] + nk["num_repeats"]]   # yolo.py:66
    ch = [make_divisible(i * width, 8) for i in bb["out_channels"] + nk["out_channels"]]                # yolo.py:67
    nl = hd["num_layers"]
    g = Graph(name, num_classes, list(hd["strides"]), bool(hd["use_dfl"]) and not distill_ns, 0 if distill_ns else int(hd["reg_max"]),
              cfg["training_mode"])
    if distill_ns and (fuse_ab or nl != 3):
        raise ValueError("distill_ns is the 3-level N / S student head (yolo.py:113-120); it excludes fuse_ab")
    csp = "CSP" in bb["type"]
    p6 = bb["type"] in ("EfficientRep6", "CSPBepBackbone_P6")
    nstage = 6 if p6 else 5
    if bb["type"] not in ("EfficientRep", "EfficientRep6", "CSPBepBackbone", "CSPBepBackbone_P6"):
        raise NotImplementedError(f"backbone {bb['type']} is outside the hot-path scope (SURVEY.md section 2)")
    if nk["type"] not in ("RepBiFPANNeck", "RepBiFPANNeck6", "CSPRepBiFPANNeck", "CSPRepBiFPANNeck_P6"):
        raise NotImplementedError(f"neck {nk['type']} is outside the hot-path scope (SURVEY.md section 2)")
    # the CSP variants take the backbone's stage_block_type for the backbone AND the neck (yolo.py:75-96)
    stage_kind = bb.get("stage_block_type", "BepC3") if csp else "RepBlock"
    if stage_kind not in STAGE_BLOCKS + ("RepBlock",):
        raise ValueError(f"stage_block_type {stage_kind!r} is not one of {STAGE_BLOCKS} (efficientrep.py:271-276)")

    # ---- backbone (efficientrep.py:7-118, 250-374, 377-516) ----
    layout = "rep" if g.mode == "repvgg" else "qa" if g.mode in QA_MODES else "cba"
    stem = T(g.buf(1, ch[0], "stem"), 0, ch[0])
    g.ops.append(Op("stem", "backbone.stem", layout, None, stem, 3, ch[0], 3, 2, "relu" if layout != "cba" else g.act))
    x = stem
    outs = []
    for s in range(2, nstage + 1):
        p = f"backbone.ERBlock_{s}"
        x = g.block(p + ".0", x, ch[s - 1], s=2)
        x = _stage(g, stage_kind, p + ".1", x, ch[s - 1], reps[s - 1], bb.get("csp_e"))
        if s == nstage:
            # EfficientRep6 always takes the ReLU variants (efficientrep.py:209), the others SiLU ones with ConvBNSiLU blocks
            act = "relu" if bb["type"] == "EfficientRep6" else g.act
            x = (_cspsppf if bb.get("cspsppf") else _sppf)(g, p + ".2", x, ch[s - 1], act)
        if s > 2 or bb.get("fuse_P2"):
            outs.append(x)
    if not bb.get("fuse_P2"):
        raise NotImplementedError("the Rep-BiFPAN necks on the hot path need fuse_P2=True backbones")

    # ---- neck (reppan.py:132-237, 666-785, 955-1116) ----
    nb = len(bb["num_repeats"])

    def stage(name, src, cout, n, dst=None):
        return _stage(g, stage_kind, name, src, cout, n, nk.get("csp_e"), dst)

    if not p6:
        x3, x2, x1, x0 = outs
        lvl1, lvl0 = g.level(x1), g.level(x0)
        cat_n4 = g.buf(lvl0, ch[9] + ch[5], "neck.cat_n4")          # [down_feat0, fpn_out0]
        cat_n3 = g.buf(lvl1, ch[7] + ch[6], "neck.cat_n3")          # [down_feat1, fpn_out1]
        fpn0 = g.conv("neck.reduce_layer0", "cba", x0, ch[5], 1, 1, "relu", dst=T(cat_n4, ch[9], ch[5]))
        f0 = stage("neck.Rep_p4", _bifusion(g, "neck.Bifusion0", fpn0, x1, x2, ch[5]), ch[5], reps[nb + 0])
        fpn1 = g.conv("neck.reduce_layer1", "cba", f0, ch[6], 1, 1, "relu", dst=T(cat_n3, ch[7], ch[6]))
        pan2 = stage("neck.Rep_p3", _bifusion(g, "neck.Bifusion1", fpn1, x2, x3, ch[6]), ch[6], reps[nb + 1])
        g.conv("neck.downsample2", "cba", pan2, ch[7], 3, 2, "relu", dst=T(cat_n3, 0, ch[7]))
        pan1 = stage("neck.Rep_n3", T(cat_n3, 0, ch[7] + ch[6]), ch[8], reps[nb + 2])
        g.conv("neck.downsample1", "cba", pan1, ch[9], 3, 2, "relu", dst=T(cat_n4, 0, ch[9]))
        pan0 = stage("neck.Rep_n4", T(cat_n4, 0, ch[9] + ch[5]), ch[10], reps[nb + 3])
        feats = [pan2, pan1, pan0]
        head_ch = [ch[6], ch[8], ch[10]]                              # effidehead.py:144 chx = [6, 8, 10]
    else:
        x4, x3, x2, x1, x0 = outs
        cat_n6 = g.buf(g.level(x0), ch[10] + ch[6], "neck.cat_n6")
        cat_n5 = g.buf(g.level(x1), ch[9] + ch[7], "neck.cat_n5")
        cat_n4 = g.buf(g.level(x2), ch[8] + ch[8], "neck.cat_n4")
        fpn0 = g.conv("neck.reduce_layer0", "cba", x0, ch[6], 1, 1, "relu", dst=T(cat_n6, ch[10], ch[6]))
        f0 = stage("neck.Rep_p5", _bifusion(g, "neck.Bifusion0", fpn0, x1, x2, ch[6]), ch[6], reps[nb + 0])
        fpn1 = g.conv("neck.reduce_layer1", "cba", f0, ch[7], 1, 1, "relu", dst=T(cat_n5, ch[9], ch[7]))
        f1 = stage("neck.Rep_p4", _bifusion(g, "neck.Bifusion1", fpn1, x2, x3, ch[7]), ch[7], reps[nb + 1])
        fpn2 = g.conv("neck.reduce_layer2", "cba", f1, ch[8], 1, 1, "relu", dst=T(cat_n4, ch[8], ch[8]))
        pan3 = stage("neck.Rep_p3", _bifusion(g, "neck.Bifusion2", fpn2, x3, x4, ch[8]), ch[8], reps[nb + 2])
        g.conv("neck.downsample2", "cba", pan3, ch[8], 3, 2, "relu", dst=T(cat_n4, 0, ch[8]))
        pan2 = stage("neck.Rep_n4", T(cat_n4, 0, 2 * ch[8]), ch[9], reps[nb + 3])
        g.conv("neck.downsample1", "cba", pan2, ch[9], 3, 2, "relu", dst=T(cat_n5, 0, ch[9]))
        pan1 = stage("neck.Rep_n5", T(cat_n5, 0, ch[9] + ch[7]), ch[10], reps[nb + 4])
        g.conv("neck.downsample0", "cba", pan1, ch[10], 3, 2, "relu", dst=T(cat_n6, 0, ch[10]))
        pan0 = stage("neck.Rep_n6", T(cat_n6, 0, ch[10] + ch[6]), ch[11], reps[nb + 5])
        feats = [pan3, pan2, pan1, pan0]
        head_ch = [ch[8], ch[9], ch[10], ch[11]]                      # effidehead.py:144 chx = [8, 9, 10, 11]
    g.feat = feats
    assert len(feats) == nl

    # ---- head (effidehead.py:10-139, 142-293): stem 1x1 -> {cls 3x3 -> pred}, {reg 3x3 -> pred} ----
    reg_ch = 4 * (g.reg_max + 1)
    for i, (f, c) in enumerate(zip(feats, head_ch)):
        assert f.c == c
        st = g.conv(f"detect.stems.{i}", "cba", f, c, 1, 1, "silu")
        cf = g.conv(f"detect.cls_convs.{i}", "cba", st, c, 3, 1, "silu")
        rf = g.conv(f"detect.reg_convs.{i}", "cba", st, c, 3, 1, "silu")
        g.ops.append(Op("pred", f"detect.cls_preds.{i}", "plain", cf, None, c, num_classes, 1, 1, "sigmoid", head=("cls", i)))
        if distill_ns:      # effidehead_distill_ns.py:36-46,87-96: module order cls_preds, reg_preds_dist, reg_preds
            g.ops.append(Op("pred", f"detect.reg_preds_dist.{i}", "plain", rf, None, c, 4 * (int(hd["reg_max"]) + 1), 1, 1, None, head=("reg_dist", i)))
        g.ops.append(Op("pred", f"detect.reg_preds.{i}", "plain", rf, None, c, reg_ch, 1, 1, None, head=("reg", i)))
        if fuse_ab:     # effidehead_fuseab.py:44-55,112-118: num_anchors = 3 class / box predictions per pixel, training only
            g.ops.append(Op("pred", f"detect.cls_preds_ab.{i}", "plain", cf, None, c, num_classes * AB_ANCHORS, 1, 1, "sigmoid", head=("cls_ab", i)))
            g.ops.append(Op("pred", f"detect.reg_preds_ab.{i}", "plain", rf, None, c, 4 * AB_ANCHORS, 1, 1, None, head=("reg_ab", i)))
    g.fuse_ab = bool(fuse_ab)
    g.distill_ns = bool(distill_ns)
    g.dist_reg_ch = 4 * (int(hd["reg_max"]) + 1) if distill_ns else 0
    if fuse_ab:
        ai = hd.get("anchors_init")
        if ai is None or len(ai) != nl or any(len(a) != 2 * AB_ANCHORS for a in ai):
            raise ValueError("fuse_ab needs cfg.model.head.anchors_init with 3 (w, h) pairs per level (configs/yolov6*.py)")
        g.anchors_init = [[float(v) for v in a] for a in ai]
    return g


# ------------------------------------------------------------------------------------------------------------- YOLOv6Lite
def is_lite(cfg):
    return cfg["backbone"]["type"] == "Lite_EffiBackbone"


def lite_divisible(v, divisor=16):
    """make_divisible of yolo_lite.py (not arch.make_divisible): round to the nearest multiple, at least `divisor`, and not
    below 90 % of v."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def lite_channels(cfg):
    """(backbone out channels, backbone mid channels, neck in channels) of yolo_lite.build_network; the backbone forces
    out[0] = 24 after the mid channels are computed (efficientrep.py:526)."""
    width, bb = cfg["width_multiple"], cfg["backbone"]
    out = [lite_divisible(i * width) for i in bb["out_channels"]]
    mid = [lite_divisible(int(i * bb["scale_size"]), 8) for i in out]
    out[0] = 24
    return out, mid, [lite_divisible(i * width) for i in cfg["neck"]["in_channels"]]


def _ceil16(c):
    return (c + 15) // 16 * 16


class LiteGraph(Graph):
    """Every activation buffer has a channel pitch that is a multiple of 16 and zero pad channels, so a 1x1 conv can read the
    16-aligned channel window around any slice (engine.conv_window) with zero weight columns outside it."""

    def buf(self, level, c_total, name=""):
        return super().buf(level, _ceil16(c_total), name)

    def new(self, level, c, name=""):
        return T(self.buf(level, c, name), 0, c)

    def hs(self, name, src, cout, dst=None, res=None):
        """ConvBNHS 1x1 (common.py:87-94)."""
        return self.conv(name, "cba", src, cout, 1, 1, "hardswish", dst=dst, res=res)

    def dw(self, name, layout, src, k, s, act, dst=None):
        """Depthwise conv: ConvBN / ConvBNHS with groups = C ('cba') or DPBlock.conv_dw_1 ('dp')."""
        lvl = self.level(src) + (1 if s == 2 else 0)
        if dst is None:
            dst = self.new(lvl, src.c, name)
        assert dst.c == src.c and self.level(dst) == lvl, (name, dst, src)
        self.ops.append(Op("dw", name, layout, src, dst, src.c, src.c, k, s, act))
        return dst

    def se(self, name, t):
        """SEBlock (common.py:740-768), in place on slice t; reduction 4."""
        self.ops.append(Op("se", name, "se", t, t, t.c, t.c // 4))

    def dp(self, name, src, k, s, dst=None, res=None):
        """DPBlock (common.py:900-934): hardswish(BN(dw k x k + bias)) -> hardswish(BN(1x1 + bias)) [+ res]."""
        t = self.dw(name + ".conv_dw_1", "dp", src, k, s, "hardswish")
        return self.conv(name + ".conv_pw_1", "dp", t, src.c, 1, 1, "hardswish", dst=dst, res=res)


def _lite_s2(g, p, x, mid, out):
    """Lite_EffiBlockS2 (common.py:826-897), stride 2: cat(conv_1(dw_1 x), conv_2(se(dw_2(pw_2 x)))) -> dw_3 -> pw_3."""
    cat = g.buf(g.level(x) + 1, out, p + ".cat")
    g.hs(p + ".conv_1", g.dw(p + ".conv_dw_1", "cba", x, 3, 2, None), out // 2, dst=T(cat, 0, out // 2))
    t = g.dw(p + ".conv_dw_2", "cba", g.hs(p + ".conv_pw_2", x, mid // 2), 3, 2, None)
    g.se(p + ".se", t)
    g.hs(p + ".conv_2", t, out // 2, dst=T(cat, out // 2, out // 2))
    return g.hs(p + ".conv_pw_3", g.dw(p + ".conv_dw_3", "cba", T(cat, 0, out), 3, 1, "hardswish"), out)


def _lite_s1(g, p, x, mid):
    """Lite_EffiBlockS1 (common.py:783-823): x1, x2 = split(x); channel_shuffle(cat(x1, conv_1(se(dw_1(pw_1 x2)))), 2)."""
    h = x.c // 2
    t = g.dw(p + ".conv_dw_1", "cba", g.hs(p + ".conv_pw_1", T(x.buf, x.c_off + h, h), mid), 3, 1, None)
    g.se(p + ".se", t)
    x3 = g.hs(p + ".conv_1", t, h)
    y = g.new(g.level(x), x.c, p)
    g.ops.append(Op("shuffle", p + ".shuffle", src=T(x.buf, x.c_off, h), src2=x3, dst=y, cin=h, cout=x.c))
    return y


def _csp_lite(g, p, x, cout, dst=None):
    """CSPBlock(k=5, e=0.5) of Lite_EffiNeck (common.py:937-985): conv_3(cat(DarknetBlock(conv_1 x), conv_2 x))."""
    m = int(cout * 0.5)
    cat = g.buf(g.level(x), 2 * m, p + ".cat")
    g.dp(p + ".blocks.conv_2", g.hs(p + ".blocks.conv_1", g.hs(p + ".conv_1", x, m), m), 5, 1, dst=T(cat, 0, m))
    g.hs(p + ".conv_2", x, m, dst=T(cat, m, m))
    return g.hs(p + ".conv_3", T(cat, 0, 2 * m), cout, dst=dst)


def build_lite_graph(cfg, num_classes=80, name="yolov6lite"):
    """YOLOv6Lite (yolo_lite.py:49-76): Lite_EffiBackbone (efficientrep.py:518-582), Lite_EffiNeck (reppan.py:1118-1226) and the
    Lite decoupled head (effidehead_lite.py): k5 DPBlock stems / cls / reg convs, 1x1 preds, reg used directly as ltrb distances.
    Physical channel order is the reference's order, so torch.split is a slice and every intermediate compares directly."""
    bb, nk, hd = cfg["backbone"], cfg["neck"], cfg["head"]
    if nk["type"] != "Lite_EffiNeck" or hd["num_layers"] != 4:
        raise NotImplementedError(f"Lite_EffiBackbone with neck {nk['type']} / {hd['num_layers']} levels is outside the hot-path scope")
    out, mid, neck_in = lite_channels(cfg)
    g = LiteGraph(name, num_classes, list(hd["strides"]), False, 0, "lite")
    g.lite = True
    stem = g.new(1, out[0], "backbone.conv_0")
    g.ops.append(Op("stem", "backbone.conv_0", "cba", None, stem, 3, out[0], 3, 2, "hardswish"))
    x, feats = stem, []
    for s in range(1, 5):
        p = f"backbone.lite_effiblock_{s}"
        for i in range(bb["num_repeats"][s - 1]):
            x = _lite_s2(g, f"{p}.{i}", x, mid[s], out[s]) if i == 0 else _lite_s1(g, f"{p}.{i}", x, mid[s])
        if s >= 2:
            feats.append(x)
    x2, x1, x0 = feats
    assert [x0.c, x1.c, x2.c] == neck_in, (neck_in, [x0.c, x1.c, x2.c])
    U = nk["unified_channels"]
    f_cat0 = g.buf(g.level(x1), 2 * U, "neck.f_concat_layer0")      # [upsample_feat0, reduce_layer1(x1)]
    f_cat1 = g.buf(g.level(x2), 2 * U, "neck.f_concat_layer1")      # [upsample_feat1, reduce_layer2(x2)]
    p_cat1 = g.buf(g.level(x1), 2 * U, "neck.p_concat_layer1")      # [down_feat1, f_out1]
    p_cat2 = g.buf(g.level(x0), 2 * U, "neck.p_concat_layer2")      # [down_feat0, fpn_out0]
    fpn0 = g.hs("neck.reduce_layer0", x0, U, dst=T(p_cat2, U, U))
    g.hs("neck.reduce_layer1", x1, U, dst=T(f_cat0, U, U))
    g.hs("neck.reduce_layer2", x2, U, dst=T(f_cat1, U, U))
    g.ops.append(Op("up", "neck.upsample0", src=fpn0, dst=T(f_cat0, 0, U), cin=U, cout=U))
    f_out1 = _csp_lite(g, "neck.Csp_p4", T(f_cat0, 0, 2 * U), U, dst=T(p_cat1, U, U))
    g.ops.append(Op("up", "neck.upsample1", src=f_out1, dst=T(f_cat1, 0, U), cin=U, cout=U))
    pan3 = _csp_lite(g, "neck.Csp_p3", T(f_cat1, 0, 2 * U), U)
    g.dp("neck.downsample2", pan3, 5, 2, dst=T(p_cat1, 0, U))
    pan2 = _csp_lite(g, "neck.Csp_n3", T(p_cat1, 0, 2 * U), U)
    g.dp("neck.downsample1", pan2, 5, 2, dst=T(p_cat2, 0, U))
    pan1 = _csp_lite(g, "neck.Csp_n4", T(p_cat2, 0, 2 * U), U)
    top = g.dp("neck.p6_conv_1", fpn0, 5, 2)
    pan0 = g.dp("neck.p6_conv_2", pan1, 5, 2, res=top)               # top_features + p6_conv_2(pan_out1): hardswish, then add
    g.feat = [pan3, pan2, pan1, pan0]
    for i, f in enumerate(g.feat):
        st = g.dp(f"detect.stems.{i}", f, 5, 1)
        cf = g.dp(f"detect.cls_convs.{i}", st, 5, 1)
        rf = g.dp(f"detect.reg_convs.{i}", st, 5, 1)
        g.ops.append(Op("pred", f"detect.cls_preds.{i}", "plain", cf, None, U, num_classes, 1, 1, "sigmoid", head=("cls", i)))
        g.ops.append(Op("pred", f"detect.reg_preds.{i}", "plain", rf, None, U, 4, 1, 1, None, head=("reg", i)))
    return g


def dp_bn(name):
    """The BatchNorm of a DPBlock conv: conv_dw_1 -> bn_1, conv_pw_1 -> bn_2 (common.py:908-923)."""
    parent, leaf = name.rsplit(".", 1)
    return parent + (".bn_1" if leaf == "conv_dw_1" else ".bn_2")


def param_specs(g):
    """(name, shape, kind) of every tensor in the reference state_dict that this graph owns.
    kind in {'conv', 'bn', 'bias', 'alpha', 'buffer', 'const'}; BN expands to its five tensors."""
    specs = []

    def bn(prefix, c):
        specs.append((prefix + ".weight", (c,), "bn_w"))
        specs.append((prefix + ".bias", (c,), "bn_b"))
        specs.append((prefix + ".running_mean", (c,), "bn_mean"))
        specs.append((prefix + ".running_var", (c,), "bn_var"))
        specs.append((prefix + ".num_batches_tracked", (), "bn_count"))

    seen_alpha = set()
    for op in g.ops:
        n = op.name
        if op.kind in ("pool", "shuffle", "up"):
            continue
        if op.kind == "se":
            cr = op.cin // 4
            specs += [(n + ".conv1.weight", (cr, op.cin, 1, 1), "conv"), (n + ".conv1.bias", (cr,), "bias"),
                      (n + ".conv2.weight", (op.cin, cr, 1, 1), "conv"), (n + ".conv2.bias", (op.cin,), "bias")]
            continue
        if op.alpha and op.alpha not in seen_alpha:
            seen_alpha.add(op.alpha)
            specs.append((op.alpha, (1,), "alpha"))
        if op.layout == "rep":
            if op.cin == op.cout and op.s == 1:
                bn(n + ".rbr_identity", op.cin)
            specs.append((n + ".rbr_dense.conv.weight", (op.cout, op.cin, 3, 3), "conv"))
            bn(n + ".rbr_dense.bn", op.cout)
            specs.append((n + ".rbr_1x1.conv.weight", (op.cout, op.cin, 1, 1), "conv"))
            bn(n + ".rbr_1x1.bn", op.cout)
        elif op.layout == "qa":     # QARepVGGBlock[V2]: identity / avg have no parameters, rbr_1x1 is a bare Conv2d
            specs.append((n + ".rbr_dense.conv.weight", (op.cout, op.cin, 3, 3), "conv"))
            bn(n + ".rbr_dense.bn", op.cout)
            specs.append((n + ".rbr_1x1.weight", (op.cout, op.cin, 1, 1), "conv"))
            bn(n + ".bn", op.cout)
        elif op.layout == "cba":
            specs.append((n + ".block.conv.weight", (op.cout, 1 if op.kind == "dw" else op.cin, op.k, op.k), "conv"))
            bn(n + ".block.bn", op.cout)
        elif op.layout == "dp":
            specs.append((n + ".weight", (op.cout, 1 if op.kind == "dw" else op.cin, op.k, op.k), "conv"))
            specs.append((n + ".bias", (op.cout,), "bias"))
            bn(dp_bn(n), op.cout)
        elif op.layout == "cm":
            if op.w_row0 == 0:
                specs.append((n + ".conv.weight", (op.param_rows, op.cin, op.k, op.k), "conv"))
                bn(n + ".bn", op.param_rows)
        elif op.layout == "plain":
            specs.append((n + ".weight", (op.cout, op.cin, 1, 1), "conv"))
            specs.append((n + ".bias", (op.cout,), "bias"))
        elif op.layout == "convT":
            specs.append((n + ".upsample_transpose.weight", (op.cin, op.cout, 2, 2), "conv"))
            specs.append((n + ".upsample_transpose.bias", (op.cout,), "bias"))
    if g.lite:       # the Lite Detect has no DFL projection (effidehead_lite.py:10-45)
        return specs
    # build_network does not forward reg_max to Detect (yolo.py:130-131), so its DFL projection always
    # has Detect's default reg_max = 16 entries even for the N/S models that predict 4 reg channels.
    specs.append(("detect.proj", (DETECT_DEFAULT_REG_MAX + 1,), "const"))
    specs.append(("detect.proj_conv.weight", (1, DETECT_DEFAULT_REG_MAX + 1, 1, 1), "const"))
    return specs
