"""oracle/qa.py -- CPU restatement of the quantization-aware RepVGG networks (TEST INFRASTRUCTURE ONLY).

Extends oracle/model.py, in its style and with its layer functions (float64-capable functional PyTorch, `train_mode()`,
`bf16_storage()`), to the networks get_block('qarepvgg' | 'qarepvggv2') builds (common.py:721-737): YOLOv6-N / S / M of
configs/qarepvgg with QARepVGGBlock (common.py:322-393) or QARepVGGBlockV2 (common.py:396-477) as the basic block.  Those
have one BatchNorm AFTER the branch sum, so oracle/model.py's basic_block cannot express them; it stays as it is and the
stages that call the block are restated here for the P5 networks.

Pinned by tests/golden/make_golden_qa.py (tests/test_model_qa.py).
"""
import torch
import torch.nn.functional as F

from . import model as om

CONFIGS = {f"{n}_qa": dict(om.CONFIGS[n], mode="qarepvggv2") for n in ("yolov6n", "yolov6s", "yolov6m")}


def qa_block(sd, p, x, stride, mode):
    """QARepVGGBlock[V2].forward in train form: relu(bn(BN_d(3x3 x) + 1x1 x [+ x [+ avg3x3 x]])).  The 1x1 conv has no bias
    and no BN; identity and avg exist for Cin == Cout at stride 1 (avg only in V2, AvgPool2d(3, 1, 1) counting the padding)."""
    u = om._bn(sd, p + ".rbr_dense.bn", om._q(F.conv2d(x, om._wq(sd[p + ".rbr_dense.conv.weight"].to(x.dtype), p), None, stride, 1)))
    t = u + om._q(F.conv2d(x, om._wq(sd[p + ".rbr_1x1.weight"].to(x.dtype), p), None, stride, 0))
    if stride == 1 and x.shape[1] == t.shape[1]:
        t = t + x
        if mode == "qarepvggv2":
            t = t + F.avg_pool2d(x, 3, 1, 1, count_include_pad=True)
    return om._q(torch.relu(om._bn(sd, p + ".bn", om._q(t))))


def basic_block(sd, p, x, stride, mode):
    if mode in ("qarepvgg", "qarepvggv2"):
        return qa_block(sd, p, x, stride, mode)
    return om.basic_block(sd, p, x, stride, mode)


def rep_block(sd, p, x, n, mode):
    """RepBlock with a plain basic block, common.py:569-588."""
    x = basic_block(sd, p + ".conv1", x, 1, mode)
    for i in range(n - 1):
        x = basic_block(sd, f"{p}.block.{i}", x, 1, mode)
    return x


def bottle_rep(sd, p, x, mode):
    """BottleRep.forward, common.py:591-608: conv2(conv1(x)) + alpha * x when Cin == Cout (after the block's ReLU)."""
    y = basic_block(sd, p + ".conv2", basic_block(sd, p + ".conv1", x, 1, mode), 1, mode)
    if y.shape[1] == x.shape[1]:
        y = y + sd[p + ".alpha"].to(x.dtype) * x
    return y


def bepc3(sd, p, x, n, mode):
    """BepC3.forward, common.py:634-650 (ConvBNReLU around the BottleRep stage)."""
    a = om.conv_bn_act(sd, p + ".cv1", x, 1, "relu")
    a = bottle_rep(sd, p + ".m.conv1", a, mode)
    for i in range(n // 2 - 1):
        a = bottle_rep(sd, f"{p}.m.block.{i}", a, mode)
    return om.conv_bn_act(sd, p + ".cv3", torch.cat((a, om.conv_bn_act(sd, p + ".cv2", x, 1, "relu")), 1), 1, "relu")


def _stage(cfg, sd, p, x, n):
    return bepc3(sd, p, x, n, cfg["mode"]) if cfg["backbone"].startswith("CSP") else rep_block(sd, p, x, n, cfg["mode"])


def backbone(sd, cfg, x):
    """EfficientRep / CSPBepBackbone (efficientrep.py:7-118, 250-374)."""
    reps, _ = om.scaled_lists(cfg)
    outs = []
    x = basic_block(sd, "backbone.stem", x, 2, cfg["mode"])
    for s in range(2, 6):
        p = f"backbone.ERBlock_{s}"
        x = _stage(cfg, sd, p + ".1", basic_block(sd, p + ".0", x, 2, cfg["mode"]), reps[s - 1])
        if s == 5:
            x = om.cspsppf(sd, p + ".2", x, "relu") if cfg["cspsppf"] else om.sppf(sd, p + ".2", x, "relu")
        outs.append(x)
    return outs


def neck(sd, cfg, feats):
    """RepBiFPANNeck / CSPRepBiFPANNeck (reppan.py:132-237, 666-785)."""
    reps, _ = om.scaled_lists(cfg)
    nb = len(cfg["bb_repeats"])
    cbr = om.conv_bn_act
    x3, x2, x1, x0 = feats
    fpn0 = cbr(sd, "neck.reduce_layer0", x0, 1, "relu")
    f0 = _stage(cfg, sd, "neck.Rep_p4", om.bifusion(sd, "neck.Bifusion0", [fpn0, x1, x2]), reps[nb + 0])
    fpn1 = cbr(sd, "neck.reduce_layer1", f0, 1, "relu")
    pan2 = _stage(cfg, sd, "neck.Rep_p3", om.bifusion(sd, "neck.Bifusion1", [fpn1, x2, x3]), reps[nb + 1])
    pan1 = _stage(cfg, sd, "neck.Rep_n3", torch.cat([cbr(sd, "neck.downsample2", pan2, 2, "relu"), fpn1], 1), reps[nb + 2])
    pan0 = _stage(cfg, sd, "neck.Rep_n4", torch.cat([cbr(sd, "neck.downsample1", pan1, 2, "relu"), fpn0], 1), reps[nb + 3])
    return [pan2, pan1, pan0]


def forward(sd, cfg, x, train_outputs=False):
    """Model.forward, yolo.py:33-41 (see oracle.model.forward).  Eval: [B,A,5+nc]; train_outputs: (cls, reg, sizes)."""
    feats = neck(sd, cfg, backbone(sd, cfg, x))
    sizes = [tuple(f.shape[2:]) for f in feats]
    cls, reg = om.head_raw(sd, cfg, feats)
    if train_outputs:
        return cls, reg, sizes
    return om.decode_eval(cfg, cls, reg, sizes)
