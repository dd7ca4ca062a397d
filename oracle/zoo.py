"""oracle/zoo.py -- CPU restatement of the rest of the reference's released detectors (TEST INFRASTRUCTURE ONLY).

Extends oracle/model.py, in its style and with its layer functions (float64-capable functional PyTorch, `train_mode()`,
`bf16_storage()`), to YOLOv6-L, -N6, -S6, -M6 and the MBLA models of configs/mbla: EfficientRep6 (efficientrep.py:121-247),
RepBiFPANNeck6 (reppan.py:394-543), MBLABlock (common.py:653-692) and BottleRep3 (common.py:611-631).  oracle/model.py itself
stays as it is; `forward` here covers its four models too, so `CONFIGS` holds all twelve.

Pinned by tests/golden/make_golden_zoo.py (tests/test_model_zoo.py).
"""
import torch

from . import model as om

_P6 = dict(bb_repeats=[1, 6, 12, 18, 6, 6], bb_channels=[64, 128, 256, 512, 768, 1024],
           neck_repeats=[12, 12, 12, 12, 12, 12], neck_channels=[512, 256, 128, 256, 512, 1024],
           fuse_P2=True, num_layers=4, strides=[8, 16, 32, 64], atss_warmup_epoch=4)
_P5 = dict(bb_repeats=[1, 6, 12, 18, 6], bb_channels=[64, 128, 256, 512, 1024],
           neck_repeats=[12, 12, 12, 12], neck_channels=[256, 128, 128, 256, 256, 512],
           fuse_P2=True, num_layers=3, strides=[8, 16, 32], atss_warmup_epoch=0)


def _mbla(depth, width):
    """configs/mbla/yolov6{s,m,l,x}_mbla.py."""
    return dict(_P5, depth=depth, width=width, backbone="CSPBepBackbone", neck="CSPRepBiFPANNeck",
                bb_repeats=[1, 4, 8, 8, 4], neck_repeats=[8, 8, 8, 8], cspsppf=False, csp_e=0.5,
                use_dfl=True, reg_max=16, iou_type="giou", mode="conv_silu", stage_block_type="MBLABlock")


CONFIGS = dict(om.CONFIGS)
CONFIGS.update({
    "yolov6l": dict(_P5, depth=1.0, width=1.0, backbone="CSPBepBackbone", neck="CSPRepBiFPANNeck", cspsppf=False, csp_e=0.5,
                    use_dfl=True, reg_max=16, iou_type="giou", mode="conv_silu"),
    "yolov6n6": dict(_P6, depth=0.33, width=0.25, backbone="EfficientRep6", neck="RepBiFPANNeck6", cspsppf=True, csp_e=None,
                     use_dfl=False, reg_max=0, iou_type="siou", mode="repvgg"),
    "yolov6s6": dict(_P6, depth=0.33, width=0.50, backbone="EfficientRep6", neck="RepBiFPANNeck6", cspsppf=True, csp_e=None,
                     use_dfl=False, reg_max=0, iou_type="giou", mode="repvgg"),
    "yolov6m6": dict(_P6, depth=0.60, width=0.75, backbone="CSPBepBackbone_P6", neck="CSPRepBiFPANNeck_P6", cspsppf=False,
                     csp_e=2.0 / 3, use_dfl=True, reg_max=16, iou_type="giou", mode="repvgg"),
    "yolov6s_mbla": _mbla(0.5, 0.5),
    "yolov6m_mbla": _mbla(0.5, 0.75),
    "yolov6l_mbla": _mbla(0.5, 1.0),
    "yolov6x_mbla": _mbla(1.0, 1.0),
})


def bottle_rep3(sd, p, x, mode):
    """BottleRep3.forward, common.py:627-631: conv3(conv2(conv1(x))) + alpha * x (in == out in MBLABlock)."""
    y = om.basic_block(sd, p + ".conv1", x, 1, mode)
    y = om.basic_block(sd, p + ".conv3", om.basic_block(sd, p + ".conv2", y, 1, mode), 1, mode)
    return y + sd[p + ".alpha"].to(x.dtype) * x


def mbla_block(sd, p, x, n, e, mode):
    """MBLABlock.forward, common.py:653-692: y = split(cv1 x); branch i chains its BottleRep3 blocks, each reading the
    previous one's output; cv2(cat(y0, y1, b1_1.., y2, b2_1..)).  cv1 / cv2 are bare ConvModules."""
    n = max(n // 2, 1)
    if n == 1:
        n_list = [0, 1]
    else:
        steps = 1
        while steps * 2 < n:
            steps *= 2
        n_list = [0, steps, n]
    act = "silu" if mode == "conv_silu" else "relu"
    c = int(sd[p + ".cv2.conv.weight"].shape[0] * e)
    assert sd[p + ".cv1.conv.weight"].shape[0] == len(n_list) * c
    y = list(om.conv_module(sd, p + ".cv1", x, 1, act).split(c, 1))
    out = [y[0]]
    for i, k in enumerate(n_list[1:]):
        out.append(y[i + 1])
        for j in range(k):
            out.append(bottle_rep3(sd, f"{p}.m.{i}.{j}", out[-1], mode))
    return om.conv_module(sd, p + ".cv2", torch.cat(out, 1), 1, act)


def stage(sd, cfg, p, x, n, e):
    """The stage block: RepBlock on EfficientRep* / RepBiFPANNeck*, else the backbone's stage_block_type (yolo.py:75-96)."""
    if not cfg["backbone"].startswith("CSP"):
        return om.rep_block(sd, p, x, n, cfg["mode"])
    if cfg.get("stage_block_type", "BepC3") == "MBLABlock":
        return mbla_block(sd, p, x, n, e, cfg["mode"])
    return om.bepc3(sd, p, x, n, cfg["mode"])


def backbone(sd, cfg, x):
    """EfficientRep / EfficientRep6 / CSPBepBackbone / CSPBepBackbone_P6 (efficientrep.py:7-516)."""
    reps, _ = om.scaled_lists(cfg)
    mode = cfg["mode"]
    # EfficientRep6 always uses SimSPPF / SimCSPSPPF (efficientrep.py:209); the others the SiLU variants with ConvBNSiLU
    act = "relu" if cfg["backbone"] == "EfficientRep6" or mode != "conv_silu" else "silu"
    nstage = 6 if cfg["backbone"] in ("EfficientRep6", "CSPBepBackbone_P6") else 5
    outs = []
    x = om.basic_block(sd, "backbone.stem", x, 2, mode)
    for s in range(2, nstage + 1):
        p = f"backbone.ERBlock_{s}"
        x = om.basic_block(sd, p + ".0", x, 2, mode)
        x = stage(sd, cfg, p + ".1", x, reps[s - 1], cfg["csp_e"])
        if s == nstage:
            x = om.cspsppf(sd, p + ".2", x, act) if cfg["cspsppf"] else om.sppf(sd, p + ".2", x, act)
        if s > 2 or cfg["fuse_P2"]:
            outs.append(x)
    return outs


def neck(sd, cfg, feats):
    """RepBiFPANNeck / RepBiFPANNeck6 / CSPRepBiFPANNeck / CSPRepBiFPANNeck_P6 (reppan.py:132-237, 394-543, 666-785, 955-1116)."""
    reps, _ = om.scaled_lists(cfg)
    nb = len(cfg["bb_repeats"])
    e = cfg["csp_e"]
    cbr = om.conv_bn_act

    if cfg["num_layers"] == 3:
        x3, x2, x1, x0 = feats
        fpn0 = cbr(sd, "neck.reduce_layer0", x0, 1, "relu")
        f0 = stage(sd, cfg, "neck.Rep_p4", om.bifusion(sd, "neck.Bifusion0", [fpn0, x1, x2]), reps[nb + 0], e)
        fpn1 = cbr(sd, "neck.reduce_layer1", f0, 1, "relu")
        pan2 = stage(sd, cfg, "neck.Rep_p3", om.bifusion(sd, "neck.Bifusion1", [fpn1, x2, x3]), reps[nb + 1], e)
        pan1 = stage(sd, cfg, "neck.Rep_n3", torch.cat([cbr(sd, "neck.downsample2", pan2, 2, "relu"), fpn1], 1), reps[nb + 2], e)
        pan0 = stage(sd, cfg, "neck.Rep_n4", torch.cat([cbr(sd, "neck.downsample1", pan1, 2, "relu"), fpn0], 1), reps[nb + 3], e)
        return [pan2, pan1, pan0]
    x4, x3, x2, x1, x0 = feats
    fpn0 = cbr(sd, "neck.reduce_layer0", x0, 1, "relu")
    f0 = stage(sd, cfg, "neck.Rep_p5", om.bifusion(sd, "neck.Bifusion0", [fpn0, x1, x2]), reps[nb + 0], e)
    fpn1 = cbr(sd, "neck.reduce_layer1", f0, 1, "relu")
    f1 = stage(sd, cfg, "neck.Rep_p4", om.bifusion(sd, "neck.Bifusion1", [fpn1, x2, x3]), reps[nb + 1], e)
    fpn2 = cbr(sd, "neck.reduce_layer2", f1, 1, "relu")
    pan3 = stage(sd, cfg, "neck.Rep_p3", om.bifusion(sd, "neck.Bifusion2", [fpn2, x3, x4]), reps[nb + 2], e)
    pan2 = stage(sd, cfg, "neck.Rep_n4", torch.cat([cbr(sd, "neck.downsample2", pan3, 2, "relu"), fpn2], 1), reps[nb + 3], e)
    pan1 = stage(sd, cfg, "neck.Rep_n5", torch.cat([cbr(sd, "neck.downsample1", pan2, 2, "relu"), fpn1], 1), reps[nb + 4], e)
    pan0 = stage(sd, cfg, "neck.Rep_n6", torch.cat([cbr(sd, "neck.downsample0", pan1, 2, "relu"), fpn0], 1), reps[nb + 5], e)
    return [pan3, pan2, pan1, pan0]


def forward(sd, cfg, x, train_outputs=False):
    """Model.forward, yolo.py:33-41 (see oracle.model.forward).  Eval: [B,A,5+nc]; train_outputs: (cls, reg, sizes)."""
    feats = neck(sd, cfg, backbone(sd, cfg, x))
    sizes = [tuple(f.shape[2:]) for f in feats]
    cls, reg = om.head_raw(sd, cfg, feats)
    if train_outputs:
        return cls, reg, sizes
    return om.decode_eval(cfg, cls, reg, sizes)
