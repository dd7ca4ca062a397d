"""oracle/lite.py -- CPU restatement of the YOLOv6Lite-S / M / L detectors (TEST INFRASTRUCTURE ONLY).

Extends oracle/model.py, with its BatchNorm (`_bn`, `train_mode()`) and decode helpers, to the networks yolo_lite.py builds:
Lite_EffiBackbone (efficientrep.py:518-582), Lite_EffiNeck (reppan.py:1118-1226) and the Lite head (effidehead_lite.py),
from the layers of layers/common.py:740-985 (SEBlock, channel_shuffle, Lite_EffiBlockS1 / S2, DPBlock, CSPBlock).
`forward(..., record=d)` also fills d with named intermediates (block outputs, keyed by the reference module path), so
the CUDA path can be compared op by op.

Pinned by tests/golden/make_golden_lite.py (tests/test_model_lite.py).
"""
import torch
import torch.nn.functional as F

from . import model as om


# the widths come from the state_dict's shapes; the three models share everything else (configs/yolov6_lite/*.py)
_LITE = dict(bb_repeats=[1, 3, 7, 3], num_layers=4, strides=[8, 16, 32, 64], use_dfl=False, reg_max=0)
CONFIGS = {"yolov6lite_s": _LITE, "yolov6lite_m": _LITE, "yolov6lite_l": _LITE}


def _act(x, act):
    if act == "hardswish":
        return F.hardswish(x)
    return om._act(x, act)


def conv_module(sd, p, x, stride, act):
    """ConvModule with groups (common.py:26-49): conv (no bias, pad k // 2, groups = Cin / weight's in-channels) -> BN -> act."""
    w = sd[p + ".conv.weight"].to(x.dtype)
    groups = x.shape[1] // w.shape[1]
    return _act(om._bn(sd, p + ".bn", F.conv2d(x, w, None, stride, w.shape[-1] // 2, 1, groups)), act)


def cbn(sd, p, x, stride=1, act=None):
    """ConvBN / ConvBNHS (common.py:77-94): a ConvModule under `.block`."""
    return conv_module(sd, p + ".block", x, stride, act)


def se(sd, p, x):
    """SEBlock.forward, common.py:760-768."""
    m = x.mean(dim=(2, 3), keepdim=True)
    h = torch.relu(F.conv2d(m, sd[p + ".conv1.weight"].to(x.dtype), sd[p + ".conv1.bias"].to(x.dtype)))
    return x * F.hardsigmoid(F.conv2d(h, sd[p + ".conv2.weight"].to(x.dtype), sd[p + ".conv2.bias"].to(x.dtype)))


def channel_shuffle(x, groups):
    """common.py:771-780."""
    b, c, h, w = x.shape
    return x.view(b, groups, c // groups, h, w).transpose(1, 2).contiguous().view(b, c, h, w)


def block_s1(sd, p, x):
    """Lite_EffiBlockS1.forward, common.py:813-823."""
    x1, x2 = x.split(x.shape[1] // 2, 1)
    x3 = cbn(sd, p + ".conv_dw_1", cbn(sd, p + ".conv_pw_1", x2, act="hardswish"))
    x3 = cbn(sd, p + ".conv_1", se(sd, p + ".se", x3), act="hardswish")
    return channel_shuffle(torch.cat([x1, x3], 1), 2)


def block_s2(sd, p, x):
    """Lite_EffiBlockS2.forward, common.py:887-897."""
    x1 = cbn(sd, p + ".conv_1", cbn(sd, p + ".conv_dw_1", x, 2), act="hardswish")
    x2 = cbn(sd, p + ".conv_dw_2", cbn(sd, p + ".conv_pw_2", x, act="hardswish"), 2)
    x2 = cbn(sd, p + ".conv_2", se(sd, p + ".se", x2), act="hardswish")
    out = cbn(sd, p + ".conv_dw_3", torch.cat([x1, x2], 1), act="hardswish")
    return cbn(sd, p + ".conv_pw_3", out, act="hardswish")


def dp_block(sd, p, x, stride=1):
    """DPBlock.forward, common.py:926-929: both convs carry a bias."""
    w = sd[p + ".conv_dw_1.weight"].to(x.dtype)
    y = F.conv2d(x, w, sd[p + ".conv_dw_1.bias"].to(x.dtype), stride, w.shape[-1] // 2, 1, x.shape[1])
    y = F.hardswish(om._bn(sd, p + ".bn_1", y))
    y = F.conv2d(y, sd[p + ".conv_pw_1.weight"].to(x.dtype), sd[p + ".conv_pw_1.bias"].to(x.dtype))
    return F.hardswish(om._bn(sd, p + ".bn_2", y))


def csp_block(sd, p, x):
    """CSPBlock.forward, common.py:980-985, with DarknetBlock (common.py:958-961)."""
    x1 = dp_block(sd, p + ".blocks.conv_2", cbn(sd, p + ".blocks.conv_1", cbn(sd, p + ".conv_1", x, act="hardswish"), act="hardswish"))
    x2 = cbn(sd, p + ".conv_2", x, act="hardswish")
    return cbn(sd, p + ".conv_3", torch.cat((x1, x2), 1), act="hardswish")


def backbone(sd, cfg, x, rec):
    """Lite_EffiBackbone.forward, efficientrep.py:553-563."""
    x = rec["backbone.conv_0"] = cbn(sd, "backbone.conv_0", x, 2, "hardswish")
    outs = []
    for s, n in enumerate(cfg["bb_repeats"], 1):
        for i in range(n):
            p = f"backbone.lite_effiblock_{s}.{i}"
            x = rec[p] = (block_s2 if i == 0 else block_s1)(sd, p, x)
        if s >= 2:
            outs.append(x)
    return outs


def neck(sd, x, rec):
    """Lite_EffiNeck.forward, reppan.py:1196-1226."""
    x2, x1, x0 = x
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")   # noqa: E731
    fpn_out0 = rec["neck.reduce_layer0"] = cbn(sd, "neck.reduce_layer0", x0, act="hardswish")
    x1 = cbn(sd, "neck.reduce_layer1", x1, act="hardswish")
    x2 = cbn(sd, "neck.reduce_layer2", x2, act="hardswish")
    f_out1 = rec["neck.Csp_p4"] = csp_block(sd, "neck.Csp_p4", torch.cat([up(fpn_out0), x1], 1))
    pan_out3 = rec["neck.Csp_p3"] = csp_block(sd, "neck.Csp_p3", torch.cat([up(f_out1), x2], 1))
    pan_out2 = rec["neck.Csp_n3"] = csp_block(sd, "neck.Csp_n3", torch.cat([dp_block(sd, "neck.downsample2", pan_out3, 2), f_out1], 1))
    pan_out1 = rec["neck.Csp_n4"] = csp_block(sd, "neck.Csp_n4", torch.cat([dp_block(sd, "neck.downsample1", pan_out2, 2), fpn_out0], 1))
    pan_out0 = rec["neck.p6"] = dp_block(sd, "neck.p6_conv_1", fpn_out0, 2) + dp_block(sd, "neck.p6_conv_2", pan_out1, 2)
    return [pan_out3, pan_out2, pan_out1, pan_out0]


def head_raw(sd, feats):
    """Detect.forward of effidehead_lite.py:58-113 up to the per-level outputs: (cls [B,A,nc] post-sigmoid, reg [B,A,4])."""
    cls_all, reg_all = [], []
    for i, x in enumerate(feats):
        x = dp_block(sd, f"detect.stems.{i}", x)
        cf = dp_block(sd, f"detect.cls_convs.{i}", x)
        rf = dp_block(sd, f"detect.reg_convs.{i}", x)
        c = F.conv2d(cf, sd[f"detect.cls_preds.{i}.weight"].to(x.dtype), sd[f"detect.cls_preds.{i}.bias"].to(x.dtype))
        r = F.conv2d(rf, sd[f"detect.reg_preds.{i}.weight"].to(x.dtype), sd[f"detect.reg_preds.{i}.bias"].to(x.dtype))
        cls_all.append(torch.sigmoid(c).flatten(2).permute(0, 2, 1))
        reg_all.append(r.flatten(2).permute(0, 2, 1))
    return torch.cat(cls_all, 1), torch.cat(reg_all, 1)


def forward(sd, cfg, x, train_outputs=False, record=None):
    """Model.forward of yolo_lite.py:31-39.  Eval: [B,A,5+nc] (reg used directly as ltrb distances); train_outputs:
    (cls, reg, sizes) of the train branch (eval-mode BN, or batch statistics inside om.train_mode())."""
    rec = {} if record is None else record
    feats = neck(sd, backbone(sd, cfg, x, rec), rec)
    sizes = [tuple(f.shape[2:]) for f in feats]
    cls, reg = head_raw(sd, feats)
    if train_outputs:
        return cls, reg, sizes
    return om.decode_eval(cfg, cls, reg, sizes)
