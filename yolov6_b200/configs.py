"""Built-in model configurations (the `model` dict and `training_mode` of reference configs/yolov6{n,s,m,l,n6,s6,m6,l6}.py and
configs/mbla/yolov6{s,m,l,x}_mbla.py, and the YOLOv6Lite models of configs/yolov6_lite/yolov6_lite_{s,m,l}.py under their release
names yolov6lite_{s,m,l}, and the quantization-aware RepVGG networks of configs/qarepvgg/yolov6{n,s,m}_qa.py; `training_mode`
defaults to "repvgg" as tools/train.py:99-100 does) so that
tests, smoke() and bench.py run where /root/reference is not mounted, plus a normaliser that accepts
the reference's own mmcv-style Config object (yolov6/utils/config.py) for drop-in use."""
import copy

_P5_HEAD = dict(type="EffiDeHead", in_channels=[128, 256, 512], num_layers=3, begin_indices=24, anchors=3,
                anchors_init=[[10, 13, 19, 19, 33, 23], [30, 61, 59, 59, 59, 119], [116, 90, 185, 185, 373, 326]],   # fuse_ab head
                out_indices=[17, 20, 23], strides=[8, 16, 32], atss_warmup_epoch=0)
_P6_HEAD = dict(type="EffiDeHead", in_channels=[128, 256, 512, 1024], num_layers=4, anchors=1, strides=[8, 16, 32, 64],
                atss_warmup_epoch=4)

CONFIGS = {
    "yolov6n": dict(
        training_mode="repvgg", depth_multiple=0.33, width_multiple=0.25,
        backbone=dict(type="EfficientRep", num_repeats=[1, 6, 12, 18, 6], out_channels=[64, 128, 256, 512, 1024],
                      fuse_P2=True, cspsppf=True),
        neck=dict(type="RepBiFPANNeck", num_repeats=[12, 12, 12, 12], out_channels=[256, 128, 128, 256, 256, 512]),
        head=dict(_P5_HEAD, iou_type="siou", use_dfl=False, reg_max=0)),
    "yolov6s": dict(
        training_mode="repvgg", depth_multiple=0.33, width_multiple=0.50,
        backbone=dict(type="EfficientRep", num_repeats=[1, 6, 12, 18, 6], out_channels=[64, 128, 256, 512, 1024],
                      fuse_P2=True, cspsppf=True),
        neck=dict(type="RepBiFPANNeck", num_repeats=[12, 12, 12, 12], out_channels=[256, 128, 128, 256, 256, 512]),
        head=dict(_P5_HEAD, iou_type="giou", use_dfl=False, reg_max=0)),
    "yolov6m": dict(
        training_mode="repvgg", depth_multiple=0.60, width_multiple=0.75,
        backbone=dict(type="CSPBepBackbone", num_repeats=[1, 6, 12, 18, 6], out_channels=[64, 128, 256, 512, 1024],
                      csp_e=2.0 / 3, fuse_P2=True),
        neck=dict(type="CSPRepBiFPANNeck", num_repeats=[12, 12, 12, 12], out_channels=[256, 128, 128, 256, 256, 512],
                  csp_e=2.0 / 3),
        head=dict(_P5_HEAD, iou_type="giou", use_dfl=True, reg_max=16)),
    "yolov6l": dict(
        training_mode="conv_silu", depth_multiple=1.0, width_multiple=1.0,
        backbone=dict(type="CSPBepBackbone", num_repeats=[1, 6, 12, 18, 6], out_channels=[64, 128, 256, 512, 1024],
                      csp_e=0.5, fuse_P2=True),
        neck=dict(type="CSPRepBiFPANNeck", num_repeats=[12, 12, 12, 12], out_channels=[256, 128, 128, 256, 256, 512],
                  csp_e=0.5),
        head=dict(_P5_HEAD, iou_type="giou", use_dfl=True, reg_max=16)),
    "yolov6n6": dict(
        training_mode="repvgg", depth_multiple=0.33, width_multiple=0.25,
        backbone=dict(type="EfficientRep6", num_repeats=[1, 6, 12, 18, 6, 6], out_channels=[64, 128, 256, 512, 768, 1024],
                      fuse_P2=True, cspsppf=True),
        neck=dict(type="RepBiFPANNeck6", num_repeats=[12, 12, 12, 12, 12, 12], out_channels=[512, 256, 128, 256, 512, 1024]),
        head=dict(_P6_HEAD, iou_type="siou", use_dfl=False, reg_max=0)),
    "yolov6s6": dict(
        training_mode="repvgg", depth_multiple=0.33, width_multiple=0.50,
        backbone=dict(type="EfficientRep6", num_repeats=[1, 6, 12, 18, 6, 6], out_channels=[64, 128, 256, 512, 768, 1024],
                      fuse_P2=True, cspsppf=True),
        neck=dict(type="RepBiFPANNeck6", num_repeats=[12, 12, 12, 12, 12, 12], out_channels=[512, 256, 128, 256, 512, 1024]),
        head=dict(_P6_HEAD, iou_type="giou", use_dfl=False, reg_max=0)),
    "yolov6m6": dict(
        training_mode="repvgg", depth_multiple=0.60, width_multiple=0.75,
        backbone=dict(type="CSPBepBackbone_P6", num_repeats=[1, 6, 12, 18, 6, 6],
                      out_channels=[64, 128, 256, 512, 768, 1024], csp_e=2.0 / 3, fuse_P2=True),
        neck=dict(type="CSPRepBiFPANNeck_P6", num_repeats=[12, 12, 12, 12, 12, 12],
                  out_channels=[512, 256, 128, 256, 512, 1024], csp_e=2.0 / 3),
        head=dict(_P6_HEAD, iou_type="giou", use_dfl=True, reg_max=16)),
    "yolov6l6": dict(
        training_mode="conv_silu", depth_multiple=1.0, width_multiple=1.0,
        backbone=dict(type="CSPBepBackbone_P6", num_repeats=[1, 6, 12, 18, 6, 6],
                      out_channels=[64, 128, 256, 512, 768, 1024], csp_e=0.5, fuse_P2=True),
        neck=dict(type="CSPRepBiFPANNeck_P6", num_repeats=[12, 12, 12, 12, 12, 12],
                  out_channels=[512, 256, 128, 256, 512, 1024], csp_e=0.5),
        head=dict(_P6_HEAD, iou_type="giou", use_dfl=True, reg_max=16)),
}


def _mbla(depth, width):
    """configs/mbla/yolov6{s,m,l,x}_mbla.py: CSP networks with MBLABlock stages, which differ only in depth and width."""
    return dict(
        training_mode="conv_silu", depth_multiple=depth, width_multiple=width,
        backbone=dict(type="CSPBepBackbone", num_repeats=[1, 4, 8, 8, 4], out_channels=[64, 128, 256, 512, 1024],
                      csp_e=0.5, fuse_P2=True, stage_block_type="MBLABlock"),
        neck=dict(type="CSPRepBiFPANNeck", num_repeats=[8, 8, 8, 8], out_channels=[256, 128, 128, 256, 256, 512],
                  csp_e=0.5, stage_block_type="MBLABlock"),
        head=dict(_P5_HEAD, iou_type="giou", use_dfl=True, reg_max=16))


CONFIGS.update({"yolov6s_mbla": _mbla(0.5, 0.5), "yolov6m_mbla": _mbla(0.5, 0.75), "yolov6l_mbla": _mbla(0.5, 1.0),
                "yolov6x_mbla": _mbla(1.0, 1.0)})


def _lite(kind, width):
    """configs/yolov6_lite/yolov6_lite_{s,m,l}.py: one network at three widths; no depth_multiple, no training_mode."""
    return dict(
        type=f"YOLOv6-lite-{kind}", width_multiple=width,
        backbone=dict(type="Lite_EffiBackbone", num_repeats=[1, 3, 7, 3], out_channels=[24, 32, 64, 128, 256], scale_size=0.5),
        neck=dict(type="Lite_EffiNeck", in_channels=[256, 128, 64], unified_channels=96),
        head=dict(type="Lite_EffideHead", in_channels=[96, 96, 96, 96], num_layers=4, anchors=1, strides=[8, 16, 32, 64],
                  atss_warmup_epoch=4, iou_type="siou", use_dfl=False, reg_max=0))


CONFIGS.update({"yolov6lite_s": _lite("s", 0.7), "yolov6lite_m": _lite("m", 1.1), "yolov6lite_l": _lite("l", 1.5)})

# configs/qarepvgg/yolov6{n,s,m}_qa.py: the N / S / M networks built from QARepVGGBlockV2 (common.py:396-477)
CONFIGS.update({f"{n}_qa": dict(copy.deepcopy(CONFIGS[n]), training_mode="qarepvggv2") for n in ("yolov6n", "yolov6s", "yolov6m")})


def get_config(name):
    return copy.deepcopy(CONFIGS[name])


def normalize(cfg):
    """Accept a built-in name, one of the dicts above, or the reference's Config (attribute access,
    `.model.{depth_multiple,width_multiple,backbone,neck,head}`, `.training_mode`; the Lite configs have `.model.type` and
    no depth_multiple) -> plain dict."""
    if isinstance(cfg, str):
        return get_config(cfg)
    if isinstance(cfg, dict) and "backbone" in cfg:
        return copy.deepcopy(cfg)
    model = cfg["model"] if isinstance(cfg, dict) else cfg.model
    get = (lambda o, k, d=None: o.get(k, d)) if hasattr(model, "get") else (lambda o, k, d=None: getattr(o, k, d))
    mode = (cfg.get("training_mode") if isinstance(cfg, dict) else getattr(cfg, "training_mode", None)) or "repvgg"
    out = dict(training_mode=mode, depth_multiple=get(model, "depth_multiple"), width_multiple=get(model, "width_multiple"))
    for part in ("backbone", "neck", "head"):
        out[part] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in dict(get(model, part)).items()}
    if "YOLOv6-lite" in str(get(model, "type", "")):      # the trainer's Lite dispatch (core/engine.py:413-416)
        out = dict(type=get(model, "type"), width_multiple=out["width_multiple"], backbone=out["backbone"], neck=out["neck"],
                   head=out["head"])
    return out
