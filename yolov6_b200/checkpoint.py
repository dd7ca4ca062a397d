"""Checkpoints of the reference for the drop-in model.

The reference saves *pickled modules* (`{'model': Model, 'ema': Model, ...}`, core/engine.py:178-196) and loads them
with `load_checkpoint` (yolov6/utils/checkpoint.py:22-32), which returns the unpickled `yolov6.models.yolo.Model`
itself -- an object of the reference's class, whose `forward` is the reference's PyTorch path.  An import swap therefore
does not reach released `.pt` files.  `from_reference(module)` converts such a module into the kernel-backed model (same
`state_dict()` keys and shapes, so the conversion is `load_state_dict`), and `load_checkpoint` here mirrors the
reference's function on top of it: same arguments, returns a model in eval mode.  `fuse` is accepted for signature
compatibility; BN folding / RepVGG re-parameterisation happen inside the inference engine either way (fold.py).
"""
import torch

from . import arch, configs
from .model import Model


def _matching_config(sd, num_classes):
    """The built-in configuration whose state_dict has exactly these keys and shapes (each built-in layout is unique)."""
    want = {k: tuple(v.shape) for k, v in sd.items()}
    for name in configs.CONFIGS:
        have = {k: tuple(shape) for k, shape, _ in arch.param_specs(arch.build_graph(configs.get_config(name), num_classes))}
        if have == want:
            return name
    return None


def strip_deploy_keys(sd):
    """A module that went through `fuse_model` / `switch_to_deploy` (inferer.py:59-68) no longer holds train-form tensors."""
    return any(".rbr_reparam." in k for k in sd)


def from_reference(module, cfg=None, device=None):
    """module: an instance of the reference's `yolov6.models.yolo.Model` (e.g. `ckpt['model']`), train form.
    cfg: the reference Config / a built-in name / None (then the built-in configurations are matched against the
    module's state_dict).  Returns a `yolov6_b200.model.Model` with the same weights, mode (train / eval) and device."""
    sd = {k: v.detach().float() if v.dtype.is_floating_point else v.detach() for k, v in module.state_dict().items()}
    if strip_deploy_keys(sd):
        raise RuntimeError("the module is already in deploy form (rbr_reparam); convert the train-form checkpoint instead -- "
                           "yolov6_b200 folds BatchNorm and the RepVGG branches itself")
    det = getattr(module, "detect", None)
    nc = int(getattr(det, "nc", 80))
    if cfg is None:
        cfg = _matching_config(sd, nc)
        if cfg is None:
            raise RuntimeError(f"no built-in configuration ({', '.join(configs.CONFIGS)}) has this state_dict layout; "
                               "pass the reference Config as `cfg`")
    m = Model(cfg, num_classes=nc)
    m.load_state_dict(sd, strict=True)
    if device is None:
        p = next(iter(module.parameters()), None)
        device = p.device if p is not None else torch.device("cpu")
    m = m.to(device)
    m.train(module.training)
    return m


def load_checkpoint(weights, map_location=None, inplace=True, fuse=True, cfg=None):
    """yolov6/utils/checkpoint.py:22-32 for the drop-in model: `weights` is a `.pt` written by the reference's Trainer
    (pickled modules -- the reference package must be importable for unpickling) or a file holding a plain state_dict
    under 'model'."""
    ckpt = torch.load(weights, map_location=map_location, weights_only=False)
    obj = ckpt['ema' if ckpt.get('ema') else 'model']
    if isinstance(obj, dict):
        if cfg is None:
            cfg = _matching_config(obj, 80)
        m = Model(cfg)
        m.load_state_dict(obj, strict=True)
        return m.eval()
    if isinstance(obj, Model):
        return obj.float().eval()
    return from_reference(obj.float(), cfg=cfg).eval()
