"""tests/golden/make_golden_zoo.py -- golden vectors for the rest of the reference's released detectors, minted by running the
UNMODIFIED reference from /root/reference on CPU (build container only), in the formats of the older scripts:

  * keys_zoo.json.gz: {name: [[key, shape], ...]}, the state_dict layout of each model (the content of make_golden.py's
    keys_<name>.json, in one compressed file);
  * model_<name>.npz (make_golden.py): eval, train-branch and deploy outputs at 64 px (P5) or 128 px (P6), batch 2, for
    YOLOv6-L, -N6, -S6, -M6 and the four MBLA models (configs/mbla);
  * configs_zoo.npz (make_golden_configs.py): YOLOv6-N6 at 1280 px batch 1 and YOLOv6-S-MBLA at 640 px batch 4, every
    32nd anchor row of the [B, A, 85] output plus float64 column sums over all rows;
  * train_<name>.npz (make_golden_train.py): train-mode head outputs, L, every parameter-gradient norm and full gradients
    of a few tensors for YOLOv6-N6 and YOLOv6-S-MBLA, in float64.

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_zoo.py
"""
import gzip
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(HERE, "refshim"), "/root/reference", ROOT]

torch.cuda.is_available = lambda: False
nn.Module.cuda = lambda self, *a, **k: self

from yolov6.layers.common import RepVGGBlock  # noqa: E402
from yolov6.models.yolo import build_model  # noqa: E402
from yolov6.utils.config import Config  # noqa: E402
from yolov6.utils.torch_utils import fuse_model  # noqa: E402

from oracle import fabricate as fab  # noqa: E402

MODELS = {"yolov6l": 64, "yolov6n6": 128, "yolov6s6": 128, "yolov6m6": 128,
          "yolov6s_mbla": 64, "yolov6m_mbla": 64, "yolov6l_mbla": 64, "yolov6x_mbla": 64}   # name -> golden input size
NATIVE = [("yolov6n6", 1, 1280, 32), ("yolov6s_mbla", 4, 640, 32)]                         # name, batch, size, row stride
TRAIN = {"yolov6n6": (2, 128), "yolov6s_mbla": (2, 64)}                                     # name -> (batch, size)
FULL = {  # gradients stored in full
    "yolov6n6": ["backbone.ERBlock_6.0.rbr_dense.bn.weight", "backbone.ERBlock_6.1.conv1.rbr_identity.weight",
                 "backbone.ERBlock_6.2.cspsppf.cv7.block.bn.bias", "detect.cls_preds.3.bias"],
    "yolov6s_mbla": ["backbone.ERBlock_3.1.cv1.conv.weight", "backbone.ERBlock_3.1.cv1.bn.weight", "backbone.ERBlock_3.1.m.1.0.alpha",
                     "backbone.ERBlock_3.1.m.1.1.conv3.block.bn.weight", "detect.reg_preds.1.bias"],
}
BN = {"yolov6n6": "backbone.ERBlock_2.0.rbr_dense.bn", "yolov6s_mbla": "backbone.ERBlock_2.0.block.bn"}


def load_cfg(name):
    path = f"/root/reference/configs/{'mbla/' if name.endswith('_mbla') else ''}{name}.py"
    cfg = Config.fromfile(path)
    if not hasattr(cfg, "training_mode"):
        setattr(cfg, "training_mode", "repvgg")  # tools/train.py:99-100
    return cfg


def golden_models():
    layouts = {}
    for name, size in MODELS.items():
        m = build_model(load_cfg(name), 80, torch.device("cpu"))
        keys = layouts[name] = [(k, list(v.shape)) for k, v in m.state_dict().items()]
        sd = fab.fabricate_state_dict(keys, seed=0)
        m.load_state_dict(sd, strict=True)
        m.eval()
        x = fab.synthetic_images(2, size, size, seed=0)
        with torch.no_grad():
            out_eval = m(x)[0]
            m.detect.training = True           # train branch of Detect.forward with eval-mode BN
            feats = m.neck(m.backbone(x))
            _, cls_t, reg_t = m.detect(list(feats))
            m.detect.training = False
            fuse_model(m)                       # reference deploy order: fuse BN, then re-parameterise
            for layer in m.modules():
                if isinstance(layer, RepVGGBlock):
                    layer.switch_to_deploy()
            out_deploy = m(x)[0]
        np.savez_compressed(os.path.join(HERE, f"model_{name}.npz"), eval_out=out_eval.numpy(),
                            cls_train=cls_t.numpy(), reg_train=reg_t.numpy(), deploy_out=out_deploy.numpy(),
                            x_checksum=np.float64(fab.checksum(x)),
                            w_checksum=np.float64(sum(fab.checksum(v) for v in sd.values())))
        print(name, len(keys), "keys", tuple(out_eval.shape), "deploy drift", (out_eval - out_deploy).abs().max().item())
    with gzip.GzipFile(os.path.join(HERE, "keys_zoo.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(layouts).encode())


def golden_native():
    store = {}
    for name, B, size, step in NATIVE:
        m = build_model(load_cfg(name), 80, torch.device("cpu"))
        keys = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
        m.load_state_dict(fab.fabricate_state_dict(keys, seed=0), strict=True)
        m.eval()
        x = fab.synthetic_images(B, size, size, seed=40)
        t0 = time.time()
        with torch.no_grad():
            out = m(x)[0]
        print(name, tuple(out.shape), f"{time.time() - t0:.1f}s")
        store[f"{name}_rows"] = out[:, ::step].numpy()
        store[f"{name}_colsum"] = out.double().sum(1).numpy()
        store[f"{name}_abs_colsum"] = out.double().abs().sum(1).numpy()
        store[f"{name}_x_checksum"] = np.float64(fab.checksum(x))
    np.savez_compressed(os.path.join(HERE, "configs_zoo.npz"), **store)


def golden_train():
    for name, (B, size) in TRAIN.items():
        m = build_model(load_cfg(name), 80, torch.device("cpu"))
        keys = [(k, list(v.shape)) for k, v in m.state_dict().items()]
        sd = fab.fabricate_state_dict(keys, seed=0)
        for k in sd:      # keep the head logits O(1) under batch-statistics BN
            if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
                sd[k] = sd[k] * 0.1
            if k.endswith(".alpha"):
                sd[k] = sd[k] * 0.75
        m.load_state_dict(sd, strict=True)
        m = m.double()
        m.train()
        x = fab.synthetic_images(B, size, size, seed=7).double()
        (feats, cls, reg), _ = m(x)
        g = torch.Generator().manual_seed(11)
        wc = torch.randn(cls.shape, generator=g).double()
        wr = torch.randn(reg.shape, generator=g).double()
        L = (cls * wc).sum() + (reg * wr).sum()
        L.backward()
        names = [k for k, p in m.named_parameters() if p.grad is not None]
        store = dict(cls=cls.detach().numpy(), reg=reg.detach().numpy(), L=np.float64(L.item()),
                     grad_names=np.array(names), grad_norms=np.array([float(p.grad.norm()) for k, p in m.named_parameters()
                                                                       if p.grad is not None]),
                     x_checksum=np.float64(fab.checksum(x.float())))
        params = dict(m.named_parameters())
        missing = [k for k in FULL[name] if k not in params]
        assert not missing, missing
        for k in FULL[name]:
            store["grad::" + k] = params[k].grad.numpy()
        bufs = dict(m.named_buffers())
        store["bn_name"] = np.array(BN[name])
        store["running_mean"] = bufs[BN[name] + ".running_mean"].numpy()
        store["running_var"] = bufs[BN[name] + ".running_var"].numpy()
        np.savez_compressed(os.path.join(HERE, f"train_{name}.npz"), **store)
        print(name, "L", L.item(), "params with grad", len(names), "feat shapes", [tuple(f.shape) for f in feats])


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_models()
    golden_train()
    golden_native()
    print("golden vectors written to", HERE)
