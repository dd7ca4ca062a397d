"""tests/golden/make_golden_qa.py -- golden vectors for the quantization-aware RepVGG networks (configs/qarepvgg), minted by
running the UNMODIFIED reference from /root/reference on CPU (build container only), in the formats of make_golden_zoo.py:

  * keys_qa.json.gz: {name: [[key, shape], ...]}, the state_dict layouts of YOLOv6-N / S / M-QA (QARepVGGBlockV2) and of
    yolov6s_qa_v1, the same S network with training_mode = 'qarepvgg' (QARepVGGBlock, no average-pool branch);
  * model_<name>.npz: eval, train-branch and deploy (fuse_model + switch_to_deploy) outputs at 64 px, batch 2, for the three
    QA models; model_yolov6s_qa_v1.npz holds the eval output of the v1 network;
  * train_yolov6{n,m}_qa.npz: float64 train-mode head outputs, L, every parameter-gradient norm and full gradients of a few
    tensors (the stem, a bare rbr_1x1 weight, a post-sum bn weight, a BottleRep alpha).

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_qa.py
"""
import gzip
import json
import os
import sys

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

MODELS = ["yolov6n_qa", "yolov6s_qa", "yolov6m_qa"]
SIZE = 64
TRAIN = {"yolov6n_qa": (2, 64), "yolov6m_qa": (2, 64)}                      # name -> (batch, size)
FULL = {  # gradients stored in full
    "yolov6n_qa": ["backbone.stem.rbr_dense.conv.weight", "backbone.stem.rbr_1x1.weight", "backbone.stem.bn.weight",
                   "backbone.ERBlock_3.1.conv1.rbr_1x1.weight", "backbone.ERBlock_3.1.conv1.bn.weight",
                   "backbone.ERBlock_3.1.conv1.rbr_dense.bn.bias", "detect.cls_preds.1.bias"],
    "yolov6m_qa": ["backbone.stem.rbr_1x1.weight", "backbone.ERBlock_3.1.m.conv1.alpha", "backbone.ERBlock_3.1.m.conv1.conv2.rbr_1x1.weight",
                   "backbone.ERBlock_3.1.m.conv1.conv2.bn.weight", "neck.Rep_n3.m.conv1.conv1.bn.bias", "detect.reg_preds.1.bias"],
}
BN = {"yolov6n_qa": "backbone.ERBlock_2.1.conv1.bn", "yolov6m_qa": "backbone.ERBlock_2.0.bn"}


def load_cfg(name, mode="qarepvggv2"):
    cfg = Config.fromfile(f"/root/reference/configs/qarepvgg/{name}.py")
    assert cfg.training_mode == "qarepvggv2"
    cfg.training_mode = mode
    return cfg


def golden_models():
    layouts = {}
    for name, mode in [(n, "qarepvggv2") for n in MODELS] + [("yolov6s_qa_v1", "qarepvgg")]:
        m = build_model(load_cfg(name.replace("_v1", ""), mode), 80, torch.device("cpu"))
        keys = layouts[name] = [(k, list(v.shape)) for k, v in m.state_dict().items()]
        sd = fab.fabricate_state_dict(keys, seed=0)
        m.load_state_dict(sd, strict=True)
        m.eval()
        x = fab.synthetic_images(2, SIZE, SIZE, seed=0)
        store = dict(x_checksum=np.float64(fab.checksum(x)), w_checksum=np.float64(sum(fab.checksum(v) for v in sd.values())))
        with torch.no_grad():
            store["eval_out"] = m(x)[0].numpy()
            if mode == "qarepvggv2":
                m.detect.training = True           # train branch of Detect.forward with eval-mode BN
                _, cls_t, reg_t = m.detect(list(m.neck(m.backbone(x))))
                m.detect.training = False
                fuse_model(m)                       # reference deploy order: fuse BN, then re-parameterise
                for layer in m.modules():
                    if isinstance(layer, RepVGGBlock):
                        layer.switch_to_deploy()
                store.update(cls_train=cls_t.numpy(), reg_train=reg_t.numpy(), deploy_out=m(x)[0].numpy())
        np.savez_compressed(os.path.join(HERE, f"model_{name}.npz"), **store)
        drift = float(np.abs(store["eval_out"] - store.get("deploy_out", store["eval_out"])).max())
        print(name, len(keys), "keys", store["eval_out"].shape, "deploy drift", drift)
    with gzip.GzipFile(os.path.join(HERE, "keys_qa.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(layouts).encode())


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
    print("golden vectors written to", HERE)
