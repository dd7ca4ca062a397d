"""tests/golden/make_golden_lite.py -- golden vectors for the YOLOv6Lite-S / M / L detectors, minted by running the UNMODIFIED
reference from /root/reference on CPU (build container only), in the formats of make_golden_zoo.py:

  * keys_lite.json.gz: {name: [[key, shape], ...]}, the state_dict layout of each model;
  * model_yolov6lite_{s,m,l}.npz: eval, train-branch and `fuse_model` deploy outputs at 128 px, batch 2;
  * configs_lite.npz: Lite-S at 320 x 320 batch 4 and Lite-L at 192 x 320 batch 2 (rectangular: catches H / W mix-ups),
    every 16th anchor row of the [B, A, 85] output plus float64 column sums over all rows.

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_lite.py
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

from yolov6.models.yolo_lite import build_model  # noqa: E402
from yolov6.utils.config import Config  # noqa: E402
from yolov6.utils.torch_utils import fuse_model  # noqa: E402

from oracle import fabricate as fab  # noqa: E402

MODELS = {"yolov6lite_s": "s", "yolov6lite_m": "m", "yolov6lite_l": "l"}
NATIVE = [("yolov6lite_s", 4, 320, 320, 16), ("yolov6lite_l", 2, 192, 320, 16)]     # name, batch, H, W, row stride


def load_model(name):
    cfg = Config.fromfile(f"/root/reference/configs/yolov6_lite/yolov6_lite_{MODELS[name]}.py")
    m = build_model(cfg, 80, torch.device("cpu"))
    keys = [(k, list(v.shape)) for k, v in m.state_dict().items()]
    sd = fab.fabricate_state_dict(keys, seed=0)
    m.load_state_dict(sd, strict=True)
    return m.eval(), keys, sd


def golden_models():
    layouts = {}
    for name in MODELS:
        m, keys, sd = load_model(name)
        layouts[name] = keys
        x = fab.synthetic_images(2, 128, 128, seed=0)
        with torch.no_grad():
            out_eval = m(x)[0]
            m.detect.training = True           # train branch of Detect.forward with eval-mode BN
            _, cls_t, reg_t = m.detect(list(m.neck(m.backbone(x))))
            m.detect.training = False
            fuse_model(m)
            out_deploy = m(x)[0]
        np.savez_compressed(os.path.join(HERE, f"model_{name}.npz"), eval_out=out_eval.numpy(),
                            cls_train=cls_t.numpy(), reg_train=reg_t.numpy(), deploy_out=out_deploy.numpy(),
                            x_checksum=np.float64(fab.checksum(x)),
                            w_checksum=np.float64(sum(fab.checksum(v) for v in sd.values())))
        print(name, len(keys), "keys", tuple(out_eval.shape), "deploy drift", (out_eval - out_deploy).abs().max().item())
    with gzip.GzipFile(os.path.join(HERE, "keys_lite.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(layouts).encode())


def golden_native():
    store = {}
    for name, B, H, W, step in NATIVE:
        m, _, _ = load_model(name)
        x = fab.synthetic_images(B, H, W, seed=40)
        t0 = time.time()
        with torch.no_grad():
            out = m(x)[0]
        print(name, tuple(out.shape), f"{time.time() - t0:.1f}s")
        store[f"{name}_rows"] = out[:, ::step].numpy()
        store[f"{name}_colsum"] = out.double().sum(1).numpy()
        store[f"{name}_abs_colsum"] = out.double().abs().sum(1).numpy()
        store[f"{name}_x_checksum"] = np.float64(fab.checksum(x))
    np.savez_compressed(os.path.join(HERE, "configs_lite.npz"), **store)


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_models()
    golden_native()
    print("golden vectors written to", HERE)
