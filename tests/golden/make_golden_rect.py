"""tests/golden/make_golden_rect.py -- golden minimum-rectangle (letterbox auto=True) canvases and rescaled boxes from the
UNMODIFIED reference: Inferer.check_img_size, Inferer.process_image(im, img_size, stride, False) and Inferer.rescale
(yolov6/core/inferer.py:161-209) with the cv2 they call, on seeded sources (oracle/letterbox.py's synthetic_source) at the
strides Inferer uses: 32 for the P5 detectors at 640, 64 for the P6 ones at 1280 and for Lite at 320 (build container only).

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_rect.py

Writes rect_cases.json (per case: the source, img_size and stride, the checked img_size, the canvas shape, the reference's
r / left / top, the SHA-256 of the uint8 [3, H, W] canvas Inferer.process_image gives before `/255`) and rect.npz (per case
seeded NMS-like rows on that canvas and their Inferer.rescale(...).round()).
"""
import hashlib
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(HERE, "refshim"), "/root/reference", ROOT]
warnings.filterwarnings("ignore")
torch.cuda.is_available = lambda: False

import cv2  # noqa: E402
from yolov6.core.inferer import Inferer  # noqa: E402
from yolov6.data.data_augment import letterbox  # noqa: E402

from oracle import letterbox as ol  # noqa: E402

# (h0, w0, kind): 1080p, 720p, portrait 1080p, 4:3 VGA, odd sizes, a tiny frame and one that is scaled up
SOURCES = [(1080, 1920, "noise"), (720, 1280, "grad"), (1920, 1080, "noise"), (480, 640, "grad"), (333, 517, "noise"),
           (3, 5, "grad"), (200, 300, "noise")]
# (img_size, stride): P5 at 640, P6 at 1280, Lite at 320; 600 is not a multiple of 32 and is rounded up to 608
SIZES = [(640, 32), (1280, 64), (320, 64), (600, 32)]

if __name__ == "__main__":
    inferer = Inferer.__new__(Inferer)          # check_img_size / make_divisible use no other state
    store, cases = {}, []
    for j, (img_size, stride) in enumerate(SIZES):
        checked = inferer.check_img_size(img_size, s=stride)
        for i, (h0, w0, kind) in enumerate(SOURCES):
            if img_size == 600 and i > 1:
                continue
            im = ol.synthetic_source(h0, w0, kind, 100 + i)
            _, r, (left, top) = letterbox(im.copy(), checked, stride=stride)
            x, _ = Inferer.process_image(im.copy(), checked, stride, False)
            canvas = (x * 255).round().to(torch.uint8).numpy()
            H, W = canvas.shape[1:]
            k = len(cases)
            det = ol.synthetic_detections(H, W, 200 + k)
            ref = torch.from_numpy(det.copy())
            ref[:, :4] = Inferer.rescale((H, W), ref[:, :4], (h0, w0, 3)).round()
            store[f"c{k}_det"], store[f"c{k}_out"] = det, ref.numpy()
            cases.append(dict(h0=h0, w0=w0, kind=kind, seed=100 + i, img_size=img_size, stride=stride, checked=list(checked),
                              H=int(H), W=int(W), r=float(r), left=int(left), top=int(top), src_sum=int(im.astype(np.int64).sum()),
                              canvas_sha256=hashlib.sha256(np.ascontiguousarray(canvas).tobytes()).hexdigest()))
            print(k, (h0, w0), "img_size", img_size, "stride", stride, "->", (H, W), "r", r, "left/top", left, top)
    np.savez_compressed(os.path.join(HERE, "rect.npz"), **store)
    with open(os.path.join(HERE, "rect_cases.json"), "w") as f:
        json.dump(dict(cv2=cv2.__version__, cases=cases), f, indent=1)
