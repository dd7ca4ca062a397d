"""tests/golden/make_golden_letterbox.py -- golden letterbox canvases and rescaled boxes from the UNMODIFIED reference
(yolov6/data/data_augment.py:29-58 `letterbox`, yolov6/core/inferer.py:161-188 `Inferer.process_image` / `Inferer.rescale`)
and the cv2 it calls, on the seeded sources of oracle/letterbox.py (build container only).

    PYTHONPATH=tests/golden/refshim:/root/reference:. python tests/golden/make_golden_letterbox.py

Writes letterbox_cases.json (shapes, the reference's r / left / top, source checksums, the SHA-256 of each canvas -- uint8
[3, H, W] as Inferer.process_image sees it before `/255` -- and per case the pixels where the oracle's restatement differs
from cv2: none with the cv2 this was generated with) and letterbox.npz (rescale inputs and outputs).  The canvases are kept
as digests: a byte-identical canvas has the same digest, and the noise canvases would not compress.
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

NO_STRIDE = 1 << 20      # process_image pads to a stride multiple (auto=True); a stride above any canvas pads to the full canvas

if __name__ == "__main__":
    store, cases = {}, []
    for i, (h0, w0, H, W, scaleup, kind) in enumerate(ol.CASES):
        im = ol.synthetic_source(h0, w0, kind, i)
        _, r, (left, top) = letterbox(im.copy(), (H, W), auto=False, scaleup=scaleup)
        if scaleup:
            x, _ = Inferer.process_image(im.copy(), (H, W), NO_STRIDE, False)
            canvas = (x * 255).round().to(torch.uint8).numpy()
        else:                 # process_image always scales up; the Evaler's dataset path calls letterbox with scaleup=False
            lb = letterbox(im.copy(), (H, W), auto=False, scaleup=False)[0]
            canvas = np.ascontiguousarray(lb.transpose(2, 0, 1)[::-1])
        assert canvas.shape == (3, H, W)
        diff = np.abs(canvas.astype(np.int64) - ol.letterbox(im, H, W, scaleup).astype(np.int64))
        cases.append(dict(h0=h0, w0=w0, H=H, W=W, scaleup=scaleup, kind=kind, seed=i, r=r, left=left, top=top,
                          src_sum=int(im.astype(np.int64).sum()),
                          canvas_sha256=hashlib.sha256(np.ascontiguousarray(canvas).tobytes()).hexdigest(), oracle_mismatch=int((diff > 0).sum()),
                          oracle_max_diff=int(diff.max())))
        print(i, (h0, w0), "->", (H, W), "scaleup" if scaleup else "no-scaleup", kind, "r", r, "left/top", left, top,
              "oracle mismatches", int((diff > 0).sum()))
    for j, (h0, w0, H, W) in enumerate(ol.RESCALE_CASES):
        det = ol.synthetic_detections(H, W, j)
        ref = torch.from_numpy(det.copy())
        ref[:, :4] = Inferer.rescale((H, W), ref[:, :4], (h0, w0, 3)).round()
        store[f"r{j}_det"] = det
        store[f"r{j}_out"] = ref.numpy()
        assert np.array_equal(ref.numpy(), ol.rescale(det, H, W, h0, w0))
    np.savez_compressed(os.path.join(HERE, "letterbox.npz"), **store)
    with open(os.path.join(HERE, "letterbox_cases.json"), "w") as f:
        json.dump(dict(cv2=cv2.__version__, cases=cases, rescale_cases=[list(c) for c in ol.RESCALE_CASES]), f, indent=1)
