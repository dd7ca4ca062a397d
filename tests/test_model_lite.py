"""The YOLOv6Lite-S / M / L detectors on the CPU.

Pins oracle/lite.py to the goldens of tests/golden/make_golden_lite.py, the built graphs (state_dict layout, folded weights,
the 16-aligned channel windows of the 1x1 convs and the launch list) to the oracle, checkpoint matching, the refusals of
Lite training, the conv planner on every Lite conv launch, and the ctypes mirrors of the Lite descriptors."""
import ctypes as C
import functools
import gzip
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT, golden_npz
from oracle import fabricate as fab
from oracle import lite
from yolov6_b200 import _lib, arch, configs, ops
from yolov6_b200.checkpoint import _matching_config
from yolov6_b200.engine import forward_launches, stem_channels, window_weights
from yolov6_b200.fold import fold_op, se_weights
from yolov6_b200.model import build_model

NAMES = ["yolov6lite_s", "yolov6lite_m", "yolov6lite_l"]


@functools.lru_cache(maxsize=None)
def _layouts():
    with gzip.open(os.path.join(GOLDEN, "keys_lite.json.gz")) as f:
        return json.load(f)


def lite_keys(name):
    return [(k, tuple(shape)) for k, shape in _layouts()[name]]


def rel_err(a, b):
    return float((np.abs(a - b) / (1.0 + np.abs(b))).max())


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def reference_config(name):
    """The reference's Config of configs/yolov6_lite/yolov6_lite_*.py: `model.type` 'YOLOv6-lite-*', no depth_multiple and
    no training_mode."""
    c = configs.get_config(name)
    return _Cfg(model=_Cfg(pretrained=None, **{k: _Cfg(v) if isinstance(v, dict) else v for k, v in c.items()}))


def test_widths_follow_the_lite_make_divisible():
    want = {"yolov6lite_s": ([24, 32, 48, 96, 176], [8, 12, 24, 44]), "yolov6lite_m": ([24, 32, 64, 144, 288], [8, 16, 36, 72]),
            "yolov6lite_l": ([24, 48, 96, 192, 384], [12, 24, 48, 96])}
    for name, (out, half_mid) in want.items():
        o, mid, neck_in = arch.lite_channels(configs.get_config(name))
        assert o == out and [m // 2 for m in mid[1:]] == half_mid and neck_in == out[:1:-1]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_reference_layout(name):
    want = lite_keys(name)
    assert len(want) == 820
    for cfg in (name, reference_config(name)):
        m = build_model(cfg, 80, "cpu")
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == dict(want)
        m.load_state_dict(fab.fabricate_state_dict(want, seed=0), strict=True)
    d = m.detect
    assert (d.nc, d.no, d.nl, d.prior_prob, d.grid_cell_offset, d.grid_cell_size) == (80, 85, 4, 1e-2, 0.5, 5.0)
    assert torch.equal(d.stride, torch.tensor([8, 16, 32, 64])) and len(d.grid) == 4
    assert all(len(getattr(d, n)) == 4 for n in ("stems", "cls_convs", "reg_convs", "cls_preds", "reg_preds"))
    assert not any(hasattr(d, a) for a in ("proj", "proj_conv", "use_dfl", "reg_max"))
    m = build_model(name, 80, "cpu")        # initialize_biases of effidehead_lite.py
    with torch.no_grad():
        assert float(m.detect.cls_preds[0].bias[0]) == pytest.approx(-np.log(99)) and float(m.detect.reg_preds[3].bias[2]) == 1.0
        assert float(m.detect.cls_preds[1].weight.abs().max()) == 0.0


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    g = golden_npz(f"model_{name}.npz")
    sd = fab.fabricate_state_dict(lite_keys(name), seed=0)
    x = fab.synthetic_images(2, 128, 128, seed=0)
    assert abs(fab.checksum(x) - float(g["x_checksum"])) < 1e-6 * abs(float(g["x_checksum"])), "input RNG drift"
    wsum = sum(fab.checksum(v) for v in sd.values())
    assert abs(wsum - float(g["w_checksum"])) < 1e-6 * abs(float(g["w_checksum"])), "weight RNG drift"
    cfg = lite.CONFIGS[name]
    with torch.no_grad():
        out = lite.forward(sd, cfg, x.double()).numpy()
        cls, reg, _ = lite.forward(sd, cfg, x.double(), train_outputs=True)
    assert out.shape == (2, 340, 85)
    assert rel_err(out, g["eval_out"]) < 1e-5
    assert rel_err(cls.numpy(), g["cls_train"]) < 1e-5
    assert rel_err(reg.numpy(), g["reg_train"]) < 1e-5
    assert rel_err(out, g["deploy_out"]) < 1e-4


@pytest.mark.parametrize("name,B,H,W,step", [("yolov6lite_s", 4, 320, 320, 16), ("yolov6lite_l", 2, 192, 320, 16)])
def test_oracle_matches_reference_at_native_size(name, B, H, W, step):
    g = golden_npz("configs_lite.npz")
    sd = fab.fabricate_state_dict(lite_keys(name), seed=0)
    x = fab.synthetic_images(B, H, W, seed=40)
    assert abs(fab.checksum(x) - float(g[f"{name}_x_checksum"])) < 1e-9 * abs(float(g[f"{name}_x_checksum"])), "input RNG drift"
    with torch.no_grad():
        out = lite.forward(sd, lite.CONFIGS[name], x.double()).numpy()
    assert out.shape[1] == sum((H // s) * (W // s) for s in (8, 16, 32, 64))
    assert rel_err(out[:, ::step], g[f"{name}_rows"].astype(np.float64)) < 1e-5
    A = out.shape[1]
    assert float((np.abs(out.sum(1) - g[f"{name}_colsum"]) / (A + g[f"{name}_abs_colsum"])).max()) < 1e-5


def run_lite_cpu(g, sd, x):
    """Replays the launch list of the Lite graph in float64 on the CPU, on buffers with the engine's channel pitches: the conv
    launches read the channel window of their descriptor (forward_launches) with the zero-column weights of window_weights, the
    stem writes its padded channel count, and the depthwise / SE / shuffle / upsample ops run as their kernels define them.
    Returns (cls, reg) and the buffers."""
    N, _, H, W = x.shape
    bufs = [torch.zeros(N, b.c_total, H >> b.level, W >> b.level, dtype=torch.float64) for b in g.bufs]
    base = lambda b: (b + 1) << 32        # noqa: E731
    descs = {r.name: r.desc for r in forward_launches(g, N, H, W, 1, lambda kind, key, q=0: base(key) if kind == "buf" else 1 << 20,
                                                      lambda d: {"halo": 0}) if r.kind == "conv"}
    heads = {"cls": [None] * 4, "reg": [None] * 4}
    act = {"hardswish": F.hardswish, "sigmoid": torch.sigmoid, None: lambda t: t}

    def rd(t):
        return bufs[t.buf][:, t.c_off:t.c_off + t.c]

    for i, op in enumerate(g.ops):
        if op.kind == "se":
            w1, b1, w2, b2 = se_weights(sd, op)
            t = rd(op.src)
            s = F.hardsigmoid(torch.relu(t.mean((2, 3)) @ w1.t() + b1) @ w2.t() + b2)
            t.mul_(s[:, :, None, None])
        elif op.kind == "shuffle":
            rd(op.dst)[:, 0::2] = rd(op.src)
            rd(op.dst)[:, 1::2] = rd(op.src2)
        elif op.kind == "up":
            rd(op.dst).copy_(F.interpolate(rd(op.src), scale_factor=2, mode="nearest"))
        elif op.kind == "dw":
            w, b = fold_op(sd, op)
            rd(op.dst).copy_(act[op.act](F.conv2d(rd(op.src), w.permute(0, 3, 1, 2), b, op.s, op.k // 2, 1, op.cin)))
        elif op.kind == "stem":
            w, b = fold_op(sd, op)
            cp = stem_channels(g, op)
            w, b = torch.cat([w, w.new_zeros((cp - op.cout,) + w.shape[1:])]), torch.cat([b, b.new_zeros(cp - op.cout)])
            bufs[op.dst.buf][:] = act[op.act](F.conv2d(x.double(), w.permute(0, 3, 1, 2), b, 2, 1))
        else:
            d = descs[op.name]
            off = (d.x - base(op.src.buf)) // 2
            w, b = fold_op(sd, op)
            w = window_weights(g, op, w)
            assert w.shape[-1] == d.Cin
            y = act[op.act](F.conv2d(bufs[op.src.buf][:, off:off + d.Cin], w.permute(0, 3, 1, 2), b))
            if op.res is not None:
                y = y + rd(op.res)
            if op.kind == "pred":
                heads[op.head[0]][op.head[1]] = y.flatten(2).permute(0, 2, 1)
            else:
                rd(op.dst).copy_(y)
    return torch.cat(heads["cls"], 1), torch.cat(heads["reg"], 1), bufs


@pytest.mark.parametrize("name,H,W", [("yolov6lite_s", 128, 128), ("yolov6lite_m", 128, 128), ("yolov6lite_l", 192, 320)])
def test_folded_launch_replay_equals_oracle(name, H, W):
    sd = fab.fabricate_state_dict(lite_keys(name), 0)
    x = fab.synthetic_images(1, H, W, seed=3)
    g = arch.build_graph(configs.get_config(name), 80)
    with torch.no_grad():
        cls, reg, bufs = run_lite_cpu(g, sd, x)
        rec = {}
        ocls, oreg, _ = lite.forward(sd, lite.CONFIGS[name], x.double(), train_outputs=True, record=rec)
    assert float((cls - ocls).abs().max()) < 1e-9
    assert float((reg - oreg).abs().max()) < 1e-9
    used = [set() for _ in bufs]
    for op in g.ops:
        for t in (op.src, op.src2, op.dst, op.res):
            if t is not None:
                used[t.buf].update(range(t.c_off, t.c_off + t.c))
    for j, b in enumerate(bufs):     # pad channels stay zero, so the zero weight columns of the windows multiply zeros
        pad = [c for c in range(b.shape[1]) if c not in used[j]]
        assert b.shape[1] % 16 == 0 and (not pad or float(b[:, pad].abs().max()) == 0.0), g.bufs[j].name
    feats = [bufs[t.buf][:, t.c_off:t.c_off + t.c] for t in g.feat]
    for f, key in zip(feats, ("neck.Csp_p3", "neck.Csp_n3", "neck.Csp_n4", "neck.p6")):
        assert float((f - rec[key]).abs().max()) < 1e-9, key


H100 = (132, 232448, 66)


def _plan(d):
    out = (C.c_int32 * 12)()
    rc = _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(ops.PLAN_KEYS, out))


@pytest.mark.parametrize("name", NAMES)
def test_every_conv_launch_is_aligned_and_gets_a_plan_that_fits_the_sm(name):
    g = arch.build_graph(configs.get_config(name), 80, name)
    for batch, H, W in ((32, 320, 320), (1, 192, 320), (2, 128, 128)):
        convs = [r for r in forward_launches(g, batch, H, W, 1, lambda *key: 1 << 20, _plan) if r.kind == "conv"]
        assert len(convs) == sum(1 for op in g.ops if op.kind in ("conv", "pred"))
        for r in convs:
            d = r.desc
            assert d.Cin % 16 == 0 and d.x % 16 == 0 and d.x_c_total % 16 == 0, (r.name, d.Cin, d.x)
            p = _plan(d)
            assert 0 < p["smem"] <= H100[1] and p["threads"] == 384, (r.name, p)
            assert 1 <= p["grid"] <= H100[0] and p["stages"] >= 2, (r.name, p)


def test_every_lite_layout_is_matched_back_to_its_name():
    for name in NAMES:
        assert _matching_config(fab.fabricate_state_dict(lite_keys(name), seed=0), 80) == name


def test_lite_training_and_training_heads_are_refused():
    m = build_model("yolov6lite_s", 80, "cpu")
    with pytest.raises(NotImplementedError, match="YOLOv6Lite"):
        m.train()(torch.zeros(1, 3, 64, 64))
    with pytest.raises(NotImplementedError, match="YOLOv6Lite"):
        m.train_engine()
    from yolov6_b200.step import TrainStep
    with pytest.raises(NotImplementedError, match="YOLOv6Lite"):
        TrainStep(m, None, 2, 64, 64, graph=False)
    for kw in (dict(fuse_ab=True), dict(distill_ns=True)):
        with pytest.raises(ValueError, match="YOLOv6Lite"):
            build_model("yolov6lite_m", 80, "cpu", **kw)


def test_ctypes_mirrors_of_the_lite_descriptors_match_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "yv6.h"\nint main(){printf("%zu %zu\\n", sizeof(yv6_dw_desc), sizeof(yv6_se_desc));'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.DwDesc), C.sizeof(_lib.SeDesc)]
