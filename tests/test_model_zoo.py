"""The rest of the reference's released detectors on the CPU: YOLOv6-L, -N6, -S6, -M6 and the MBLA models (configs/mbla).

Pins oracle/zoo.py to the goldens of tests/golden/make_golden_zoo.py, the built graphs (state_dict layout, folded deploy
weights) to the oracle, checkpoint matching, and the conv planner on every launch of the new networks."""
import ctypes as C
import functools
import gzip
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, golden_npz
from oracle import fabricate as fab
from oracle import zoo
from test_graph import _run_graph_cpu
from yolov6_b200 import _lib, arch, configs, ops
from yolov6_b200.checkpoint import _matching_config
from yolov6_b200.engine import forward_launches, siblings
from yolov6_b200.model import Model, build_model

MODELS = {"yolov6l": 64, "yolov6n6": 128, "yolov6s6": 128, "yolov6m6": 128,
          "yolov6s_mbla": 64, "yolov6m_mbla": 64, "yolov6l_mbla": 64, "yolov6x_mbla": 64}   # name -> golden input size
NEW = list(MODELS)


@functools.lru_cache(maxsize=None)
def _layouts():
    with gzip.open(os.path.join(GOLDEN, "keys_zoo.json.gz")) as f:
        return json.load(f)


def zoo_keys(name):
    """The reference's state_dict layout of `name`: [(key, shape)] (tests/golden/make_golden_zoo.py)."""
    return [(k, tuple(shape)) for k, shape in _layouts()[name]]


def rel_err(a, b):
    return float((np.abs(a - b) / (1.0 + np.abs(b))).max())


class _Cfg(dict):
    """The reference's mmcv-style Config: attribute access, `.model.{backbone,neck,head}`, `.training_mode`."""
    __getattr__ = dict.__getitem__


def reference_config(name):
    c = configs.get_config(name)
    mode = c.pop("training_mode")
    model = _Cfg(type=name, pretrained=None, **{k: _Cfg(v) if isinstance(v, dict) else v for k, v in c.items()})
    out = _Cfg(model=model)
    if mode != "repvgg":            # the reference's P6 / N / S / M configs carry no training_mode (tools/train.py:99-100)
        out["training_mode"] = mode
    return out


@pytest.mark.parametrize("name", NEW)
def test_state_dict_matches_reference_layout(name):
    want = zoo_keys(name)
    for cfg in (name, reference_config(name)):
        m = build_model(cfg, 80, "cpu")
        have = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert have == dict(want)
        m.load_state_dict(fab.fabricate_state_dict(want, seed=0), strict=True)


def test_mbla_branches_follow_the_reference():
    # common.py:657-668 -- n // 2 blocks (at least one), plus the largest power of two below half of that
    assert [arch.mbla_branches(n) for n in (1, 2, 3, 4, 6, 8, 10, 12, 16, 18)] == [
        [0, 1], [0, 1], [0, 1], [0, 1, 2], [0, 2, 3], [0, 2, 4], [0, 4, 5], [0, 4, 6], [0, 4, 8], [0, 8, 9]]


def test_mbla_cv1_is_one_launch_per_contiguous_run_of_concat_slots():
    g = arch.build_graph(configs.get_config("yolov6s_mbla"), 80)
    cv1 = {}
    for op in g.ops:
        if op.name.endswith(".cv1") and op.layout == "cm":
            cv1.setdefault(op.name, []).append(op)
    two = cv1["backbone.ERBlock_2.1.cv1"]               # n = 1: [y0, y1] -> one launch over every row
    assert [(o.w_row0, o.cout, o.dst.c_off) for o in two] == [(0, 2 * 32, 0)]
    three = cv1["backbone.ERBlock_3.1.cv1"]             # n = 4 -> [0, 1, 2]: [y0, y1, b1_1, y2, b2_1, b2_2]
    c = 64
    assert [(o.w_row0, o.cout, o.dst.c_off, o.w_rows) for o in three] == [(0, 2 * c, 0, 3 * c), (2 * c, c, 3 * c, 3 * c)]


def test_unknown_stage_block_type_is_refused():
    cfg = configs.get_config("yolov6s_mbla")
    cfg["backbone"]["stage_block_type"] = "MBLABlok"
    with pytest.raises(ValueError, match="stage_block_type"):
        arch.build_graph(cfg, 80)
    cfg["backbone"]["stage_block_type"] = "BepC3"       # explicit default: the BepC3 network of YOLOv6-M / L
    assert any(op.name.endswith(".m.conv1.conv1") for op in arch.build_graph(cfg, 80).ops)


@pytest.mark.parametrize("name", NEW)
def test_folded_graph_equals_oracle(name):
    size = MODELS[name]
    sd = fab.fabricate_state_dict(zoo_keys(name), 0)
    x = fab.synthetic_images(1, size, size, seed=3)
    g = arch.build_graph(configs.get_config(name), 80)
    with torch.no_grad():
        cls, reg = _run_graph_cpu(g, sd, x)
        ocls, oreg, _ = zoo.forward(sd, zoo.CONFIGS[name], x.double(), train_outputs=True)
    assert float((cls - ocls).abs().max()) < 1e-9
    assert float((reg - oreg).abs().max()) < 1e-8


@pytest.mark.parametrize("name", NEW)
def test_oracle_matches_reference(name):
    g = golden_npz(f"model_{name}.npz")
    sd = fab.fabricate_state_dict(zoo_keys(name), seed=0)
    size = MODELS[name]
    x = fab.synthetic_images(2, size, size, seed=0)
    assert abs(fab.checksum(x) - float(g["x_checksum"])) < 1e-6 * abs(float(g["x_checksum"])), "input RNG drift"
    wsum = sum(fab.checksum(v) for v in sd.values())
    assert abs(wsum - float(g["w_checksum"])) < 1e-6 * abs(float(g["w_checksum"])), "weight RNG drift"
    cfg = zoo.CONFIGS[name]
    with torch.no_grad():
        out = zoo.forward(sd, cfg, x).numpy()
        cls, reg, _ = zoo.forward(sd, cfg, x, train_outputs=True)
        out64 = zoo.forward(sd, cfg, x.double()).numpy()
    assert rel_err(out, g["eval_out"]) < 1e-5
    assert rel_err(cls.numpy(), g["cls_train"]) < 1e-5
    assert rel_err(reg.numpy(), g["reg_train"]) < 1e-5
    assert rel_err(out64, g["eval_out"]) < 1e-5
    assert rel_err(out64, g["deploy_out"]) < 2e-4


@pytest.mark.parametrize("name,batch,size", [("yolov6n6", 2, 128), ("yolov6s_mbla", 2, 64)])
def test_oracle_train_mode_matches_reference(name, batch, size):
    """Train mode (batch-statistics BatchNorm, BottleRep3 alpha, row slices of MBLA's cv1) against the reference in float64."""
    g = golden_npz(f"train_{name}.npz")
    sd = fab.fabricate_state_dict(zoo_keys(name), seed=0)
    for k in sd:
        if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
        if k.endswith(".alpha"):
            sd[k] = sd[k] * 0.75
    x = fab.synthetic_images(batch, size, size, seed=7)
    assert abs(fab.checksum(x) - float(g["x_checksum"])) < 1e-6 * abs(float(g["x_checksum"])), "input RNG drift"
    sd64 = {k: (v.double().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    with zoo.om.train_mode():
        cls, reg, _ = zoo.forward(sd64, zoo.CONFIGS[name], x.double(), train_outputs=True)
    assert rel_err(cls.detach().numpy(), g["cls"]) < 1e-9
    assert rel_err(reg.detach().numpy(), g["reg"]) < 1e-9
    gen = torch.Generator().manual_seed(11)
    wc = torch.randn(cls.shape, generator=gen).double()
    wr = torch.randn(reg.shape, generator=gen).double()
    L = (cls * wc).sum() + (reg * wr).sum()
    assert abs(L.item() - float(g["L"])) < 1e-8 * max(1.0, abs(float(g["L"])))
    L.backward()
    names, norms = [str(n) for n in g["grad_names"]], g["grad_norms"]
    assert len(names) > 300
    for n, ref in zip(names, norms):
        assert sd64[n].grad is not None, n
        got = float(sd64[n].grad.norm())
        assert abs(got - ref) <= 1e-7 * max(1.0, ref), (n, got, ref)
    for k in g.files:
        if k.startswith("grad::"):
            n = k[6:]
            np.testing.assert_allclose(sd64[n].grad.numpy().reshape(g[k].shape), g[k], rtol=1e-7, atol=1e-9 * (1 + np.abs(g[k]).max()))


@pytest.mark.parametrize("name,B,size,step", [("yolov6n6", 1, 1280, 32), ("yolov6s_mbla", 4, 640, 32)])
def test_oracle_matches_reference_at_native_size(name, B, size, step):
    g = golden_npz("configs_zoo.npz")
    sd = fab.fabricate_state_dict(zoo_keys(name), seed=0)
    x = fab.synthetic_images(B, size, size, seed=40)
    assert abs(fab.checksum(x) - float(g[f"{name}_x_checksum"])) < 1e-9 * abs(float(g[f"{name}_x_checksum"])), "input RNG drift"
    with torch.no_grad():
        out = zoo.forward(sd, zoo.CONFIGS[name], x).double().numpy()
    assert rel_err(out[:, ::step], g[f"{name}_rows"].astype(np.float64)) < 1e-5
    A = out.shape[1]
    assert float((np.abs(out.sum(1) - g[f"{name}_colsum"]) / (A + g[f"{name}_abs_colsum"])).max()) < 1e-5


def test_every_built_in_layout_is_unique_and_matched_back_to_its_name():
    layouts = {}
    for name in configs.CONFIGS:
        sd = Model(name).state_dict()
        layouts.setdefault(tuple((k, tuple(v.shape)) for k, v in sd.items()), []).append(name)
        assert _matching_config(sd, 80) == name
    assert all(len(v) == 1 for v in layouts.values()), [v for v in layouts.values() if len(v) > 1]
    for name in NEW:       # the reference's own layout (fabricated tensors) finds its name too
        assert _matching_config(fab.fabricate_state_dict(zoo_keys(name), seed=0), 80) == name


H100 = (132, 232448, 66)


def _plan(d):
    out = (C.c_int32 * 12)()
    rc = _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(ops.PLAN_KEYS, out))


@pytest.mark.parametrize("name", NEW)
def test_every_conv_launch_gets_a_plan_that_fits_the_sm(name):
    """Every conv launch of the bf16 inference forward at the native size (P5 640 bs32, P6 1280 bs8) and at one small size."""
    g = arch.build_graph(configs.get_config(name), 80, name)
    native, small = (1280, 8) if len(g.strides) == 4 else (640, 32), (MODELS[name], 2)
    for size, batch in (native, small):
        convs = [r for r in forward_launches(g, batch, size, size, 1, lambda *key: 1 << 20, _plan) if r.kind == "conv"]
        assert sum(1 for op in g.ops if op.kind in ("conv", "pred", "convT")) <= len(convs) + len(siblings(g))
        for r in convs:
            p = _plan(r.desc)
            assert 0 < p["smem"] <= H100[1] and p["threads"] == 384, (r.name, p)
            assert 1 <= p["grid"] <= H100[0] and p["stages"] >= 2, (r.name, p)
