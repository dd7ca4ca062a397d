"""The quantization-aware RepVGG networks on the CPU: YOLOv6-N / S / M-QA (configs/qarepvgg, QARepVGGBlockV2) and the v1 block.

Pins oracle/qa.py to the goldens of tests/golden/make_golden_qa.py, the built graphs (state_dict layout, folded deploy weights)
to the oracle, the refused training modes, checkpoint matching, the training engine's parameter order, the conv planner on every
launch and the ctypes mirror of the QA kernels' descriptor."""
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

from conftest import GOLDEN, golden_npz
from oracle import fabricate as fab
from oracle import qa
from test_graph import _run_graph_cpu
from test_model_zoo import H100, _Cfg, _plan
from yolov6_b200 import _lib, arch, configs
from yolov6_b200.checkpoint import _matching_config
from yolov6_b200.engine import conv_launches, siblings
from yolov6_b200.model import build_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["yolov6n_qa", "yolov6s_qa", "yolov6m_qa"]
SIZE = 64


@functools.lru_cache(maxsize=None)
def _layouts():
    with gzip.open(os.path.join(GOLDEN, "keys_qa.json.gz")) as f:
        return json.load(f)


def qa_keys(name):
    """The reference's state_dict layout of `name` (or of yolov6s_qa_v1): [(key, shape)] in the reference's order."""
    return [(k, tuple(shape)) for k, shape in _layouts()[name]]


def rel_err(a, b):
    return float((np.abs(a - b) / (1.0 + np.abs(b))).max())


def reference_config(name, mode="qarepvggv2"):
    """configs/qarepvgg/<name>.py as the reference's Config object: the N / S / M model dict and training_mode."""
    c = configs.get_config(name)
    c.pop("training_mode")
    model = _Cfg(type=name, pretrained=None, **{k: _Cfg(v) if isinstance(v, dict) else v for k, v in c.items()})
    return _Cfg(model=model, training_mode=mode)


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_reference_layout_in_order(name):
    want = qa_keys(name)
    for cfg in (name, reference_config(name)):
        m = build_model(cfg, 80, "cpu")
        _assert_layout(m, want)
        m.load_state_dict(fab.fabricate_state_dict(want, seed=0), strict=True)


def _assert_layout(m, want):
    """Same keys and shapes, and inside every QA block the reference's key order (rbr_dense.conv, rbr_dense.bn, rbr_1x1, bn)."""
    have = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert dict(have) == dict(want)
    blocks = [op.name for op in m.graph.ops if op.layout == "qa"]
    assert len(blocks) > 20
    for b in blocks:
        mine = [k for k, _ in have if k.startswith(b + ".")]
        assert mine == [k for k, _ in want if k.startswith(b + ".")]
        assert len(mine) == 12 and mine[:2] == [b + ".rbr_dense.conv.weight", b + ".rbr_dense.bn.weight"]
        assert mine[6:8] == [b + ".rbr_1x1.weight", b + ".bn.weight"]


def test_v1_layout_matches_reference():
    m = build_model(reference_config("yolov6s_qa", "qarepvgg"), 80, "cpu")
    _assert_layout(m, qa_keys("yolov6s_qa_v1"))
    g = m.graph
    assert not any(op.avg for op in g.ops) and sum(op.identity for op in g.ops if op.layout == "qa") > 10


def test_qa_parameters_land_in_the_optimizer_groups():
    """flat.py assigns build_optimizer's groups from the module types: the post-sum bn weight is a BatchNorm weight, the bare
    rbr_1x1 weight a conv weight."""
    import torch.nn as nn
    m = build_model("yolov6s_qa", 80, "cpu")
    mods = dict(m.named_modules())
    p = "backbone.ERBlock_3.1.conv1"
    assert isinstance(mods[p + ".bn"], nn.BatchNorm2d) and isinstance(mods[p + ".rbr_1x1"], nn.Conv2d)
    assert isinstance(mods[p + ".rbr_dense.bn"], nn.BatchNorm2d) and mods[p + ".rbr_1x1"].bias is None
    stem = [op for op in m.graph.ops if op.kind == "stem"][0]
    assert stem.layout == "qa" and not stem.identity and not stem.avg


@pytest.mark.parametrize("mode", ["hyper_search", "repopt", "qarepvgg3"])
def test_unsupported_training_modes_are_refused(mode):
    cfg = configs.get_config("yolov6s")
    cfg["training_mode"] = mode
    with pytest.raises(ValueError, match="training_mode"):
        arch.build_graph(cfg, 80)
    with pytest.raises(ValueError, match="qarepvggv2"):
        build_model(reference_config("yolov6s_qa", mode), 80, "cpu")


@pytest.mark.parametrize("name", NAMES + ["yolov6s_qa_v1"])
def test_folded_graph_equals_oracle(name):
    v1 = name.endswith("_v1")
    mode = "qarepvgg" if v1 else "qarepvggv2"
    cfg = configs.get_config(name.replace("_v1", ""))
    cfg["training_mode"] = mode
    sd = fab.fabricate_state_dict(qa_keys(name), 0)
    x = fab.synthetic_images(1, SIZE, SIZE, seed=3)
    g = arch.build_graph(cfg, 80)
    assert sum(op.avg for op in g.ops) == (0 if v1 else sum(op.identity for op in g.ops))
    with torch.no_grad():
        cls, reg = _run_graph_cpu(g, sd, x)
        ocls, oreg, _ = qa.forward(sd, dict(qa.CONFIGS[name.replace("_v1", "")], mode=mode), x.double(), train_outputs=True)
    assert float((cls - ocls).abs().max()) < 1e-9
    assert float((reg - oreg).abs().max()) < 1e-9 * (1 + float(oreg.abs().max()))


@pytest.mark.parametrize("name", NAMES + ["yolov6s_qa_v1"])
def test_oracle_matches_reference(name):
    g = golden_npz(f"model_{name}.npz")
    sd = fab.fabricate_state_dict(qa_keys(name), seed=0)
    x = fab.synthetic_images(2, SIZE, SIZE, seed=0)
    assert abs(fab.checksum(x) - float(g["x_checksum"])) < 1e-6 * abs(float(g["x_checksum"])), "input RNG drift"
    wsum = sum(fab.checksum(v) for v in sd.values())
    assert abs(wsum - float(g["w_checksum"])) < 1e-6 * abs(float(g["w_checksum"])), "weight RNG drift"
    cfg = qa.CONFIGS[name.replace("_v1", "")]
    if name.endswith("_v1"):
        cfg = dict(cfg, mode="qarepvgg")
    with torch.no_grad():
        out = qa.forward(sd, cfg, x).numpy()
        out64 = qa.forward(sd, cfg, x.double()).numpy()
        assert rel_err(out, g["eval_out"]) < 1e-5
        assert rel_err(out64, g["eval_out"]) < 1e-5
        if "deploy_out" in g.files:
            cls, reg, _ = qa.forward(sd, cfg, x, train_outputs=True)
            assert rel_err(cls.numpy(), g["cls_train"]) < 1e-5
            assert rel_err(reg.numpy(), g["reg_train"]) < 1e-5
            assert rel_err(out64, g["deploy_out"]) < 2e-4


def train_sd(name):
    sd = fab.fabricate_state_dict(qa_keys(name), seed=0)
    for k in sd:      # keep the head logits O(1) under batch-statistics BN
        if (".cls_preds." in k or ".reg_preds." in k) and k.endswith("weight"):
            sd[k] = sd[k] * 0.1
        if k.endswith(".alpha"):
            sd[k] = sd[k] * 0.75
    return sd


@pytest.mark.parametrize("name,batch,size", [("yolov6n_qa", 2, 64), ("yolov6m_qa", 2, 64)])
def test_oracle_train_mode_matches_reference(name, batch, size):
    """Train mode (batch statistics in both BatchNorms of every block, BottleRep alpha) against the reference in float64."""
    g = golden_npz(f"train_{name}.npz")
    sd = train_sd(name)
    x = fab.synthetic_images(batch, size, size, seed=7)
    assert abs(fab.checksum(x) - float(g["x_checksum"])) < 1e-6 * abs(float(g["x_checksum"])), "input RNG drift"
    sd64 = {k: (v.double().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    with qa.om.train_mode():
        cls, reg, _ = qa.forward(sd64, qa.CONFIGS[name], x.double(), train_outputs=True)
    assert rel_err(cls.detach().numpy(), g["cls"]) < 1e-9
    assert rel_err(reg.detach().numpy(), g["reg"]) < 1e-9
    gen = torch.Generator().manual_seed(11)
    wc = torch.randn(cls.shape, generator=gen).double()
    wr = torch.randn(reg.shape, generator=gen).double()
    L = (cls * wc).sum() + (reg * wr).sum()
    assert abs(L.item() - float(g["L"])) < 1e-8 * max(1.0, abs(float(g["L"])))
    L.backward()
    names, norms = [str(n) for n in g["grad_names"]], g["grad_norms"]
    assert len(names) > 300 and any(n.endswith(".rbr_1x1.weight") for n in names)
    for n, ref in zip(names, norms):
        assert sd64[n].grad is not None, n
        got = float(sd64[n].grad.norm())
        assert abs(got - ref) <= 1e-7 * max(1.0, ref), (n, got, ref)
    full = [k for k in g.files if k.startswith("grad::")]
    assert len(full) >= 6
    for k in full:
        n = k[6:]
        np.testing.assert_allclose(sd64[n].grad.numpy().reshape(g[k].shape), g[k], rtol=1e-7, atol=1e-9 * (1 + np.abs(g[k]).max()))


def test_matching_config_finds_each_qa_name_from_the_reference_layout():
    for name in NAMES:
        assert _matching_config(fab.fabricate_state_dict(qa_keys(name), seed=0), 80) == name


def test_ctypes_mirror_of_the_qa_descriptor_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yv6.h"\n'
                   'int main(){printf("%zu %zu %zu\\n", sizeof(yv6_qa_desc), offsetof(yv6_qa_desc, momentum), offsetof(yv6_qa_desc, dx));'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.QaDesc), _lib.QaDesc.momentum.offset, _lib.QaDesc.dx.offset]


def test_qa_ops_train_with_both_batchnorms_and_the_bare_1x1():
    """The training engine's parameter order of a QA block: both conv weights, BN_d, the post-sum bn (and alpha)."""
    from yolov6_b200.train import op_param_names
    g = arch.build_graph(configs.get_config("yolov6m_qa"), 80)
    op = next(o for o in g.ops if o.layout == "qa" and o.alpha)
    p = op.name
    assert op_param_names(op) == [p + ".rbr_dense.conv.weight", p + ".rbr_dense.bn.weight", p + ".rbr_dense.bn.bias",
                                  p + ".rbr_1x1.weight", p + ".bn.weight", p + ".bn.bias", op.alpha]
    m = build_model("yolov6m_qa", 80, "cpu")
    trainable = {k for k, v in m.named_parameters() if v.requires_grad}
    assert trainable == {n for o in g.ops for n in op_param_names(o)}


def _descs(name, N, S):
    g = arch.build_graph(configs.get_config(name), 80, name)
    launches = conv_launches(g, N, S, S, 1, siblings(g), lambda *key: 1 << 20, _plan)
    return g, [(g.ops[i].kind, bytes(d)) for i in sorted(launches) for d in launches[i]]


@pytest.mark.parametrize("base", ["yolov6n", "yolov6s", "yolov6m"])
def test_folded_inference_graph_is_the_float_models_graph(base):
    """Folded, a QA block is the 3x3 conv + bias + ReLU of the float model's RepVGG block: same ops, same conv launches."""
    for N, S in ((32, 640), (2, SIZE)):
        gq, dq = _descs(base + "_qa", N, S)
        gf, df = _descs(base, N, S)
        assert [(o.kind, o.name, o.src, o.dst, o.k, o.s, o.act, o.res, o.alpha) for o in gq.ops] == \
               [(o.kind, o.name, o.src, o.dst, o.k, o.s, o.act, o.res, o.alpha) for o in gf.ops]
        assert dq == df


@pytest.mark.parametrize("name", NAMES)
def test_every_conv_launch_gets_a_plan_that_fits_the_sm(name):
    g = arch.build_graph(configs.get_config(name), 80, name)
    for size, batch in ((640, 32), (SIZE, 2)):
        launches = conv_launches(g, batch, size, size, 1, siblings(g), lambda *key: 1 << 20, _plan)
        assert sum(1 for op in g.ops if op.kind in ("conv", "pred", "convT")) <= sum(len(v) for v in launches.values()) + len(siblings(g))
        for i, ds in launches.items():
            for d in ds:
                p = _plan(d)
                assert 0 < p["smem"] <= H100[1] and p["threads"] == 384, (g.ops[i].name, p)
                assert 1 <= p["grid"] <= H100[0] and p["stages"] >= 2, (g.ops[i].name, p)
