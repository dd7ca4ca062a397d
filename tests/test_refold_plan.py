"""CPU checks of the record-driven weight fold (yolov6_b200/refold.py, yv6_fold): the fold records of every built-in detector in
every precision mode, replayed on the host over a seeded train-form state, give byte for byte the host packing the engine used
to do (oracle/pack.py); the seeded states hold -0.0 off-centre 3x3 weights, folded values whose fp64 -> fp16 rounding differs
from a direct conversion, and a BatchNorm that pushes a folded weight beyond fp16's range; the fold's ctypes mirrors match the
header; and is_val_epoch is the reference Trainer's schedule."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle.pack import pack, tensors
from yolov6_b200 import _lib, configs
from yolov6_b200.engine import InferEngine
from yolov6_b200.evaluate import is_val_epoch
from yolov6_b200.fold import fold_op
from yolov6_b200.model import build_model
from yolov6_b200.synth import randomize_

DETECTORS = list(configs.CONFIGS)
MODES = ("bf16", "fp16", "fp32")


def seeded_state(name, seed=0):
    """A randomized CPU model of `name` whose 3x3 weights have -0.0 at some off-centre taps (the +0.0 of the 1x1 branch's
    padding flips them to +0.0 in the fold)."""
    m = randomize_(build_model(name, 80, torch.device("cpu")), seed=seed).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for k, v in m.state_dict().items():
            if v.dim() == 4 and v.shape[2:] == (3, 3):
                mask = torch.rand(v.shape, generator=g) < 0.05
                mask[:, :, 1, 1] = False
                v[mask] = -0.0
    return m


def dry_pack(m, precision, sd=None):
    """InferEngine.weights of a CPU-device engine: the fold records replayed on the host."""
    eng = InferEngine.__new__(InferEngine)
    eng.g, eng.device, eng.precision, eng.nsplit = m.graph, torch.device("cpu"), precision, 3 if precision == "fp32" else 1
    eng.weights = {}
    eng._pack(m.state_dict() if sd is None else sd)
    return eng


def same_bytes(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("name", DETECTORS)
def test_fold_records_replay_the_host_packing_byte_for_byte(name, precision):
    m = seeded_state(name)
    got, want = dry_pack(m, precision).weights, pack(m.graph, m.state_dict(), precision)
    a, b = tensors(got), tensors(want)
    assert [(i, k) for i, k, _ in a] == [(i, k) for i, k, _ in b]
    for (i, k, x), (_, _, y) in zip(a, b):
        assert same_bytes(x, y), f"{m.graph.ops[i].name} {k}"
    assert all(got[i].get("alpha") == want[i].get("alpha") for i in want)


def test_seeded_state_exercises_signed_zeros_and_double_rounding():
    m = seeded_state("yolov6s")
    sd = m.state_dict()
    op = next(op for op in m.graph.ops if op.layout == "rep" and op.kind == "conv")
    w = sd[op.name + ".rbr_dense.conv.weight"]
    assert bool(((w == 0) & torch.signbit(w)).any()), "no -0.0 off-centre weights"
    k, _ = fold_op(sd, op)
    off = k.clone()
    off[:, 1, 1, :] = 1.0
    assert not bool(((off == 0) & torch.signbit(off)).any()), "the fold keeps a -0.0"
    vals = np.concatenate([fold_op(sd, o)[0].numpy().ravel() for o in m.graph.ops if o.kind == "conv" and o.layout in ("rep", "cba")])
    direct, via32 = vals.astype(np.float16), vals.astype(np.float32).astype(np.float16)
    assert int((direct != via32).sum()) > 0, "no folded value whose fp64 -> fp16 rounding depends on the path"
    e16 = dry_pack(m, "fp16").weights          # and the fold takes torch's path (through fp32)
    i = m.graph.ops.index(op)
    assert torch.equal(e16[i]["w"][0], k.to(torch.float16))


@pytest.mark.parametrize("name", ["yolov6n", "yolov6m_qa", "yolov6lite_s"])
def test_fp16_range_error_names_the_first_failing_layer(name):
    m = seeded_state(name)
    sd = m.state_dict()
    convs = [op for op in m.graph.ops if op.kind == "conv" and op.layout in ("rep", "qa", "cba", "dp")]
    layer = convs[len(convs) // 2]
    bn = {"rep": ".rbr_dense.bn", "qa": ".bn", "cba": ".block.bn"}.get(layer.layout)
    if bn is None:
        from yolov6_b200.arch import dp_bn
        bn = dp_bn(layer.name)[len(layer.name):]
    sd[layer.name + bn + ".running_var"][1] = 0.0        # scale = gamma / sqrt(0 + 1e-3)
    sd[layer.name + bn + ".weight"][1] = 5e5
    with pytest.raises(ValueError) as want:
        pack(m.graph, sd, "fp16")
    with pytest.raises(ValueError) as got:
        dry_pack(m, "fp16", sd)
    assert str(got.value) == str(want.value) and str(got.value).startswith(layer.name + ":")
    for precision in ("bf16", "fp32"):
        dry_pack(m, precision, sd)


def test_fold_struct_mirrors_match_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "yv6.h"\nint main(){printf("%zu %zu\\n", sizeof(yv6_fold_chan), sizeof(yv6_fold_rec));'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(_lib.FoldChan), C.sizeof(_lib.FoldRec)]
    assert "yv6_fold" in _lib.exported_symbols()


def reference_condition(epoch, max_epoch, eval_interval, heavy_eval_range, eval_final_only):
    """Trainer.after_epoch, yolov6/core/engine.py:183-185, as written there."""
    remaining_epochs = max_epoch - 1 - epoch
    eval_interval = eval_interval if remaining_epochs >= heavy_eval_range else min(3, eval_interval)
    return (remaining_epochs == 0) or ((not eval_final_only) and ((epoch + 1) % eval_interval == 0))


def test_is_val_epoch_is_the_trainers_schedule():
    n = 0
    for max_epoch in (1, 2, 5, 12, 40, 300):
        for interval in (1, 2, 3, 4, 7, 20):
            for heavy in (0, 1, 3, 10, 50):
                for final_only in (False, True):
                    for epoch in range(max_epoch):
                        assert is_val_epoch(epoch, max_epoch, interval, heavy, final_only) == \
                            reference_condition(epoch, max_epoch, interval, heavy, final_only)
                        n += 1
    assert n > 10000
