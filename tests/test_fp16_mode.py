"""The fp16 inference precision mode, checked without a GPU: the launches of an fp16 forward are the bf16 forward's launches
with fp16 dtypes (same kernels, spans, geometry and tile plans), the C ABI's fp16 additions are mirrored in ctypes, and a
folded weight beyond fp16's range is refused by name instead of becoming inf."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from yolov6_b200 import _lib, arch, configs, ops
from yolov6_b200.engine import InferEngine, forward_launches
from yolov6_b200.fold import to_f16
from yolov6_b200.model import build_model
from yolov6_b200.synth import randomize_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100 = (132, 232448, 66)
NAMES = list(configs.CONFIGS)
# the shapes of tests/test_model_lite.py and tests/test_infer_plan.py
SHAPES = ((32, 320, 320), (1, 192, 320), (2, 128, 128), (2, 64, 64))
DTYPE_FIELDS = {"reserved0", "y_dtype"}       # where the fp16 descriptors differ from the bf16 ones


def _plan(d):
    out = (C.c_int32 * 12)()
    rc = _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(ops.PLAN_KEYS, out))


def _fields(d, skip=()):
    return {k: getattr(d, k) for k, _ in d._fields_ if k not in skip}


def _addr(kind, key, q=0):
    """Distinct, 16-byte aligned stand-in addresses, the same for both dtypes."""
    return (hash((kind, str(key), q)) % (1 << 30) + 1) << 8 if kind != "alpha" else 1.0


@pytest.mark.parametrize("name", NAMES)
def test_fp16_launches_are_the_bf16_launches_with_fp16_dtypes(name):
    g = arch.build_graph(configs.get_config(name), 80, name)
    for N, H, W in SHAPES:
        if H % max(g.strides) or W % max(g.strides):
            continue
        for u8 in (False, True):
            a = forward_launches(g, N, H, W, 1, _addr, _plan, u8)
            b = forward_launches(g, N, H, W, 1, _addr, _plan, u8, f16=True)
            assert len(a) == len(b)
            for ra, rb in zip(a, b):
                where = (name, N, H, W, ra.name)
                assert (ra.kind, ra.name, ra.reads, ra.writes, ra.head, ra.conv) == (rb.kind, rb.name, rb.reads, rb.writes, rb.head,
                                                                                      rb.conv), where
                if ra.kind in ("stem", "pool", "dw"):
                    assert rb.fn == ra.fn + "_f16", where
                else:
                    assert rb.fn == ra.fn, where
                if ra.desc is None:
                    assert rb.args == ra.args, where
                    continue
                assert _fields(rb.desc, DTYPE_FIELDS) == _fields(ra.desc, DTYPE_FIELDS), where
                if ra.kind == "conv":
                    assert ra.desc.reserved0 == 0 and rb.desc.reserved0 == _lib.DT_F16, where
                    assert rb.desc.y_dtype == (_lib.DT_F32 if ra.conv["y_f32"] else _lib.DT_F16), where
                    assert ra.desc.y_dtype == (_lib.DT_F32 if ra.conv["y_f32"] else _lib.DT_BF16), where
                    assert _plan(rb.desc) == _plan(ra.desc), where
                elif ra.kind == "se":
                    assert (ra.desc.reserved0, rb.desc.reserved0) == (0, _lib.DT_F16), where
                else:
                    assert _fields(rb.desc) == _fields(ra.desc), where
                if ra.kind == "pool":        # yv6_sppf_pool_f16 takes the packed kernel only: C % 16 == 0, the plane in shared memory
                    _, _, h, w, c = rb.args[:5]
                    assert c % 16 == 0 and 4 * h * w * 32 <= H100[1], where


@pytest.mark.parametrize("case", [dict(Cin=64, Cout=128, k=3, s=1), dict(Cin=32, Cout=64, k=3, s=2), dict(Cin=256, Cout=80, k=1, s=1),
                                  dict(Cin=128, Cout=64, k=3, s=1), dict(Cin=16, Cout=32, k=1, s=1)])
def test_conv_plan_host_is_the_same_for_both_operand_dtypes(case):
    for N, H, W in ((32, 80, 80), (1, 40, 64), (2, 20, 20)):
        for y_f32 in (False, True):
            d16, d = (ops.conv_desc(16, (N, H, W, case["Cin"]), 16, (case["Cout"], case["k"], case["k"], case["Cin"]), 16,
                                    (H * W * case["Cout"], W * case["Cout"], case["Cout"]), stride=case["s"], y_f32=y_f32, f16=f)
                      for f in (True, False))
            assert _plan(d16) == _plan(d)


def test_conv_plan_host_refuses_other_operand_dtypes():
    lib = _lib.lib()
    out = (C.c_int32 * 12)()

    def rc(**kw):
        d = ops.conv_desc(16, (1, 16, 16, 64), 16, (64, 3, 3, 64), 16, (16 * 16 * 64, 16 * 64, 64))
        for k, v in kw.items():
            setattr(d, k, v)
        return lib.yv6_conv_plan_host(*H100, C.byref(d), out)

    assert rc() == 0 and rc(reserved0=_lib.DT_F16, y_dtype=_lib.DT_F16) == 0 and rc(reserved0=_lib.DT_F16, y_dtype=_lib.DT_F32) == 0
    assert rc(reserved0=_lib.DT_F16) == -1                                   # bf16 output from fp16 operands
    assert rc(y_dtype=_lib.DT_F16) == -1                                     # fp16 output from bf16 operands
    assert rc(reserved0=_lib.DT_F16, y_dtype=_lib.DT_F16, nsplit=3) == -1    # fp16 has no split planes
    for bad in (_lib.DT_F32, _lib.DT_U8, 4, -1):
        assert rc(reserved0=bad) == -1


def test_ctypes_mirrors_of_the_fp16_additions_match_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    inc = os.path.join(ROOT, "include")
    src = tmp_path / "f16.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yv6.h"\n'
                   'int main(){printf("%d %zu %zu %zu %zu\\n", (int)YV6_DT_F16, sizeof(yv6_conv_desc), offsetof(yv6_conv_desc, reserved0), '
                   'sizeof(yv6_se_desc), offsetof(yv6_se_desc, reserved0)); return 0;}\n')
    exe = tmp_path / "f16"
    subprocess.run(["gcc", "-I", inc, str(src), "-o", str(exe)], check=True)
    vals = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert vals == [_lib.DT_F16, C.sizeof(_lib.ConvDesc), _lib.ConvDesc.reserved0.offset, C.sizeof(_lib.SeDesc), _lib.SeDesc.reserved0.offset]
    # the fp16 entry points are declared with the argument lists of their bf16 twins
    decl = tmp_path / "decl.c"
    decl.write_text('#include "yv6.h"\n'
                    'int (*a)(yv6_handle*, const yv6_stem_desc*, void*) = yv6_stem_fwd_f16;\n'
                    'int (*b)(yv6_handle*, const yv6_dw_desc*, void*) = yv6_dwconv_fwd_f16;\n'
                    'int (*c)(yv6_handle*, void*, int32_t, int32_t, int32_t, int32_t, int32_t, int32_t, int64_t, void*) = yv6_sppf_pool_f16;\n')
    subprocess.run(["gcc", "-Werror", "-c", "-I", inc, str(decl), "-o", str(tmp_path / "decl.o")], check=True)
    for name in ("yv6_stem_fwd_f16", "yv6_sppf_pool_f16", "yv6_dwconv_fwd_f16"):
        assert name in _lib.exported_symbols()
        assert _lib._SIGNATURES[name] == _lib._SIGNATURES[name[:-4]]


def test_the_library_exports_the_fp16_entry_points():
    lib = _lib.lib()
    for name in ("yv6_stem_fwd_f16", "yv6_sppf_pool_f16", "yv6_dwconv_fwd_f16"):
        assert getattr(lib, name) is not None


def test_set_precision_accepts_fp16_and_still_refuses_other_strings():
    m = build_model("yolov6n", 80, torch.device("cpu"))
    assert m.set_precision("fp16").precision == "fp16"
    for bad in ("half", "FP16", "f16", "int8", "bf16x3"):
        with pytest.raises(AssertionError):
            m.set_precision(bad)
    assert m.set_precision("bf16").precision == "bf16"


def _dry_pack(m, precision):
    eng = InferEngine.__new__(InferEngine)
    eng.g, eng.device, eng.precision, eng.nsplit = m.graph, torch.device("cpu"), precision, 1
    eng.weights = {}
    eng._pack(m.state_dict())
    return eng


def test_fp16_weights_are_the_fp64_fold_rounded_once():
    m = randomize_(build_model("yolov6n", 80, torch.device("cpu")), seed=0).eval()
    e16, e = _dry_pack(m, "fp16"), _dry_pack(m, "bf16")
    assert e16.weights.keys() == e.weights.keys()
    from yolov6_b200.engine import window_weights
    from yolov6_b200.fold import fold_op
    sd = m.state_dict()
    for i, ent in e16.weights.items():
        op = m.graph.ops[i]
        for key in ("w", "w_pair", "w_fused"):
            if key in ent:
                ws = ent[key] if key == "w" else [ent[key]]
                assert all(t.dtype == torch.float16 for t in ws), op.name
                assert [tuple(t.shape) for t in ws] == [tuple(t.shape) for t in (e.weights[i][key] if key == "w" else [e.weights[i][key]])]
        if op.kind == "conv" and "w" in ent and i not in e16.sibling:
            assert torch.equal(ent["w"][0], window_weights(m.graph, op, fold_op(sd, op)[0]).to(torch.float16)), op.name
        for key in ("bias", "w_dev", "b_dev"):
            if key in ent:
                assert torch.equal(ent[key], e.weights[i][key]), op.name


def test_a_folded_weight_beyond_fp16_range_raises_naming_the_layer():
    m = randomize_(build_model("yolov6n", 80, torch.device("cpu")), seed=0).eval()
    sd = m.state_dict()
    layer = next(op for op in m.graph.ops if op.kind == "conv" and op.layout == "rep")
    bn = layer.name + ".rbr_dense.bn"
    sd[bn + ".running_var"][3] = 1e-12        # scale = gamma / sqrt(var + eps): tiny var -> a huge folded weight
    sd[bn + ".weight"][3] = 1e6
    m.load_state_dict(sd)
    with pytest.raises(ValueError, match=layer.name.replace(".", r"\.")):
        _dry_pack(m, "fp16")
    _dry_pack(m, "bf16")                         # bf16 holds it (8 exponent bits)
    with pytest.raises(ValueError, match="stem"):
        to_f16(torch.tensor([7e4], dtype=torch.float64), "backbone.stem")
    assert to_f16(torch.tensor([65504.0, -65504.0], dtype=torch.float64), "x").tolist() == [65504.0, -65504.0]
