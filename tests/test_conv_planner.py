"""CPU checks of the conv tile planner (`plan_conv` of yolov6_b200/csrc/yv6_conv_igemm.cu) through the host-only C-ABI entry
`yv6_conv_plan_host`, with the H100 SXM's device properties stated explicitly (132 SMs, 232448 bytes of opt-in shared memory, 66
co-resident CTA pairs):
every conv launch the inference engine makes (engine.conv_launches: fused head siblings, column-pair views) for every supported
model (reference configs/yolov6{n,s,m}.py, yolov6l6.py) at the BASELINE.json configurations gets a plan that fits the SM, and the
YOLOv6-S plans of the benchmark configuration are pinned.  No compute, no GPU."""
import ctypes as C

import pytest

from yolov6_b200 import _lib, ops
from yolov6_b200.arch import build_graph
from yolov6_b200.configs import get_config
from yolov6_b200.engine import conv_launches, siblings

H100 = (132, 232448, 66)


def plan(d):
    out = (C.c_int32 * 12)()
    rc = _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(ops.PLAN_KEYS, out))


def layer_descs(name, batch, size):
    """(op name, descriptor) of every conv launch of the bf16 inference engine's forward, at fake 16-byte-aligned addresses."""
    g = build_graph(get_config(name), 80, name)
    launches = conv_launches(g, batch, size, size, 1, siblings(g), lambda *key: 1 << 20, plan)
    return [(g.ops[i].name, d) for i, ds in launches.items() for d in ds]


@pytest.mark.parametrize("name,batch,size", [("yolov6n", 32, 640), ("yolov6s", 32, 640), ("yolov6s", 1, 64), ("yolov6m", 8, 640),
                                             ("yolov6m", 64, 640), ("yolov6l6", 2, 1280), ("yolov6l6", 16, 1280), ("yolov6l6", 1, 128),
                                             ("yolov6s", 4, 416), ("yolov6n", 2, 96)])
def test_every_layer_of_every_model_gets_a_plan_that_fits_the_sm(name, batch, size):
    descs = layer_descs(name, batch, size)
    for lname, d in descs:
        p = plan(d)              # asserts rc == 0: no YV6_REQUIRE of the planner fires, shared memory fits
        assert 0 < p["smem"] <= H100[1] and p["threads"] == 384, (lname, p)
        assert p["BW"] * p["BH"] * p["BI"] <= 128 and p["BN"] in (32, 64, 96, 128), (lname, p)
        assert 1 <= p["grid"] <= H100[0] and p["stages"] >= 2, (lname, p)
        if p["a_res"] // 10 % 10:                               # CTA pairs: an even grid of at most 66 clusters
            assert p["grid"] % 2 == 0 and p["grid"] <= 2 * H100[2], (lname, p)
    # conv launches per forward: the head's cls / reg 3x3 convs run as one launch wherever Cout % 64 == 0
    assert len(descs) == {"yolov6n": 74, "yolov6s": 73, "yolov6m": 111, "yolov6l6": 206}[name]


def test_yolov6s_bench_plans():
    """The plans of the benchmark configuration on the H100: stride-2 halo mainloop on six of the eight 3x3 stride-2 layers,
    the stride-1 halo mainloop on the 3x3 layers, resident weights for the 64-channel layers, the plain mainloop elsewhere; no CTA
    pairs in auto mode."""
    descs = layer_descs("yolov6s", 32, 640)
    got = {}
    for ln, d in descs:
        got.setdefault(ln, plan(d))
    assert {ln for ln, d in descs if d.pair_view} == {"backbone.ERBlock_2.0", "backbone.ERBlock_3.0", "backbone.ERBlock_4.0",
                                                       "neck.Bifusion0.downsample", "neck.Bifusion1.downsample", "neck.downsample2"}
    want = {   # name: (BW, BH, BN, stages, halo, a_res)
        "backbone.ERBlock_2.0": (8, 16, 64, 6, 2, 301), "backbone.ERBlock_3.0": (8, 16, 128, 5, 2, 200),
        "backbone.ERBlock_4.0": (8, 16, 128, 5, 2, 200), "backbone.ERBlock_5.0": (20, 5, 128, 4, 0, 0),
        "neck.Bifusion0.downsample": (8, 16, 128, 5, 2, 200), "neck.Bifusion1.downsample": (8, 16, 64, 9, 2, 301),
        "neck.downsample2": (8, 16, 64, 9, 2, 301), "neck.downsample1": (20, 5, 128, 4, 0, 0),
        "backbone.ERBlock_2.1.conv1": (8, 16, 64, 9, 1, 501), "backbone.ERBlock_3.1.conv1": (8, 16, 128, 5, 1, 300),
        "backbone.ERBlock_4.1.conv1": (8, 16, 128, 5, 1, 300), "neck.Bifusion1.cv2": (32, 4, 64, 7, 0, 0),
    }
    for ln, w in want.items():
        p = got[ln]
        assert (p["BW"], p["BH"], p["BN"], p["stages"], p["halo"], p["a_res"]) == w, (ln, p)
    # forced CTA pairs: same tiles, an even grid of at most 66 clusters
    for ln, d in descs:
        if ln == "backbone.ERBlock_3.1.conv1":
            d.force_pair = 1
            p = plan(d)
            assert (p["BN"], p["halo"], p["a_res"], p["grid"]) == (128, 1, 310, 132), p
            break


def test_planner_rejects_what_the_kernel_cannot_run():
    d = _lib.ConvDesc()
    d.x = d.w = d.y = 4096
    d.N, d.H, d.W, d.Cin, d.x_c_total, d.Cout, d.kh, d.kw, d.stride, d.pad, d.nsplit = 1, 8, 8, 24, 24, 16, 1, 1, 1, 0, 1
    d.pad_w = _lib.PAD_SAME
    out = (C.c_int32 * 12)()
    assert _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out) != 0          # Cin must be a multiple of 16
    assert b"Cin" in _lib.lib().yv6_last_error()
    d.Cin = d.x_c_total = 32
    d.kh = 5
    assert _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out) != 0          # kernel sizes 1..3 only

