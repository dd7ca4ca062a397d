"""CPU checks of the per-launch forward test (tests/test_gpu_forward_launches.py).

Coverage: the host planner (yv6_conv_plan_host at the H100 SXM's properties, as in tests/test_infer_plan.py) plans the launch
records of every configuration of the GPU test without a GPU.  Together they must produce every InferLaunch kind, both decode
forms (plain ltrb and DFL), every conv form (plain, residual, fused cls / reg siblings, transposed-conv quadrant scatter, fp32
head pred, column-pair view), halo modes 0, 1 and 2, halo plans with resident and with streamed weights, and bf16 and fp32
outputs.  A planner change that stops the GPU test from reaching one of them fails here.  The planner takes CTA pairs only
when a descriptor forces them (force_pair); no engine launch does, so every plan is single-CTA and this is asserted too: a
change that lets the engine take pairs must bring them under the GPU test's coverage list.

Harness: the GPU test's comparison helpers fail on a reference that lost one tap of one border pixel, and on an output
buffer with one element outside the written view changed -- the per-launch checks do not compare a buffer with itself."""
import pytest
import torch

import test_gpu_backward_launches as bwd
import test_gpu_forward_launches as fwd
from test_infer_plan import host_plan
from yolov6_b200 import _lib, configs
from yolov6_b200.engine import forward_launches
from yolov6_b200.model import build_model


def fake_addr():
    """Distinct 4 GB-aligned stand-in addresses for every tensor forward_launches asks for (alpha: 1.0)."""
    table = {}

    def addr(kind, key, q=0):
        if kind == "alpha":
            return 1.0
        return table.setdefault((kind, key, q), (len(table) + 1) << 32)
    return addr


def records(c):
    cfg = configs.get_config(c["cfg"])
    g = build_model(cfg, 80, torch.device("cpu")).graph
    nsplit = 3 if c.get("precision") == "fp32" else 1
    return g, forward_launches(g, c["N"], c["H"], c["W"], nsplit, fake_addr(), host_plan, c.get("u8", False))


def test_forward_launch_configs_reach_every_launch_kind_and_conv_mode():
    kinds, forms, decode = set(), set(), set()
    halo, resident, pair, f32_out = set(), set(), set(), set()
    for c in fwd.CONFIGS.values():
        g, recs = records(c)
        decode.add("dfl" if g.use_dfl and g.reg_max else "ltrb")
        for r in recs:
            kinds.add(r.kind)
            if r.kind != "conv":
                continue
            forms.add(fwd.conv_form(r))
            p = host_plan(r.desc)
            halo.add(p["halo"])
            if p["halo"]:
                resident.add(p["a_res"] % 10)
            pair.add(p["a_res"] // 10 % 10)
            f32_out.add(r.desc.y_dtype == _lib.DT_F32)
    assert kinds == {"stem", "conv", "pool", "dw", "se", "shuffle", "up"}, kinds
    assert decode == {"ltrb", "dfl"}, decode
    assert forms == {"plain", "residual", "fused", "convT", "pred", "pair_view"}, forms
    assert halo == {0, 1, 2}, halo
    assert resident == {0, 1}, resident
    assert pair == {0}, f"the engine now takes CTA pairs ({pair}): add them to the GPU test's coverage"
    assert f32_out == {False, True}, f32_out


def test_forward_launch_checks_catch_a_dropped_tap_and_a_stray_write():
    gen = torch.Generator().manual_seed(3)
    N, H, W, Cin, Cout = 2, 9, 11, 16, 8
    x = torch.randn(N, H, W, Cin, generator=gen).to(torch.bfloat16)
    w = torch.randn(Cout, 3, 3, Cin, generator=gen).to(torch.bfloat16) / 8
    b = torch.randn(Cout, generator=gen)
    ref, R, z = fwd.conv_ref(x, w, b, 1, 1, fwd.ACT_SILU)
    got = ref.to(torch.bfloat16)                   # a correct kernel: the exact value, rounded once
    bar = fwd.out_bar(ref, R, z, fwd.ACT_SILU, bf16_out=True, planes3=False, fast_silu=True)
    assert bwd.ratio(got, ref, bar) <= 1.0
    # drop the tap (r, s) = (1, 0) -- the left neighbour -- of the right border pixel (0, 4, W - 1)
    bad = ref.clone()
    zz = z[0, 4, W - 1] - (x[0, 4, W - 2].double() * w[:, 1, 0].double()).sum(-1)
    bad[0, 4, W - 1] = fwd.act64(zz, fwd.ACT_SILU)
    assert bwd.ratio(got, bad, bar) > 1.0, "a reference without one border tap passes the bar"
    # check_launch's post-run sequence (settle) on a stand-in launch: input slice [0, Cin) of one buffer, output slice
    # [8, 8 + Cout) of another, everything else the sentinel.  A clean launch settles; one stray element is caught.
    def launch(stray):
        tensors = {("buf", 0): torch.full((N, H, W, 32), fwd.SENTINEL, dtype=torch.bfloat16),
                   ("buf", 1): torch.full((N, H, W, 32), fwd.SENTINEL, dtype=torch.bfloat16)}
        xin, out = tensors[("buf", 0)][..., :Cin], tensors[("buf", 1)][..., 8:8 + Cout]
        xin.copy_(x)
        snap = [(xin, xin.clone())]
        out.copy_(got)                                 # what the kernel computes
        if stray:
            tensors[("buf", 1)][1, H - 1, 0, 8 + Cout] = 0.5
        fwd.settle(tensors, [out], [xin], snap, "stand-in launch")

    launch(False)
    with pytest.raises(AssertionError, match="wrote outside"):
        launch(True)
