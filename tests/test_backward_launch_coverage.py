"""CPU checks of the per-launch backward test (tests/test_gpu_backward_launches.py).

Coverage: the training engine of every configuration of the GPU test is planned on the CPU (tests/test_train_plan.py's
stand-ins for the library, streams and events) at the GPU test's batch and image size, and the weight-gradient launches are
planned by yv6_wgrad_plan_host at the H100 SXM's properties (132 SMs, 232448 bytes of opt-in shared memory).  Together the
configurations must reach every backward launch kind, every wgrad tile form (Cin tile NT 16 / 32 / 64 / 128, one tap or a
filter row of three taps per CTA), a split-K with more than 2^13 pixels summed in fp32 per split (the regime in which only
exact integer operands can tell a lost split from rounding), bn_bwd with one, two and three branches with and without a
shortcut, and the four-parity dgrad of a 3x3 stride-2 conv.  A planner change that stops the GPU test from reaching one of
them fails here.

The N / S self-distillation student must reach the backward of its reg_preds_dist pred conv at every level: the head-gradient
repack of the 68 DFL channels (no scores, padded to 80), the weight gradient, the bias sums and a dgrad that accumulates into
the reg-feature gradient slice the lrtb pred's dgrad assigned.  With external neck-output gradients (the channel-wise
distillation term injects them before the backward's first launch) no Write record that overlaps a neck-output slice may
resolve to assign: an assigning launch would overwrite the injected gradient and drop the whole term.  Checked on every
configuration of the GPU test that sets the flag and on N, S, M and L6 at the GPU test's shapes.

Harness: the GPU test's exact comparison fails on a weight gradient that lost one split's partial sum, its engine-memory
check fails on one stray element, and its check of a first (assigning) writer fails on a `full` write that missed a pixel;
the neck-slice check fails on a hand-built plan whose neck slice has an assigning first writer."""
import ctypes as C
import types

import pytest
import torch

import test_gpu_backward_launches as bwd
from test_train_plan import dry_engine_of
from yolov6_b200 import _lib
from yolov6_b200.train import TrainEngine, Write

H100 = (132, 232448)
WGRAD_KEYS = ("NT", "T", "PT", "BW", "BH", "ptiles", "ksplit", "split_pixels", "ctas", "smem")


def wgrad_plan(d):
    out = (C.c_int32 * 10)()
    rc = _lib.lib().yv6_wgrad_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(WGRAD_KEYS, out))


def first_writer_decisions(eng):
    """[(Write record, True when it assigns)] as the first-writer resolution (train.py) decides them for eng's plan, recorded by
    running the resolution again with each record's callback wrapped (the same decisions again: the plan is unchanged)."""
    log, saved = [], []
    for c in eng.bwd_calls:
        for w in c.writes:
            saved.append((w, w.assign))
            w.assign = lambda a, w=w, f=w.assign: (log.append((w, bool(a))), f(a))
    try:
        TrainEngine._resolve_first_writers(eng)
    finally:
        for w, f in saved:
            w.assign = f
    return log


def assert_neck_slices_accumulate(eng, what):
    """With external neck-output gradients every Write record that overlaps a neck-output slice accumulates, and every neck
    slice has a writer (the gradient flows on into the neck)."""
    feat = [(t.buf, t.c_off, t.c_off + t.c) for t in eng.g.feat]
    decisions = first_writer_decisions(eng)
    hits = [(w, a) for w, a in decisions if any(w.buf == b and w.off < hi and lo < w.off + w.n for b, lo, hi in feat)]
    bad = [(w.buf, w.off, w.n) for w, a in hits if a]
    assert not bad, f"{what}: Write records (buffer, channel, count) that assign into a neck-output gradient slice: {bad}"
    for b, lo, hi in feat:
        assert any(w.buf == b and w.off < hi and lo < w.off + w.n for w, _ in hits), f"{what}: neck slice {(b, lo, hi)} has no writer"
    return len(hits)


def dry_planned(cfg, batch, size, u8=False, **kw):
    eng, _ = dry_engine_of(cfg, 1, **kw)
    eng._plan(batch, size, size, torch.uint8 if u8 else torch.float32)
    return eng


@pytest.fixture(scope="module")
def plans():
    out = {}
    for name, c in bwd.MODELS.items():
        eng = dry_planned(c["cfg"], c["batch"], c["size"], c.get("u8"), fuse_ab=c.get("fuse_ab", False),
                          distill_ns=c.get("distill_ns", False), external_feat_grads=bool(c.get("feat")))
        out[name] = eng.bwd_calls
        if eng.external_feat_grads:
            FEAT_CHECKED[name] = assert_neck_slices_accumulate(eng, name)
        if eng.g.distill_ns:
            REG_DIST[name] = reg_dist_backward(eng)
        del eng
    return out


FEAT_CHECKED, REG_DIST = {}, {}


def reg_dist_backward(eng):
    """Per level, the backward launches of the reg_preds_dist pred conv and the dgrad of the lrtb pred next to it."""
    g, out = eng.g, []
    ch = 4 * 17
    decisions = {id(w): a for w, a in first_writer_decisions(eng)}
    hgp = [j for j, c in enumerate(eng.bwd_calls) if c.kind == "hgp" and c.args[4] == ch]
    for j in hgp:
        seq = eng.bwd_calls[j:j + 4]
        lrtb = [c for c in eng.bwd_calls[:j] if c.kind == "conv" and c.writes and c.writes[0].buf == seq[3].writes[0].buf
                and c.writes[0].off == seq[3].writes[0].off]
        out.append(types.SimpleNamespace(seq=seq, lrtb=lrtb, assigns=[decisions[id(c.writes[0])] for c in lrtb + [seq[3]]]))
    assert len(out) == len(g.strides), f"{len(out)} reg_preds_dist head-gradient repacks for {len(g.strides)} levels"
    return out


def test_backward_launch_configs_reach_every_kind_and_form(plans):
    kinds, nt, taps, bn_forms, parity_groups = set(), set(), set(), set(), 0
    long_split = []
    for name, calls in plans.items():
        groups = {}
        for c in calls:
            kinds.add(c.kind)
            if c.kind == "wgrad":
                p = wgrad_plan(c.desc)
                nt.add(p["NT"])
                taps.add(p["T"])
                if p["ksplit"] > 1 and p["split_pixels"] > 2 ** 13:
                    long_split.append((name, p["ksplit"], p["split_pixels"]))
                assert bwd.exact_k_bound(p["ptiles"] * p["PT"], 2, 2), f"{name}: wgrad sum too long for exact operands"
            elif c.kind == "bn_bwd":
                bn_forms.add((c.desc.nb, bool(c.desc.res)))
            elif c.kind == "conv" and c.writes[0].group is not None:
                groups.setdefault(c.writes[0].group, []).append(c.desc)
        parity_groups += sum(1 for ds in groups.values() if len(ds) == 4)
    want = {"conv", "wgrad", "bn_bwd", "stats", "hgp", "pool_bwd", "im2col", "qa_bwd", "abg", "copy", "bucket"}
    assert kinds == want, f"backward kinds reached: {sorted(kinds)}, want {sorted(want)}"
    assert set(bwd.KINDS) == want - {"copy", "bucket"}, "the GPU test's kinds"
    assert nt == {16, 32, 64, 128}, nt
    assert taps == {1, 3}, taps
    assert long_split, "no weight gradient is split over more than 2^13 pixels per split"
    # (nb, shortcut): none of the planned models has a two-branch block with a shortcut
    assert {(1, False), (1, True), (2, False), (3, False), (3, True)} <= bn_forms, sorted(bn_forms)
    assert parity_groups, "no stride-2 3x3 dgrad in four parity launches"


def test_wgrad_host_plan_splits_the_benchmarked_stem():
    """YOLOv6-S at 640, batch 32: the stem's 1x1 weight gradient over the im2col patches (3.28 M pixels, Cout 32, N 32)."""
    d = _lib.WgradDesc()
    d.N, d.H, d.W, d.Cin, d.x_c_total, d.Cout, d.dy_c_total = 32, 320, 320, 32, 32, 32, 32
    d.kh = d.kw = d.stride = 1
    p = wgrad_plan(d)
    assert (p["NT"], p["T"], p["PT"]) == (32, 1, 128)
    assert p["ksplit"] == 264 and p["split_pixels"] == 12416 and p["ctas"] == 264, p
    d.force_ksplit = 3
    assert wgrad_plan(d)["ksplit"] == 3
    d.kh = d.kw = 5
    out = (C.c_int32 * 10)()
    assert _lib.lib().yv6_wgrad_plan_host(*H100, C.byref(d), out) != 0
    assert b"kernel" in _lib.lib().yv6_last_error()


def test_exact_comparison_catches_a_lost_split():
    """Integer operands: a weight gradient summed in fp32 split by split equals float64 exactly; without one split it does not."""
    gen = torch.Generator().manual_seed(5)
    N, H, W, Cin, Cout, ksplit = 2, 12, 10, 16, 8, 5
    x = torch.randint(-2, 3, (N, H, W, Cin), generator=gen).to(torch.bfloat16)
    dy = torch.randint(-2, 3, (N, H, W, Cout), generator=gen).to(torch.bfloat16)
    prior = torch.randint(-2, 3, (Cout, 3, 3, Cin), generator=gen).float()
    ref, _ = bwd.wgrad_ref(x, dy, Cout, 3, 1, 1)
    rows = torch.arange(N * H).chunk(ksplit)

    def split_sum(skip):
        got = prior.clone()
        for j, r in enumerate(rows):
            if j == skip:
                continue
            xm, dm = x.reshape(N * H, 1, W, Cin).clone(), dy.reshape(N * H, 1, W, Cout).clone()
            keep = torch.zeros(N * H, dtype=torch.bool)
            keep[r] = True
            dm[~keep] = 0                          # the split's output rows only; the taps still see the whole input
            got += bwd.wgrad_ref(x, dm.reshape(N, H, W, Cout), Cout, 3, 1, 1)[0].float()
        return got

    bwd.assert_exact(split_sum(None), (prior.double() + ref).float(), "wgrad")
    with pytest.raises(AssertionError, match="not exact"):
        bwd.assert_exact(split_sum(2), (prior.double() + ref).float(), "wgrad")


def test_write_checks_catch_a_stray_element_and_a_missed_pixel():
    """The engine-memory check (settle) on stand-in tensors, and the check that an assigning full write left no sentinel."""
    g = torch.full((2, 5, 6, 24), bwd.SENTINEL, dtype=torch.bfloat16)
    scratch = torch.full((64,), bwd.SENTINEL, dtype=torch.float32)
    arena = torch.zeros(256, dtype=torch.uint8)
    mem = bwd.Mem([("gbuf", g), ("poolscr", scratch), ("arena", arena)])

    def launch(stray, miss):
        g.fill_(bwd.SENTINEL)
        out = g[..., 8:16]
        out.copy_(torch.randn(out.shape).to(torch.bfloat16))
        if miss:
            out[1, 4, 5, 3] = bwd.SENTINEL
        if stray:
            g[0, 2, 3, 16] = 1.0
        bwd.assert_full_write(out, "stand-in dgrad")
        bwd.settle(mem, [], [out], "stand-in dgrad")

    launch(False, False)
    with pytest.raises(AssertionError, match="outside"):
        launch(True, False)
    with pytest.raises(AssertionError, match="not every pixel"):
        launch(False, True)


def test_distill_ns_student_reaches_the_reg_dist_backward(plans):
    """Each level's reg_preds_dist pred: the head-gradient repack without scores (68 -> 80 channels), its weight gradient
    (Cout 68), the bias sums over the 80 padded channels and a dgrad that accumulates (a residual read) into the slice the lrtb
    pred's dgrad assigned -- the first writer in backward order, as the lrtb pred comes after reg_preds_dist in the forward."""
    name = "yolov6s_640_b32_u8_distill_ns"
    assert name in plans and REG_DIST[name]
    for lv in REG_DIST[name]:
        hgp, wg, st, dg = lv.seq
        assert [c.kind for c in lv.seq] == ["hgp", "wgrad", "stats", "conv"], [c.kind for c in lv.seq]
        assert hgp.args[1] == 0 and hgp.args[4] == 68 and hgp.args[7] == 80, hgp.args
        assert wg.desc.Cout == 68 and wg.side
        assert st.desc.C == 80
        assert dg.desc.Cin == 80 and dg.desc.Cout == dg.writes[0].n
        assert len(lv.lrtb) == 1, "the lrtb pred's dgrad into the same reg-feature slice"
        assert lv.assigns == [True, False], f"first writer assigns, reg_dist dgrad accumulates: {lv.assigns}"
        assert not lv.lrtb[0].desc.res and dg.desc.res, "the reg_dist dgrad must read the slice it accumulates into"


def test_external_feat_grads_plans_accumulate_into_every_neck_slice(plans):
    """The GPU test's configuration with the flag, and N, S, M and L6 at the GPU test's shapes: no assigning write overlaps a
    neck-output gradient slice."""
    assert "yolov6m_96_b2_feat" in plans and FEAT_CHECKED.get("yolov6m_96_b2_feat", 0) > 0
    for name in ("yolov6n", "yolov6s_640_b32_u8", "yolov6m", "yolov6l6"):
        c = bwd.MODELS[name]
        eng = dry_planned(c["cfg"], c["batch"], c["size"], c.get("u8"), external_feat_grads=True)
        assert assert_neck_slices_accumulate(eng, name) >= len(eng.g.feat)
        # the same model without the flag: the first writer of each neck slice assigns (what the flag must change)
        eng.external_feat_grads = False
        with pytest.raises(AssertionError, match="assign into a neck-output"):
            assert_neck_slices_accumulate(eng, name)
        del eng


def test_neck_slice_check_catches_an_assigning_first_writer():
    """A hand-built plan: one buffer of 32 channels, the neck slice [8, 16), one full write over [0, 16).  Resolved with the
    external gradient flag off, the write assigns over the neck slice and the check fails; with it on, the write accumulates."""
    noop = lambda a: None                  # noqa: E731
    eng = types.SimpleNamespace(g=types.SimpleNamespace(bufs=[types.SimpleNamespace(c_total=32)],
                                                        feat=[types.SimpleNamespace(buf=0, c_off=8, c=8)]),
                                bwd_calls=[types.SimpleNamespace(writes=[Write(0, 0, 16, True, noop)])], gbufs=[None],
                                external_feat_grads=False)
    with pytest.raises(AssertionError, match="assign into a neck-output"):
        assert_neck_slices_accumulate(eng, "hand-built plan")
    eng.external_feat_grads = True
    assert assert_neck_slices_accumulate(eng, "hand-built plan") == 1
