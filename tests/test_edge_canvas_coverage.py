"""CPU proof that the configurations of tests/test_gpu_edge_canvases.py reach the edges they are chosen for, so that a
planner change cannot quietly move them off.  The inference launches come from engine.forward_launches with fake addresses
and the conv tile planner on the host at the H100 SXM's properties (as tests/test_forward_launch_coverage.py plans them);
the training launches from the training planner on a CPU engine with stand-ins for the library (tests/test_train_plan.py)
and the weight-gradient planner on the host (tests/test_backward_launch_coverage.py).

Also the top-k question of label assignment.  TAL takes the top-k anchors of the whole map (13; 26 in the anchor-aided
branch of a fuse_ab model, over its three anchors per cell), and the reference's torch.topk would raise on a map with fewer;
the kernel would pad its list with -1 instead.  Both engines plan only canvases whose sides are multiples of the largest
stride (the training planner used to plan any shape, 8 x 8 among them: one anchor), so the smallest map is the largest
stride square: 21 anchors for P5 (63 anchor-aided) and 85 for P6, every one above its top-k, and the padding path cannot be
reached from a model; tal_compact refuses a map with fewer anchors than top-k on the host, as the reference does.  ATSS
takes min(topk, anchors of the level) per level, and there a 1-anchor level is reachable: the GPU test covers it against
float64."""
import pytest
import torch

import test_gpu_edge_canvases as edge
from test_backward_launch_coverage import wgrad_plan
from test_forward_launch_coverage import records
from test_infer_plan import H100, host_plan
from test_train_plan import dry_engine_of
from yolov6_b200 import _lib, configs

HALO_H = {1: 18, 2: 33}        # input rows of the halo box (yv6_conv_igemm.cu kHaloH, HaloGeom<true>::H)
TR_THREADS = 256               # yv6_train.cu kTrThreads


def map_hw(g, op, H, W):
    lvl = g.bufs[op.src.buf].level
    return H >> lvl, W >> lvl


def upper_half_dead(p, N, Ho, Wo, w0, h0, i0):
    """yv6_conv_igemm.cu upper_half_dead restated: rows 64-127 of the tile at (w0, h0, i0) are all outside the output."""
    BW, BH, BI = p["BW"], p["BH"], p["BI"]
    q = 64 // BW
    r = (64 % BW, q % BH, BI if BW * BH * BI <= 64 else q // BH)
    ni, nh, nw = min(N - i0, BI), min(Ho - h0, BH), min(Wo - w0, BW)
    if ni <= 0 or nh <= 0 or nw <= 0:
        return True
    if ni - 1 != r[2]:
        return ni - 1 < r[2]
    if nh - 1 != r[1]:
        return nh - 1 < r[1]
    return nw - 1 < r[0]


def conv_out(d):
    if d.pair_view:
        return (d.H + 2 - 3) // 2 + 1, d.W
    pw = d.pad if d.pad_w == _lib.PAD_SAME else d.pad_w
    sw = d.stride_w or d.stride
    return (d.H + 2 * d.pad - d.kh) // d.stride + 1, (d.W + 2 * pw - d.kw) // sw + 1


@pytest.fixture(scope="module")
def inference():
    """Per configuration of the GPU test's inference tables: (config, graph, records, {record index: host plan})."""
    out = {}
    for name, c in list(edge.INFER.items()) + [("fp16 " + k, v) for k, v in edge.INFER_FP16.items()]:
        g, recs = records(c)
        out[name] = (c, g, recs, {j: host_plan(r.desc) for j, r in enumerate(recs) if r.kind == "conv"})
    return out


def test_inference_configs_reach_the_conv_edges(inference):
    halo_tall, dead_full, one_tile, pair_row = [], [], [], []
    for name, (c, g, recs, plans) in inference.items():
        for j, p in plans.items():
            d = recs[j].desc
            Ho, Wo = conv_out(d)
            if p["halo"] and d.H < HALO_H[p["halo"]]:
                halo_tall.append((name, recs[j].name, d.H))
            tiles = [(w0, h0, i0) for i0 in range(0, d.N, p["BI"]) for h0 in range(0, Ho, p["BH"]) for w0 in range(0, Wo, p["BW"])]
            if p["BW"] * p["BH"] * p["BI"] == 128 and all(upper_half_dead(p, d.N, Ho, Wo, *t) for t in tiles):
                dead_full.append((name, recs[j].name, len(tiles)))
            if p["tiles"] == p["grid"] == 1:
                one_tile.append((name, recs[j].name))
            if d.pair_view and Ho == 1:
                pair_row.append((name, recs[j].name))
    assert halo_tall, "no halo-mode conv whose input box is taller than its map (box rows > H)"
    assert dead_full, "no conv with a 128-row tile whose upper half (rows 64-127) is dead in every M tile"
    assert one_tile, "no conv whose whole output is one tile (tiles = grid = 1 persistent CTA)"
    assert pair_row, "no column-pair (stride-2 3x3) conv with a one-row output (Ho = 1)"
    print(f"\nhalo box taller than the map: {halo_tall[:3]}; dead upper half in every 128-row tile: {dead_full[:3]}; "
          f"one tile: {len(one_tile)} convs; one-row column-pair output: {pair_row[:3]}")


def test_inference_configs_reach_the_single_row_and_column_maps(inference):
    hits = {"pool": [], "convT": [], "dw": [], "se": []}
    one_anchor, se_min = [], set()
    for name, (c, g, recs, _) in inference.items():
        op_of = {op.name: op for op in g.ops}
        se_hw = [r.desc.HW for r in recs if r.kind == "se"]
        if se_hw:
            se_min.add(min(se_hw))
        for r in recs:
            if r.kind == "pool":
                h, w = r.args[2], r.args[3]
            elif r.kind == "dw":
                h, w = r.desc.H, r.desc.W
            elif r.kind == "se":
                h, w = map_hw(g, op_of[r.name], c["H"], c["W"])
                assert h * w == r.desc.HW
            elif r.kind == "conv" and "[" in r.conv["name"]:
                h, w = r.desc.H, r.desc.W
            else:
                continue
            if h == 1 or w == 1:
                hits["convT" if r.kind == "conv" else r.kind].append((name, r.name, h, w))
        one_anchor += [(name, s) for s in g.strides if (c["H"] // s) * (c["W"] // s) == 1]
    for kind, what in (("pool", "SPPF 5x5 max-pool"), ("convT", "ConvTranspose quadrant scatter"), ("dw", "depthwise conv")):
        assert hits[kind], f"no {what} launch on a map with H = 1 or W = 1"
        assert any(h == 1 for _, _, h, _ in hits[kind]) and any(w == 1 for _, _, _, w in hits[kind]), \
            f"the {what} launches reach H = 1 or W = 1 but not both: {hits[kind][:4]}"
    # SE sits only in the Lite backbone, at strides up to 32, and the Lite graph's largest stride is 64: its smallest map is
    # 2 x 2 (HW = 4), reached at 64 x 64, and its thinnest a 2-row strip, reached at 64 x 640
    assert not hits["se"], f"an SE launch on a 1-pixel side: {hits['se'][:2]} (reachable now: check it against float64)"
    assert se_min == {4, 40}, f"SE launches over HW = {sorted(se_min)} pixels, want the 2 x 2 and 2 x 20 maps (HW 4 and 40)"
    assert one_anchor, "no head decode level with exactly one anchor (map 1 x 1)"
    print("\n" + "; ".join(f"{k}: {len(v)} launches on 1-pixel rows / columns" for k, v in hits.items())
          + f"; smallest SE maps HW {sorted(se_min)}; one-anchor decode levels: {one_anchor}")


@pytest.fixture(scope="module")
def training():
    out = {}
    for name, (cfg, H, W, B, fuse_ab) in edge.TRAIN.items():
        eng, _ = dry_engine_of(cfg, 1, fuse_ab=fuse_ab)
        eng._plan(B, H, W, torch.float32)
        out[name] = (list(eng.fwd_calls), list(eng.bwd_calls))
        del eng
    return out


def test_training_plans_reach_the_tiny_reductions(training):
    """A weight gradient whose dY has fewer pixels than one split's pixel tiles (the planner's split-K never splits fewer than
    eight tiles, so at these shapes the one split's TMA boxes lie mostly outside the tensor), and BatchNorm statistics over
    fewer pixels than the pixel rows of one block of bn_stats_finalize (chan_grid: most per-thread runs are empty)."""
    wg, st = [], []
    for name, (fwd_calls, bwd_calls) in training.items():
        for c in bwd_calls:
            if c.kind == "wgrad":
                d = c.desc
                Ho, Wo = (d.H + 2 * d.pad - d.kh) // d.stride + 1, (d.W + 2 * d.pad - d.kw) // d.stride + 1
                p = wgrad_plan(d)
                if d.N * Ho * Wo < p["split_pixels"]:
                    wg.append((name, d.N * Ho * Wo, p["ksplit"], p["split_pixels"]))
        for c in fwd_calls:
            if c.kind == "stats":
                rows = max(1, TR_THREADS // (c.desc.C // 8))
                if c.desc.pixels < rows:
                    st.append((name, c.desc.pixels, c.desc.C, rows))
    assert wg, "no weight gradient whose pixel count (N Ho Wo) is below the pixels of one split"
    assert min(n for _, n, _, _ in wg) <= 2, f"the smallest weight gradient sums {min(n for _, n, _, _ in wg)} pixels, not batch x 1 x 1"
    assert st, "no BatchNorm statistics launch over fewer pixels than the pixel rows of one block"
    assert min(n for _, n, _, _ in st) <= 2, "no BatchNorm statistics over batch x 1 x 1 pixels"
    print(f"\nwgrad below one split: {len(wg)} launches, e.g. {wg[:2]}; stats with empty thread rows: {len(st)}, e.g. {st[:2]}")


def test_training_plans_reach_single_pixel_maps(training):
    """The SPPF pool on a 1 x W or H x 1 map in every training configuration (its backward chain reads the same shape)."""
    for name, (fwd_calls, _) in training.items():
        pools = [c.args[2:4] for c in fwd_calls if c.kind == "pool"]
        assert pools and any(1 in hw for hw in pools), f"{name}: SPPF maps {pools} have no side of one pixel"


# ---------------------------------------------------------------------------------------------------------------- the top-k question
def min_anchors(strides, per_cell=1):
    """Anchors of the smallest canvas the engines plan (a multiple of the largest stride on both sides): s_max x s_max."""
    m = max(strides)
    return per_cell * sum((m // s) ** 2 for s in strides)


def test_no_accepted_shape_gives_tal_fewer_anchors_than_topk():
    seen = {}
    for name in configs.CONFIGS:
        head = configs.get_config(name)["head"]
        strides = head["strides"]
        seen[name] = min_anchors(strides)
        assert seen[name] >= 13, f"{name}: {seen[name]} anchors at {max(strides)} x {max(strides)}, below TAL's top-k of 13"
        if head.get("anchors_init"):                    # a fuse_ab head: loss_fuseab's three anchors per cell, top-k 26
            n = min_anchors(strides, 3)
            seen[name + " (anchor-aided)"] = n
            assert n >= 26, f"{name} fuse_ab: {n} anchor-aided anchors at {max(strides)} x {max(strides)}, below top-k 26"
    assert min(seen.values()) == 21 and seen["yolov6n (anchor-aided)"] == 63 and seen["yolov6n6"] == 85, seen
    print("\nsmallest anchor count per configuration: " + ", ".join(f"{k} {v}" for k, v in seen.items()))


@pytest.mark.parametrize("cfg,H,W", [("yolov6n", 8, 8), ("yolov6n", 16, 16), ("yolov6n", 48, 48), ("yolov6n", 32, 100),
                                     ("yolov6n6", 32, 64), ("yolov6n6", 64, 96)])
def test_training_planner_refuses_a_side_off_the_largest_stride(cfg, H, W):
    """The training planner refuses the shapes the inference engine refuses, with its message.  It used to plan them: 8 x 8
    left YOLOv6-N one anchor for TAL's top-13 (maps 1 x 1, 0 x 0, 0 x 0), and at 48 x 48 the stride-2 conv from the 3 x 3
    P4 map computes a 2 x 2 output into a 1 x 1 P5 buffer."""
    eng, _ = dry_engine_of(cfg, 1)
    s = max(eng.g.strides)
    with pytest.raises(RuntimeError, match=f"input {H}x{W} must be a multiple of the largest stride {s}"):
        eng._plan(2, H, W, torch.float32)
    eng._plan(2, s, s, torch.float32)
    assert eng.offs[-1] == min_anchors(eng.g.strides)


def test_tal_refuses_fewer_anchors_than_topk():
    """The reference's condition (torch.topk over the anchors raises) on the host, before any launch."""
    from yolov6_b200.assigners import tal_compact
    gt, mask = torch.zeros(2, 3, 5, dtype=torch.float64), torch.zeros(2, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="top-13 candidates of a map with 12 anchors"):
        tal_compact(torch.zeros(2, 12, 80), torch.zeros(2, 12, 4), torch.zeros(12, 2), gt, mask, 13)
    with pytest.raises(ValueError, match="top-26 candidates of a map with 21 anchors"):
        tal_compact(torch.zeros(2, 21, 80), torch.zeros(2, 21, 4), torch.zeros(21, 2), gt, mask, 26)


def test_smallest_edge_canvases_reach_a_one_anchor_atss_level():
    """ATSS at the GPU test's smallest canvases: a level of one anchor, below its top-k of 9 (min(topk, count) per level)."""
    for name in ("p5_32x32_atss", "p6_64x64_atss"):
        cfg, _ = edge.LOSS[name]
        counts = [(cfg["H"] // s) * (cfg["W"] // s) for s in cfg["strides"]]
        assert min(counts) == 1 < cfg["topk"], (name, counts)
        assert sum(counts) >= 13, (name, counts)
