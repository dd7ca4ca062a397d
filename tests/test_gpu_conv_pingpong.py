"""GPU parity of the conv kernel at the edges of its ping-pong schedule: the CTA's local tile j belongs to consumer warpgroup
j & 1, each warpgroup steps over the ring stages of the other's tiles, and the two hand the tensor cores to each other
between tiles.  The cases force the grid so that CTAs own an odd number of tiles, exactly one tile (the second warpgroup
idles), or dozens of tiles through resident and streamed weights.  Each runs through the parity checks of
test_gpu_conv.py, in both kernel families (CTA pairs forced on, single CTAs)."""
import pytest

import test_gpu_conv as base

pytestmark = pytest.mark.gpu

CASES = [
    # name, N, H, W, Cin, Cout, k, stride, act, out_f32, nsplit, res, x_extra, y_extra, force   (as test_gpu_conv.CASES)
    ("pp_odd_tiles_per_cta", 1, 40, 40, 64, 64, 1, 1, "silu", False, 1, True, 0, 0, dict(grid=6)),          # 3 or 2 tiles per CTA
    ("pp_one_tile_per_cta", 2, 20, 20, 64, 128, 3, 1, "relu", False, 1, False, 0, 0, dict(grid=4096)),      # grid = tile count
    ("pp_one_tile_64_rows", 1, 8, 8, 64, 96, 1, 1, "relu", True, 1, False, 0, 0, dict(grid=4096, bw=8, bh=8)),  # one 64-row pass
    ("pp_halo_resident_many", 8, 80, 80, 64, 64, 3, 1, "relu", False, 1, True, 0, 0, dict(grid=6)),        # ~67 tiles per CTA
    ("pp_halo_x3_streamed", 2, 48, 48, 64, 64, 3, 1, "relu", False, 3, False, 0, 0, dict(grid=7)),          # 6 plane pairs per tile
]

PAIR_VIEW_CASES = [
    # name, N, H, W, Cin, Cout, act, nsplit, residual, force, expect (halo, resident weights)   (as test_gpu_conv.PAIR_VIEW_CASES)
    ("pp_s2_resident_many", 8, 160, 160, 64, 64, "relu", 1, False, dict(grid=9), (2, 1)),                   # ~44 tiles per CTA
    ("pp_s2_streamed_many", 4, 128, 128, 64, 128, "silu", 1, True, dict(grid=5), (2, 0)),                  # skipped zero blocks
]


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_fwd_pingpong(case, pair):
    base.test_conv_fwd(case, pair)


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", PAIR_VIEW_CASES, ids=[c[0] for c in PAIR_VIEW_CASES])
def test_conv_stride2_pair_view_pingpong(case, pair):
    base.test_conv_stride2_pair_view(case, pair)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_plans_hit_the_schedule_edges(case):
    """The forced grids give the tile counts per CTA the cases are named for (single-CTA plans)."""
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, stride, _act, _f32, nsplit, _res, _xe, _ye, force = case
    plan = ops.conv_plan((N, H, W, Cin), (Cout, k, k, Cin), stride, nsplit, dict(force, pair=-1))
    per_cta = -(-plan["tiles"] // plan["grid"])
    if "one_tile" in name:
        assert plan["grid"] == plan["tiles"], plan
        if "64_rows" in name:
            assert plan["BW"] * plan["BH"] * plan["BI"] <= 64, plan
    elif "odd" in name:
        assert per_cta % 2 == 1, plan
    else:
        assert plan["halo"] == 1 and per_cta >= 5, plan
