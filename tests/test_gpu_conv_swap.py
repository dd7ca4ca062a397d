"""GPU parity of the 64-output-channel halo convs, whose tiles are computed transposed (64 channels x 128 pixels, weights as
the wgmma A operand, the input box as B) and written back through transposed epilogues.  Cases run through the parity checks
of test_gpu_conv.py (float64 reference, same tolerances), in both kernel families (CTA pairs forced on, single CTAs).

Already covered by BN = 64 halo plans elsewhere, so not repeated here:
  * stride 1, resident weights, bf16 TMA store: test_gpu_conv.py `3x3_persistent`; test_gpu_forward_launches.py (YOLOv6-S
    ERBlock_2.1 / Rep_p3 at their benchmarked shapes, bf16 and bf16x3);
  * stride 1, streamed weights, two channel blocks and two N tiles: test_gpu_conv.py `3x3_c128_40`, `3x3_direct_store`,
    `pair_c128_odd_tiles`; a partial N tile into a channel slice: test_gpu_conv_tma_store.py `concat_3x3_cout96_off32`;
  * residual through the chunk epilogue, resident weights: test_gpu_conv_pingpong.py `pp_halo_resident_many`;
  * bf16x3 planes, streamed weights: test_gpu_conv_pingpong.py `pp_halo_x3_streamed`;
  * column-pair view with skipped zero blocks: resident (test_gpu_conv.py `c64_skip_resident`, `c64_many_tiles`,
    test_gpu_conv_pingpong.py `pp_s2_resident_many`), streamed with a residual (`c64_cout128_streamed`), on a ragged output
    (`c64_ragged`), with bf16x3 planes (`c64_x3`).
New here: fp32 outputs (TMA store and chunk path; no model layer takes them at BN = 64), a stride-1 output cut by odd image
edges in both directions and written into a channel slice, a residual on streamed weights, and the column-pair view with a
residual on resident weights.
"""
import pytest

import test_gpu_conv as base

pytestmark = pytest.mark.gpu

CASES = [
    # name, N, H, W, Cin, Cout, k, stride, act, out_f32, nsplit, res, x_extra, y_extra, force   (as test_gpu_conv.CASES)
    ("swap_f32_resident", 2, 40, 40, 64, 64, 3, 1, "silu", True, 1, False, 0, 0, dict(halo=1)),           # fp32 TMA store
    ("swap_f32_x3_streamed", 2, 24, 24, 64, 64, 3, 1, "relu", True, 3, False, 0, 0, dict(halo=1)),        # fp32 TMA store, 6 plane pairs
    ("swap_f32_residual", 2, 24, 24, 64, 64, 3, 1, None, True, 1, True, 0, 0, dict(halo=1)),              # fp32 chunk epilogue
    ("swap_ragged_slices", 3, 23, 17, 64, 64, 3, 1, "relu", False, 1, False, 64, 128, dict(halo=1)),      # edges clip the TMA store
    ("swap_ragged_res_streamed", 2, 21, 13, 64, 64, 3, 1, "silu", False, 1, True, 0, 0, dict(halo=1, stages=4)),
]
EXPECT = {  # (halo, resident weights) of the single-CTA plan
    "swap_f32_resident": (1, 1), "swap_f32_x3_streamed": (1, 0), "swap_f32_residual": (1, 1), "swap_ragged_slices": (1, 1),
    "swap_ragged_res_streamed": (1, 0),
}

PAIR_VIEW_CASES = [
    # name, N, H, W, Cin, Cout, act, nsplit, residual, force, expect (halo, resident weights)   (as test_gpu_conv.PAIR_VIEW_CASES)
    ("swap_s2_skip_residual", 2, 32, 48, 64, 64, "relu", 1, True, None, (2, 1)),          # chunk epilogue, one zero block skipped
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cases_take_bn64_halo(case):
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, stride, _act, _f32, nsplit, _res, x_extra, _ye, force = case
    plan = ops.conv_plan((N, H, W, Cin + x_extra), (Cout, k, k, Cin), stride, nsplit, dict(force or {}, pair=-1))
    assert (plan["BN"], plan["halo"], plan["a_res"] % 10) == (64, *EXPECT[name]), plan


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_fwd_swap(case, pair):
    base.test_conv_fwd(case, pair)


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", PAIR_VIEW_CASES, ids=[c[0] for c in PAIR_VIEW_CASES])
def test_conv_stride2_pair_view_swap(case, pair):
    base.test_conv_stride2_pair_view(case, pair)
