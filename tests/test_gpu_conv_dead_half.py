"""GPU parity of conv tiles whose rows 64-127 lie wholly outside the output, for which the kernel issues only the rows 0-63
MMAs and skips the upper half in the epilogue.

The 8 x 16 halo tiles of a map with Ho % 16 in 1..8 (the 40 x 40 maps of YOLOv6-S/M at 640) keep only their pixel rows 0-63
in the last tile row; a mode-0 box of <= 64 rows, or one cut by the bottom or batch edge, can lose its upper half too.  Each
case runs in both kernel families (CTA pairs forced on, single CTAs) against the float64 conv of test_gpu_conv.py, with the
output written into a view of a larger buffer: 8 more rows below it and, in some cases, more channels on both sides.  Every
element outside the view must keep its sentinel, since the bf16 TMA store of a dead half sends whatever its staging rows hold
and relies on the store clipping them.  Ho % 16 == 9 is the control: its last tile row has one live row above 64.
"""
import pytest
import torch

import test_gpu_conv as base

pytestmark = pytest.mark.gpu
SENTINEL = 7.0
BELOW = 8          # rows of sentinel under the output view
# The planner would give these small maps BN = 64 (one wave either way), whose transposed tiles have no dead half
H128 = dict(halo=1, bn=128)

CASES = [
    # name, N, H, W, Cin, Cout, k, act, out_f32, nsplit, res, y_extra, pair_view, force, expect (halo, BN)
    ("h1_ho40_streamed", 2, 40, 40, 128, 128, 3, "relu", False, 1, False, 0, False, H128, (1, 128)),
    ("h1_ho24_two_ntiles", 2, 24, 40, 256, 256, 3, "silu", False, 1, False, 64, False, H128, (1, 128)),
    ("h1_ho33_one_live_row", 2, 33, 24, 128, 128, 3, "relu", False, 1, False, 0, False, H128, (1, 128)),
    ("h1_ho25_control", 2, 25, 24, 128, 128, 3, "relu", False, 1, False, 0, False, H128, (1, 128)),
    ("h1_residual_chunks", 2, 40, 40, 128, 128, 3, "relu", False, 1, True, 32, False, H128, (1, 128)),
    ("h1_f32_tma", 2, 40, 24, 128, 128, 3, "sigmoid", True, 1, False, 0, False, H128, (1, 128)),
    ("h1_f32_residual_chunks", 2, 24, 16, 128, 128, 3, None, True, 1, True, 0, False, H128, (1, 128)),
    ("h1_x3_planes", 2, 24, 24, 128, 128, 3, "relu", False, 3, False, 0, False, H128, (1, 128)),
    ("h1_x3_f32", 2, 40, 16, 128, 128, 3, "silu", True, 3, False, 0, False, H128, (1, 128)),
    ("h1_cout96", 2, 40, 24, 128, 96, 3, "silu", False, 1, False, 32, False, dict(halo=1, bn=96), (1, 96)),
    # a forced grid of 4 over 30 tiles: in the single-CTA plan each consumer warpgroup of CTA 1 owns full and half tiles
    ("h1_grid_mixed", 2, 40, 40, 128, 128, 3, "relu", False, 1, False, 0, False, dict(H128, grid=4), (1, 128)),
    # 3x3 stride 2 on the column-pair view [N, H, W/2, 2 Cin] (Ho = H / 2), two of its four channel blocks skipped on the left taps
    ("h2_ho40", 2, 80, 80, 128, 128, 3, "relu", False, 1, False, 0, True, H128, (2, 128)),
    ("h2_ho33_residual", 2, 66, 48, 128, 256, 3, "silu", False, 1, True, 0, True, H128, (2, 128)),
    # mode 0: a forced 8 x 8 box (every tile's upper half beyond the box), a 16 x 8 box cut by Ho = 20, two images per box
    ("m0_box8x8", 2, 20, 20, 64, 128, 3, "relu", False, 1, False, 0, False, dict(bw=8, bh=8, bn=128), (0, 128)),
    ("m0_box16x8_ho20", 2, 20, 32, 64, 128, 1, "silu", False, 1, False, 64, False, dict(bw=16, bh=8, bn=128), (0, 128)),
    ("m0_two_images_odd_batch", 3, 8, 8, 64, 64, 1, "relu", True, 1, True, 0, False, dict(bw=8, bh=8, bi=2, bn=64), (0, 64)),
]


def _out_hw(case):
    _n, _N, H, W, _ci, _co, k, *_rest = case
    pair_view = case[12]
    if pair_view:
        return H // 2, W // 2
    return H + 2 * (k // 2) - k + 1, W + 2 * (k // 2) - k + 1


def _plan(case, pair):
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, _act, _f32, nsplit, _res, _ye, pair_view, force, _exp = case
    force = dict(force or {}, pair=pair)
    if pair_view:
        _Ho, Wo = _out_hw(case)
        return ops.conv_plan((N, H, W // 2, 2 * Cin), (Cout, 3, 2, 2 * Cin), 2, nsplit, force, stride_w=1, pad=(1, 1),
                             out_hw=(0, Wo), pair_view=1)
    return ops.conv_plan((N, H, W, Cin), (Cout, k, k, Cin), 1, nsplit, force)


def _dead(plan, N, Ho, Wo):
    """[M tile] -> rows 64-127 of its box all outside the output (the kernel's upper_half_dead)."""
    BW, BH, BI = plan["BW"], plan["BH"], plan["BI"]
    tw, th, ti = -(-Wo // BW), -(-Ho // BH), -(-N // BI)
    out = []
    for m in range(tw * th * ti):
        w0, h0, i0 = (m % tw) * BW, (m // tw % th) * BH, (m // (tw * th)) * BI
        live = [bw + BW * (bh + BH * bi) >= 64
                for bi in range(BI) for bh in range(BH) for bw in range(BW)
                if i0 + bi < N and h0 + bh < Ho and w0 + bw < Wo]
        out.append(not any(live))
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cases_have_dead_upper_halves(case):
    """The single-CTA plans take the expected mainloop and BN, and every case but the control has tiles with a dead upper half."""
    name, N, *_ = case
    plan = _plan(case, -1)
    assert (plan["halo"], plan["BN"]) == case[-1], plan
    Ho, Wo = _out_hw(case)
    dead = _dead(plan, N, Ho, Wo)
    if "control" in name:
        assert not any(dead), plan
    else:
        assert any(dead) and ("box8x8" in name) == all(dead), (plan, dead)
    if "grid_mixed" in name:
        tiles_n = plan["tiles"] // len(dead)
        assert plan["grid"] == 4 and tiles_n == 1, plan
        for wg in range(2):      # CTA 1, warpgroup wg: local tiles wg, wg + 2, ... = tiles 1 + 4 (wg + 2 j)
            owned = [dead[t] for t in range(1 + 4 * wg, len(dead), 8)]
            assert any(owned) and not all(owned), (wg, owned)


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_dead_upper_half(case, pair):
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, act, out_f32, nsplit, use_res, y_extra, pair_view, force, _exp = case
    force = dict(force or {}, pair=pair)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    Ho, Wo = _out_hw(case)
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    res = torch.randn(N, Ho, Wo, Cout, generator=g) if use_res else None
    bias = ops.pad_bias(b.to(dev), Cout)
    yoff = y_extra // 2
    ydt = torch.float32 if out_f32 else torch.bfloat16
    planes = nsplit == 3 and not out_f32
    big = torch.full(((3,) if planes else ()) + (N, Ho + BELOW, Wo, Cout + y_extra), SENTINEL, dtype=ydt, device=dev)
    y = big[..., :Ho, :, :]
    kw = dict(act=act, y_c_offset=yoff, alpha=0.5, nsplit=nsplit, force=force)
    if pair_view:
        kw.update(stride=2, stride_w=1, pad=(1, 1), out_hw=(0, Wo), pair_view=1)
        wk = ops.pair_view_weights(w)
    else:
        wk = w
    if nsplit == 1:
        xk, wk, resk = x.to(torch.bfloat16), wk.to(torch.bfloat16), res.to(torch.bfloat16) if use_res else None
        ref = base.ref_conv(xk.float(), w.to(torch.bfloat16).float(), b, 2 if pair_view else 1, act,
                            resk.float() if use_res else None, 0.5)
        # fp32 outputs: the fp32 accumulation over K = 1152 (3x3 x 128 channels) leaves up to ~4e-6 of rounding against the
        # float64 sum, twice test_gpu_conv.py's bound for its K <= 576 cases; a wrong or missing row half is off by O(1)
        tol = 1e-5 if out_f32 else 2.0 ** -8
    else:
        xk, wk, resk = ops.split3(x), ops.split3(wk), ops.split3(res) if use_res else None
        ref = base.ref_conv(x, w, b, 2 if pair_view else 1, act, res, 0.5)
        tol = 5e-6
    if pair_view:
        xk = xk.view(*xk.shape[:-2], W // 2, 2 * Cin)
    ops.conv_fwd(xk.to(dev), wk.to(dev), bias, y, res=resk.to(dev) if use_res else None, **kw)
    got_all = big.float().cpu()
    outside = torch.ones(got_all.shape, dtype=torch.bool)
    outside[..., :Ho, :, yoff:yoff + Cout] = False
    assert bool((got_all[outside] == SENTINEL).all()), f"{name}: wrote outside the output view"
    got = got_all[..., :Ho, :, yoff:yoff + Cout]
    got = (got.sum(0) if planes else got).double()
    err = ((got - ref).abs() / (1.0 + ref.abs())).max().item()
    assert err <= tol, f"{name}: rel err {err:.3e} > {tol:.1e}"
