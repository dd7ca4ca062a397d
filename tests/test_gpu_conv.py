"""GPU parity of the wgmma implicit-GEMM conv kernel (through the C ABI) against an fp64 CPU
convolution of the same (bf16-rounded or bf16x3-split) operands."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

CASES = [
    # name, N, H, W, Cin, Cout, k, stride, act, out_f32, nsplit, res, x_extra, y_extra, force
    ("1x1_c64", 2, 20, 20, 64, 64, 1, 1, "relu", False, 1, False, 0, 0, None),
    ("3x3_c128_40", 2, 40, 40, 128, 128, 3, 1, "relu", False, 1, False, 0, 0, None),
    ("3x3_c512_ntiles", 2, 20, 20, 512, 512, 3, 1, "relu", False, 1, False, 0, 0, None),
    ("3x3_s2_odd", 1, 23, 17, 64, 64, 3, 2, "relu", False, 1, False, 0, 0, None),
    ("3x3_s1_odd_cout96", 3, 23, 17, 64, 96, 3, 1, "silu", False, 1, False, 0, 0, None),
    ("3x3_cin32_sw64_s2", 2, 32, 32, 32, 64, 3, 2, "relu", False, 1, False, 0, 0, None),
    ("1x1_cin48_sw32", 2, 16, 16, 48, 96, 1, 1, "relu", False, 1, False, 0, 0, None),
    ("1x1_cout80_sigmoid_f32", 2, 20, 20, 128, 80, 1, 1, "sigmoid", True, 1, False, 0, 0, None),
    ("1x1_cout4_f32", 2, 20, 20, 64, 4, 1, 1, None, True, 1, False, 0, 0, None),
    ("1x1_cout68_f32", 2, 20, 20, 64, 68, 1, 1, None, True, 1, False, 0, 0, None),
    ("3x3_residual", 2, 20, 20, 64, 64, 3, 1, "relu", False, 1, True, 0, 0, None),
    ("3x3_slices", 2, 20, 20, 64, 64, 3, 1, "relu", False, 1, False, 64, 128, None),
    ("3x3_persistent", 4, 40, 40, 64, 64, 3, 1, "relu", False, 1, False, 0, 0, dict(grid=8)),
    ("3x3_direct_store", 2, 40, 40, 128, 128, 3, 1, "relu", False, 1, False, 0, 0, dict(direct=1)),
    ("3x3_x3", 2, 20, 20, 64, 64, 3, 1, "relu", False, 3, False, 0, 0, None),
    ("3x3_x3_s2", 2, 20, 20, 64, 128, 3, 2, "relu", False, 3, False, 0, 0, None),
    ("1x1_x3_f32out", 2, 20, 20, 64, 80, 1, 1, "sigmoid", True, 3, False, 0, 0, None),
    ("3x3_x3_residual", 2, 20, 20, 64, 64, 3, 1, "relu", False, 3, True, 0, 0, None),
    ("3x3_bi_batch5", 5, 10, 10, 64, 64, 3, 1, "relu", False, 1, False, 0, 0, None),
    # many tiles per CTA (persistent loop over tiles), small weight tensors
    ("3x3_s2_cin32_many_tiles", 8, 160, 160, 32, 64, 3, 2, "relu", False, 1, False, 0, 0, None),
    ("1x1_many_tiles_res", 8, 96, 96, 64, 64, 1, 1, "silu", False, 1, True, 0, 0, None),
    ("3x3_s2_x3_many_tiles", 6, 96, 96, 32, 32, 3, 2, "relu", False, 3, False, 0, 0, None),
    # CTA-pair specifics (2-CTA clusters, weight tile multicast): odd tile counts (the missing second tile of the last unit), N split + residual,
    # channel slices, several units per cluster, bf16x3 planes, a full-size layer
    ("pair_c128_odd_tiles", 1, 24, 24, 128, 128, 3, 1, "silu", False, 1, False, 0, 0, None),
    ("pair_c256_nsplit_res", 2, 40, 40, 512, 512, 3, 1, "relu", False, 1, True, 0, 0, None),
    ("pair_c64_cout128_slices", 3, 23, 17, 64, 128, 3, 1, "relu", False, 1, False, 64, 128, None),
    ("pair_persistent", 4, 80, 80, 128, 128, 3, 1, "relu", False, 1, False, 0, 0, dict(grid=8)),
    ("pair_x3", 2, 20, 20, 128, 128, 3, 1, "relu", False, 3, True, 0, 0, None),
    ("pair_c128_80_bs8", 8, 80, 80, 128, 128, 3, 1, "relu", False, 1, False, 0, 0, None),
    ("pair_1x1_cout80_f32_many", 8, 80, 80, 64, 80, 1, 1, "sigmoid", True, 1, False, 0, 0, None),
    ("pair_s2_c128_256", 4, 80, 80, 128, 256, 3, 2, "relu", False, 1, False, 0, 0, None),
]


def ref_conv(x, w, b, stride, act, res, alpha):
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), b.double(), stride=stride,
                 padding=w.shape[1] // 2)
    y = {"relu": torch.relu, "silu": lambda t: t * torch.sigmoid(t), "sigmoid": torch.sigmoid, None: lambda t: t}[act](y)
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + alpha * res.double()
    return y


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_fwd(case, pair):
    """Every case runs through both kernel families: CTA pairs (clusters of two CTAs on adjacent M tiles, each loading half of
    the weight tile and multicasting it to both; forced on here) and the single-CTA variants."""
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, stride, act, out_f32, nsplit, use_res, x_extra, y_extra, force = case
    force = dict(force or {}, pair=pair)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    Ct = Cin + x_extra
    xfull = torch.randn(N, H, W, Ct, generator=g)
    w = torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    res = torch.randn(N, Ho, Wo, Cout, generator=g) if use_res else None
    xoff, yoff = x_extra // 2, y_extra // 2
    bias = ops.pad_bias(b.to(dev), Cout)
    ydt = torch.float32 if out_f32 else torch.bfloat16
    if nsplit == 1:
        xb, wb = xfull.to(torch.bfloat16), w.to(torch.bfloat16)
        resb = res.to(torch.bfloat16) if use_res else None
        y = torch.full((N, Ho, Wo, Cout + y_extra), 7.0, dtype=ydt, device=dev)
        ops.conv_fwd(xb.to(dev), wb.to(dev), bias, y, x_c_offset=xoff, stride=stride, act=act, y_c_offset=yoff,
                     res=resb.to(dev) if use_res else None, alpha=0.5, force=force)
        ref = ref_conv(xb.float()[..., xoff:xoff + Cin], wb.float(), b, stride, act, resb.float() if use_res else None, 0.5)
        got = y.float().cpu()
        assert bool((got[..., :yoff] == 7).all() and (got[..., yoff + Cout:] == 7).all()), "wrote outside its slice"
        got = got[..., yoff:yoff + Cout].double()
        tol = 2e-6 if out_f32 else 2.0 ** -8      # fp32 accumulate; bf16 output rounding = 2^-9 relative
    else:
        x3, w3 = ops.split3(xfull), ops.split3(w)
        res3 = ops.split3(res) if use_res else None
        y = torch.zeros((N, Ho, Wo, Cout) if out_f32 else (3, N, Ho, Wo, Cout), dtype=ydt, device=dev)
        ops.conv_fwd(x3.to(dev), w3.to(dev), bias, y, stride=stride, act=act, res=res3.to(dev) if use_res else None,
                     alpha=0.5, nsplit=3, force=force)
        ref = ref_conv(xfull, w, b, stride, act, res, 0.5)
        got = (y if out_f32 else y.float().sum(0)).cpu().double()
        tol = 5e-6                                  # fp32-equivalent mode
    err = ((got - ref).abs() / (1.0 + ref.abs())).max().item()
    assert err <= tol, f"{name}: rel err {err:.3e} > {tol:.1e}"


PAIR_VIEW_CASES = [
    # name, N, H, W, Cin, Cout, act, nsplit, residual, force, expect (halo, resident weights)
    ("c32_one_block", 2, 64, 64, 32, 64, "relu", 1, False, None, (2, 1)),                 # 2*Cin = 64: a single channel block, nothing skipped
    ("c64_skip_resident", 2, 32, 48, 64, 64, "silu", 1, False, None, (2, 1)),             # zero block of the left tap skipped, 9 resident tiles
    ("c64_cout128_streamed", 1, 64, 64, 64, 128, "relu", 1, True, None, (2, 0)),          # weights through the ring
    ("c64_ragged", 3, 34, 20, 64, 96, "relu", 1, False, dict(halo=1), (2, 0)),            # Ho = 17, Wo = 10: partial tiles in both directions
    ("c128_forced", 2, 64, 32, 128, 128, "relu", 1, False, dict(halo=1), (2, 0)),         # four channel blocks, two of them skipped on the left taps
    ("c64_x3", 2, 32, 32, 64, 64, "relu", 3, False, None, (2, 0)),                        # bf16x3 planes
    ("c64_many_tiles", 8, 160, 160, 64, 64, "relu", 1, False, None, (2, 1)),              # persistent loop, resident weights reused
    ("c64_generic_fallback", 2, 20, 20, 64, 64, "relu", 1, False, None, (0, 0)),          # 10 x 10 output: the fixed tile wastes too much
]


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", PAIR_VIEW_CASES, ids=[c[0] for c in PAIR_VIEW_CASES])
def test_conv_stride2_pair_view(case, pair):
    """A 3x3 stride-2 conv run as the 3x2 / stride (2, 1) conv on the column-pair view [N, H, W/2, 2*Cin] of its input
    (include/yv6.h `stride_w`, `pair_view`; the halo-reuse mainloop MODE 3 / 4 of yv6_conv_igemm.cu) against the fp64
    convolution of the ORIGINAL 3x3 stride-2 problem."""
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, act, nsplit, use_res, force, expect = case
    force = dict(force or {}, pair=pair)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    Ho, Wo = H // 2, W // 2
    res = torch.randn(N, Ho, Wo, Cout, generator=g) if use_res else None
    bias = ops.pad_bias(b.to(dev), Cout)
    wv = ops.pair_view_weights(w)
    plan = ops.conv_plan((N, H, W // 2, 2 * Cin), tuple(wv.shape), 2, nsplit, force, stride_w=1, pad=(1, 1), out_hw=(0, Wo), pair_view=1)
    assert plan["halo"] == expect[0], plan
    if pair < 0:        # (a CTA pair stages half of the weight tile per CTA, so more layers keep their weights resident)
        assert plan["a_res"] % 10 == expect[1], plan
    kw = dict(stride=2, stride_w=1, pad=(1, 1), out_hw=(0, Wo), pair_view=1, act=act, alpha=0.5, force=force)
    if nsplit == 1:
        xb, wb = x.to(torch.bfloat16), wv.to(torch.bfloat16)
        resb = res.to(torch.bfloat16) if use_res else None
        y = torch.zeros(N, Ho, Wo, Cout, dtype=torch.bfloat16, device=dev)
        ops.conv_fwd(xb.view(N, H, W // 2, 2 * Cin).to(dev), wb.to(dev), bias, y, res=resb.to(dev) if use_res else None, **kw)
        ref = ref_conv(xb.float(), w.to(torch.bfloat16).float(), b, 2, act, resb.float() if use_res else None, 0.5)
        got, tol = y.float().cpu().double(), 2.0 ** -8
    else:
        x3, w3 = ops.split3(x), ops.split3(wv)
        y = torch.zeros(3, N, Ho, Wo, Cout, dtype=torch.bfloat16, device=dev)
        ops.conv_fwd(x3.view(3, N, H, W // 2, 2 * Cin).to(dev), w3.to(dev), bias, y, nsplit=3, **kw)
        ref = ref_conv(x, w, b, 2, act, None, 0.5)
        got, tol = y.float().sum(0).cpu().double(), 5e-6
    err = ((got - ref).abs() / (1.0 + ref.abs())).max().item()
    assert err <= tol, f"{name}: rel err {err:.3e} > {tol:.1e}"


def test_conv_rejects_bad_arguments():
    from yolov6_b200 import ops
    dev = torch.device("cuda:0")
    x = torch.zeros(1, 8, 8, 24, dtype=torch.bfloat16, device=dev)      # Cin not a multiple of 16
    w = torch.zeros(16, 1, 1, 24, dtype=torch.bfloat16, device=dev)
    y = torch.zeros(1, 8, 8, 16, dtype=torch.bfloat16, device=dev)
    with pytest.raises(RuntimeError):
        ops.conv_fwd(x, w, None, y)


@pytest.mark.parametrize("N,H,W,Cout,act,u8,fp32_math", [
    (2, 64, 64, 32, "relu", False, 0), (1, 70, 50, 16, "relu", False, 0), (2, 33, 65, 64, "silu", True, 0),
    (1, 128, 96, 48, None, False, 0), (2, 64, 64, 32, None, False, 1), (1, 37, 41, 16, "relu", True, 1)])
def test_stem_kernels_match_torch(N, H, W, Cout, act, u8, fp32_math):
    """yv6_stem_fwd (3x3 stride-2 conv over the 3-channel image, common.py:197-255 deploy form of the first
    RepVGGBlock / ConvBNSiLU): tensor-core path on bf16-rounded image / weights, and the fp32 CUDA-core path."""
    import ctypes as C
    from yolov6_b200 import _lib, ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(H * 131 + W)
    x = (torch.rand(N, 3, H, W, generator=g) * 255).to(torch.uint8) if u8 else torch.rand(N, 3, H, W, generator=g)
    w = torch.randn(Cout, 3, 3, 3, generator=g) * 0.3
    b = torch.randn(Cout, generator=g) * 0.1
    xf = x.float() / 255 if u8 else x
    if fp32_math:
        ref = F.conv2d(xf.double(), w.double(), b.double(), stride=2, padding=1)
    else:   # the kernel rounds image and weights to bf16, accumulates in fp32
        ref = F.conv2d(xf.to(torch.bfloat16).double(), w.to(torch.bfloat16).double(), b.double(), stride=2, padding=1)
    ref = torch.relu(ref) if act == "relu" else (ref * torch.sigmoid(ref) if act == "silu" else ref)
    Ho, Wo = ref.shape[2], ref.shape[3]
    xd = x.to(dev).contiguous()
    wd = w.permute(2, 3, 1, 0).contiguous().to(dev)        # [3][3][3][Cout]
    bd = b.to(dev)
    y = torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.bfloat16, device=dev)
    d = ops.stem_desc(xd.data_ptr(), N, H, W, u8, wd.data_ptr(), bd.data_ptr(), Cout, act, y.data_ptr(), fp32_math=fp32_math)
    _lib.check(_lib.lib().yv6_stem_fwd(_lib.handle(0), C.byref(d), _lib.stream_ptr()))
    got = y.float().permute(0, 3, 1, 2).double().cpu()
    assert torch.isfinite(got).all()
    err = float((got - ref).abs().max() / (1 + ref.abs().max()))
    assert err < 6e-3, err          # bf16 output rounding (2^-9 relative)
