"""GPU parity of the conv kernel's TMA-store epilogue on the output views its tensor map describes: a channel slice of a
wider (concat) buffer at a non-zero offset, the quadrant scatter of a ConvTranspose2d k2s2, the fp32 [N, A, ch] head outputs
at a level's anchor offset, and tiles cut by the edges of the output (width, height and batch).  Every element outside the
view must keep its sentinel value.  Both kernel families (CTA pairs forced on, single CTAs)."""
import pytest
import torch

import test_gpu_conv as base

pytestmark = pytest.mark.gpu
SENTINEL = 7.0


def _operands(N, H, W, Cin, Cout, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, Cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, generator=g) * 0.1
    return x, w, b


def _check(got, ref, tol, what):
    err = ((got.double() - ref).abs() / (1.0 + ref.abs())).max().item()
    assert err <= tol, f"{what}: rel err {err:.3e} > {tol:.1e}"


SLICE_CASES = [
    # name, N, H, W, Cin, Cout, k, stride, act, channel pitch, channel offset
    ("concat_1x1_c64_off64", 2, 40, 40, 64, 64, 1, 1, "silu", 192, 64),
    ("concat_1x1_c128_off128", 2, 20, 20, 128, 128, 1, 1, "relu", 256, 128),
    ("concat_3x3_cout96_off32", 2, 24, 24, 64, 96, 3, 1, "silu", 160, 32),
    ("edges_3x3_s1_23x17", 3, 23, 17, 64, 64, 3, 1, "relu", 64, 0),
    ("edges_3x3_s2_23x17_cout32", 2, 23, 17, 64, 32, 3, 2, "silu", 96, 64),
    ("edges_batch_tiles_5x5", 7, 5, 5, 64, 64, 1, 1, "relu", 64, 0),
]


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("case", SLICE_CASES, ids=[c[0] for c in SLICE_CASES])
def test_bf16_slices_and_edges(case, pair):
    from yolov6_b200 import ops
    name, N, H, W, Cin, Cout, k, stride, act, pitch, off = case
    dev = torch.device("cuda:0")
    x, w, b = _operands(N, H, W, Cin, Cout, k, seed=2)
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    y = torch.full((N, Ho, Wo, pitch), SENTINEL, dtype=torch.bfloat16, device=dev)
    ops.conv_fwd(x.to(dev), w.to(dev), ops.pad_bias(b.to(dev), Cout), y, stride=stride, act=act, y_c_offset=off, force=dict(pair=pair))
    got = y.float().cpu()
    assert bool((got[..., :off] == SENTINEL).all() and (got[..., off + Cout:] == SENTINEL).all()), "wrote outside its slice"
    _check(got[..., off:off + Cout], base.ref_conv(x.float(), w.float(), b, stride, act, None, 0.0), 2.0 ** -8, name)


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("shape", [(2, 20, 20, 128, 64, 64, 128), (3, 13, 9, 64, 96, 32, 160)], ids=["c128_20x20", "c64_13x9_ragged"])
def test_convtranspose_quadrant_scatter(shape, pair):
    """ConvTranspose2d k2s2 as four 1x1 launches, quadrant (dy, dx) written to output pixels (2 i + dy, 2 j + dx) of a channel
    slice: the output map's W / H strides are twice the buffer's."""
    from yolov6_b200 import ops
    N, H, W, Cin, Cout, off, pitch = shape
    dev = torch.device("cuda:0")
    x, _, b = _operands(N, H, W, Cin, Cout, 1, seed=3)
    g = torch.Generator().manual_seed(4)
    wq = (torch.randn(4, Cout, 1, 1, Cin, generator=g) / Cin ** 0.5).to(torch.bfloat16)
    y = torch.full((N, 2 * H, 2 * W, pitch), SENTINEL, dtype=torch.bfloat16, device=dev)
    xd, bias = x.to(dev), ops.pad_bias(b.to(dev), Cout)
    for q in range(4):
        ops.conv_fwd(xd, wq[q].to(dev), bias, y, act="relu", y_c_offset=off, y_img_stride=4 * H * W * pitch,
                     y_h_stride=4 * W * pitch, y_w_stride=2 * pitch, y_elem_offset=(q // 2 * 2 * W + q % 2) * pitch, force=dict(pair=pair))
    got = y.float().cpu()
    assert bool((got[..., :off] == SENTINEL).all() and (got[..., off + Cout:] == SENTINEL).all()), "wrote outside its slice"
    for q in range(4):
        ref = base.ref_conv(x.float(), wq[q].float(), b, 1, "relu", None, 0.0)
        _check(got[:, q // 2::2, q % 2::2, off:off + Cout], ref, 2.0 ** -8, f"quadrant {q}")


@pytest.mark.parametrize("pair", [1, -1], ids=["cta_pair", "single_cta"])
@pytest.mark.parametrize("ch,act", [(80, "sigmoid"), (4, None), (68, None)], ids=["cls80", "reg4", "dfl68"])
def test_head_f32_level_offsets(ch, act, pair):
    """Three pyramid levels (32x32, 16x16, 8x8; strides 8 / 16 / 32 of a 256 x 256 input) written into one fp32 [N, A, ch]
    tensor at their anchor offsets, as the detection head does; the sentinel checks that no level writes into another."""
    from yolov6_b200 import ops
    N, Cin = 2, 64
    dev = torch.device("cuda:0")
    sizes = [32, 16, 8]
    offs = [0, 32 * 32, 32 * 32 + 16 * 16]
    A = offs[-1] + 8 * 8
    y = torch.full((N, A, ch), SENTINEL, dtype=torch.float32, device=dev)
    refs = []
    for lvl, s in enumerate(sizes):
        x, w, b = _operands(N, s, s, Cin, ch, 1, seed=10 + lvl)
        ops.conv_fwd(x.to(dev), w.to(dev), ops.pad_bias(b.to(dev), ch), y, act=act, y_img_stride=A * ch, y_h_stride=s * ch, y_w_stride=ch,
                     y_elem_offset=offs[lvl] * ch, force=dict(pair=pair))
        refs.append(base.ref_conv(x.float(), w.float(), b, 1, act, None, 0.0).reshape(N, s * s, ch))
    got = y.cpu()
    assert not bool((got == SENTINEL).any()), "an anchor was not written"
    _check(got, torch.cat(refs, 1), 2e-6, f"head ch={ch}")


def test_head_f32_partial_tiles():
    """fp32 output whose 128-row tiles (two 64-row boxes each) are cut by the right and bottom edges."""
    from yolov6_b200 import ops
    N, H, W, Cin, Cout = 3, 20, 12, 64, 80
    dev = torch.device("cuda:0")
    x, w, b = _operands(N, H, W, Cin, Cout, 1, seed=20)
    y = torch.full((N, H, W, Cout), SENTINEL, dtype=torch.float32, device=dev)
    ops.conv_fwd(x.to(dev), w.to(dev), ops.pad_bias(b.to(dev), Cout), y, act="sigmoid", force=dict(bw=16, bh=8))
    _check(y.cpu(), base.ref_conv(x.float(), w.float(), b, 1, "sigmoid", None, 0.0), 2e-6, "fp32 partial tiles")
