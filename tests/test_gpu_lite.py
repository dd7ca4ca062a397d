"""YOLOv6Lite on the GPU: the depthwise-conv, squeeze-excite, channel-shuffle and upsample kernels against float64, the
Hardswish epilogues of yv6_conv_fwd / yv6_stem_fwd, and the three Lite models end to end against the reference goldens
(tests/golden/make_golden_lite.py), captured into a CUDA graph, through DetectPipeline and from a saved checkpoint."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import golden_npz
from oracle import fabricate as fab
from test_model_lite import NAMES, lite_keys, rel_err
from yolov6_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _buffer(N, H, W, pitch, nsplit, gen):
    """Random activations as the engine stores them: bf16 [N,H,W,pitch] or three planes [3,N,H,W,pitch]; returns (buffer,
    float64 values it represents)."""
    v = torch.randn(N, H, W, pitch, generator=gen, dtype=torch.float64)
    if nsplit == 3:
        buf = ops.split3(v.float()).to(DEV)
        return buf, buf.double().sum(0).cpu()
    buf = v.to(torch.bfloat16).to(DEV)
    return buf, buf.double().cpu()


def _values(buf, nsplit):
    return (buf.double().sum(0) if nsplit == 3 else buf.double()).cpu()


def _tol(nsplit):
    return 1e-5 if nsplit == 3 else 8e-3          # 3 planes: fp32-equivalent; bf16: one output rounding (2^-8) plus inputs


# (C, x pitch, x channel offset, y pitch, y channel offset): vector paths, odd channel counts, unaligned offsets, pitch > C
SLICES = [(8, 16, 0, 8, 0), (12, 32, 4, 24, 10), (44, 64, 8, 48, 0), (24, 24, 0, 64, 24)]


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("act", [None, "hardswish"])
@pytest.mark.parametrize("nsplit", [1, 3])
def test_depthwise_conv_matches_float64(k, s, act, nsplit):
    gen = torch.Generator().manual_seed(k * 100 + s * 10 + nsplit)
    N, H, W = 2, 13, 22
    for C_, xp, xo, yp, yo in SLICES:
        x, xv = _buffer(N, H, W, xp, nsplit, gen)
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        w = torch.randn(C_, 1, k, k, generator=gen, dtype=torch.float64) / k
        b = torch.randn(C_, generator=gen, dtype=torch.float64) * 0.1
        y, yv0 = _buffer(N, Ho, Wo, yp, nsplit, gen)
        wd = w[:, 0].permute(1, 2, 0).reshape(k * k, C_).float().contiguous().to(DEV)
        ops.dwconv_fwd(x, wd, b.float().to(DEV), y, k=k, stride=s, act=act, x_c_offset=xo, y_c_offset=yo, nsplit=nsplit)
        torch.cuda.synchronize()
        ref = F.conv2d(xv[..., xo:xo + C_].permute(0, 3, 1, 2), w.float().double(), b.float().double(), s, k // 2, 1, C_)
        ref = (F.hardswish(ref) if act else ref).permute(0, 2, 3, 1)
        got = _values(y, nsplit)
        assert rel_err(got[..., yo:yo + C_].numpy(), ref.numpy()) < _tol(nsplit), (C_, xo, yo)
        keep = torch.ones(yp, dtype=torch.bool)
        keep[yo:yo + C_] = False
        assert torch.equal(got[..., keep], yv0[..., keep]), "channels outside the slice were written"


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("C_,HW", [(8, (40, 40)), (12, (20, 20)), (44, (10, 7)), (96, (5, 5)), (192, (10, 10))])
def test_squeeze_excite_matches_float64_and_is_deterministic(C_, HW, nsplit):
    gen = torch.Generator().manual_seed(C_ + nsplit)
    N, (H, W), pitch, off = 3, HW, C_ + 16, 8
    x, xv = _buffer(N, H, W, pitch, nsplit, gen)
    cr = C_ // 4
    w1, b1 = torch.randn(cr, C_, generator=gen, dtype=torch.float64) / C_ ** 0.5, torch.randn(cr, generator=gen, dtype=torch.float64) * 0.1
    w2, b2 = torch.randn(C_, cr, generator=gen, dtype=torch.float64) / cr ** 0.5, torch.randn(C_, generator=gen, dtype=torch.float64) * 0.1
    dw = [t.float().contiguous().to(DEV) for t in (w1, b1, w2, b2)]
    x0 = x.clone()
    ops.se_fwd(x, *dw, c_offset=off, nsplit=nsplit)
    ops.se_fwd(x0, *dw, c_offset=off, nsplit=nsplit)
    torch.cuda.synchronize()
    assert torch.equal(x, x0), "two runs differ"
    t = xv[..., off:off + C_]
    w1, b1, w2, b2 = (v.float().double() for v in (w1, b1, w2, b2))
    s = F.hardsigmoid(torch.relu(t.mean((1, 2)) @ w1.t() + b1) @ w2.t() + b2)
    got = _values(x, nsplit)
    assert rel_err(got[..., off:off + C_].numpy(), (t * s[:, None, None]).numpy()) < _tol(nsplit)
    assert torch.equal(got[..., :off], xv[..., :off]) and torch.equal(got[..., off + C_:], xv[..., off + C_:])


@pytest.mark.parametrize("nsplit", [1, 3])
def test_shuffle_and_upsample_copy_exactly(nsplit):
    gen = torch.Generator().manual_seed(5)
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    N, H, W, c = 2, 6, 5, 22
    a, av = _buffer(N, H, W, 48, nsplit, gen)
    b, bv = _buffer(N, H, W, 32, nsplit, gen)
    y = torch.zeros_like(_buffer(N, H, W, 64, nsplit, gen)[0])
    pl = lambda t: t.stride(0) if nsplit == 3 else 0      # noqa: E731
    _lib.check(lib.yv6_channel_shuffle(h, a.data_ptr() + 2 * 24, 48, pl(a), b.data_ptr() + 2 * 8, 32, pl(b), N * H * W, c,
                                       y.data_ptr() + 2 * 16, 64, pl(y), nsplit, sp))
    u = torch.zeros_like(_buffer(N, 2 * H, 2 * W, 32, nsplit, gen)[0])
    _lib.check(lib.yv6_upsample2x(h, a.data_ptr() + 2 * 8, 48, pl(a), N, H, W, c, u.data_ptr() + 2 * 4, 32, pl(u), nsplit, sp))
    torch.cuda.synchronize()
    want = torch.zeros(N, H, W, 64, dtype=torch.float64)
    want[..., 16:16 + 2 * c:2], want[..., 17:17 + 2 * c:2] = av[..., 24:24 + c], bv[..., 8:8 + c]
    assert torch.equal(_values(y, nsplit), want)
    up = F.interpolate(av[..., 8:8 + c].permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    got = _values(u, nsplit)
    assert torch.equal(got[..., 4:4 + c], up) and float(got[..., :4].abs().max()) == 0 and float(got[..., 4 + c:].abs().max()) == 0


@pytest.mark.parametrize("nsplit", [1, 3])
def test_hardswish_epilogues_of_conv_and_stem(nsplit):
    gen = torch.Generator().manual_seed(7)
    x, xv = _buffer(2, 12, 20, 48, nsplit, gen)
    w = torch.randn(40, 1, 1, 32, generator=gen, dtype=torch.float64) * 0.5
    b = torch.randn(40, generator=gen, dtype=torch.float64)
    wd = ops.split3(w.float()).to(DEV) if nsplit == 3 else w.to(torch.bfloat16).to(DEV)
    wv = wd.double().sum(0).cpu() if nsplit == 3 else wd.double().cpu()
    y = torch.zeros_like(_buffer(2, 12, 20, 48, nsplit, gen)[0])
    ops.conv_fwd(x, wd, ops.pad_bias(b.float().to(DEV), 40), y, x_c_offset=16, act="hardswish", nsplit=nsplit)
    torch.cuda.synchronize()
    ref = F.hardswish(torch.einsum("nhwc,oc->nhwo", xv[..., 16:48], wv[:, 0, 0]) + b.float().double())
    assert rel_err(_values(y, nsplit)[..., :40].numpy(), ref.numpy()) < _tol(nsplit)

    img = torch.rand(2, 3, 64, 96, generator=gen)
    ws = torch.randn(32, 3, 3, 3, generator=gen) * 0.5
    bs = torch.randn(32, generator=gen)
    y = torch.zeros((3, 2, 32, 48, 32) if nsplit == 3 else (2, 32, 48, 32), dtype=torch.bfloat16, device=DEV)
    xi, wdev, bdev = img.to(DEV), ws.permute(2, 3, 1, 0).contiguous().to(DEV), bs.to(DEV)
    d = ops.stem_desc(xi.data_ptr(), 2, 64, 96, False, wdev.data_ptr(), bdev.data_ptr(), 32, "hardswish", y.data_ptr(), nsplit,
                      y.stride(0) if nsplit == 3 else 0)
    _lib.check(_lib.lib().yv6_stem_fwd(_lib.handle(0), C.byref(d), _lib.stream_ptr()))
    torch.cuda.synchronize()
    ref = F.hardswish(F.conv2d(img.double(), ws.double(), bs.double(), 2, 1)).permute(0, 2, 3, 1)
    tol = 1e-5 if nsplit == 3 else 3e-2      # the bf16 stem takes bf16 image / weights on tensor cores
    assert rel_err(_values(y, nsplit).numpy(), ref.numpy()) < tol


def load(name, precision):
    from yolov6_b200.model import build_model
    m = build_model(name, 80, DEV)
    m.load_state_dict(fab.fabricate_state_dict(lite_keys(name), seed=0), strict=True)
    return m.eval().set_precision(precision)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_eval_matches_reference_golden(name, precision):
    m = load(name, precision)
    x = fab.synthetic_images(2, 128, 128, seed=0)
    g = golden_npz(f"model_{name}.npz")
    with torch.no_grad():
        out, feats = m(x.cuda())
        cls, reg = m.engine().head_outputs(2, 128, 128)
    e_out, e_cls, e_reg = rel_err(out.cpu().numpy(), g["eval_out"]), rel_err(cls.cpu().numpy(), g["cls_train"]), rel_err(reg.cpu().numpy(), g["reg_train"])
    print(f"{name} {precision}-mode: out {e_out:.2e} cls {e_cls:.2e} reg {e_reg:.2e}")
    tol = 1e-4 if precision == "fp32" else 6e-2
    assert e_out < tol and e_cls < tol and e_reg < tol
    assert [tuple(f.shape) for f in feats] == [(2, 96, 16, 16), (2, 96, 8, 8), (2, 96, 4, 4), (2, 96, 2, 2)]


@pytest.mark.parametrize("name,B,H,W,step", [("yolov6lite_s", 4, 320, 320, 16), ("yolov6lite_l", 2, 192, 320, 16)])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_forward_at_native_size_matches_reference(name, B, H, W, step, precision):
    g = golden_npz("configs_lite.npz")
    x = fab.synthetic_images(B, H, W, seed=40)
    m = load(name, precision)
    with torch.no_grad():
        out = m(x.cuda())[0].cpu().double().numpy()
    A = out.shape[1]
    e_rows = rel_err(out[:, ::step], g[f"{name}_rows"].astype(np.float64))
    e_sum = float((np.abs(out.sum(1) - g[f"{name}_colsum"]) / (A + g[f"{name}_abs_colsum"])).max())
    print(f"{name}@{H}x{W} {precision}: sampled rows {e_rows:.2e}, column sums {e_sum:.2e}")
    tol = 1e-4 if precision == "fp32" else 6e-2
    assert e_rows < tol and e_sum < tol


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_captured_graph_replays_the_eager_forward_bit_for_bit(precision):
    m = load("yolov6lite_m", precision)
    eng = m.engine()
    x = fab.synthetic_images(4, 192, 320, seed=1).cuda()
    eng.pin(4, 192, 320)
    with torch.no_grad():
        eager = eng.forward(x).clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eng.forward(x)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = eng.forward(x)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert eng.launch_count(4, 192, 320) == len(eng.launches(4, 192, 320)) + 1


def test_detect_pipeline_matches_eager_model_plus_nms():
    from yolov6_b200.nms import non_max_suppression
    from yolov6_b200.pipeline import DetectPipeline
    m = load("yolov6lite_s", "bf16")
    B, S = 3, 320
    kw = dict(conf_thres=0.25, iou_thres=0.45, max_det=300)
    pipe = DetectPipeline(m, B, S, S, host_input=True, **kw)
    g = torch.Generator().manual_seed(9)
    n = 0
    for _ in range(2):
        img = (torch.rand(B, 3, S, S, generator=g) * 255).to(torch.uint8)
        dets = pipe(img)
        with torch.no_grad():
            ref = non_max_suppression(m(img.to(DEV))[0], **kw)
        assert len(dets) == B
        for d, r in zip(dets, ref):
            assert torch.equal(d.cpu(), r.cpu())
            n += d.shape[0]
    assert n > 0


@pytest.mark.parametrize("name", NAMES)
def test_load_checkpoint_of_a_saved_state_dict_runs(name, tmp_path):
    from yolov6_b200.checkpoint import load_checkpoint
    path = tmp_path / f"{name}.pt"
    torch.save({"model": fab.fabricate_state_dict(lite_keys(name), seed=0)}, path)
    m = load_checkpoint(str(path), map_location="cpu").to(DEV).set_precision("fp32")
    x = fab.synthetic_images(2, 128, 128, seed=0)
    with torch.no_grad():
        out = m(x.cuda())[0].cpu().numpy()
    assert rel_err(out, golden_npz(f"model_{name}.npz")["eval_out"]) < 1e-4
