"""The fp16 inference precision mode on the GPU (model.set_precision("fp16")).

1. Every forward launch alone, at the engine's own descriptors, against float64 computed on the same fp16 operands: the
   harness of tests/test_gpu_forward_launches.py (sentinel-filled buffers, declared read / write spans, per-element bars),
   run with fp16 as the 16-bit dtype.  Its bars then hold one fp16 rounding, 2^-11 of the value, on top of the fp32
   accumulation term (1e-5 of the sum of absolute products) and the fp32 epilogue; fp16 outputs take the accurate SiLU
   (no tanh.approx term), the max-pool, shuffle and upsample are bit for bit.  Below 2^-14 fp16 is subnormal, so every bar
   also allows 2^-25 absolute.  The sentinel is 2^14, finite in fp16.  The
   conv forms the engine never plans (CTA pairs, forced tiles) are checked directly against float64 as well.
2. All 18 built-in detectors with seeded weights and input: finite head outputs, and a max deviation from the
   fp32-equivalent mode of at most 1/4 of the bf16 mode's (fp16 keeps 3 more mantissa bits: ~1/8 expected).
3. DetectPipeline and DetectFarm in fp16 return exactly what model(x) + non_max_suppression return in fp16.
4. A model switched to fp16 and back gives the bf16 output bit for bit.
"""
import pytest
import torch

import test_gpu_backward_launches as bwd
import test_gpu_forward_launches as fl

pytestmark = pytest.mark.gpu

F16 = torch.float16
F16_ULP = 2.0 ** -11
F16_SUBNORMAL = 2.0 ** -25     # half the spacing of fp16's subnormals (below 2^-14 the 2^-11 relative bound does not hold)
NAMES = ("yolov6n", "yolov6s", "yolov6m", "yolov6l", "yolov6n6", "yolov6s6", "yolov6m6", "yolov6l6", "yolov6s_mbla", "yolov6m_mbla",
         "yolov6l_mbla", "yolov6x_mbla", "yolov6n_qa", "yolov6s_qa", "yolov6m_qa", "yolov6lite_s", "yolov6lite_m", "yolov6lite_l")
# the benchmarked shapes of tests/test_gpu_forward_launches.py: name -> model config, batch, input height, width, uint8 input
CONFIGS = {
    "yolov6s_640_b32": dict(cfg="yolov6s", N=32, H=640, W=640),
    "yolov6n_384x640_b8_u8": dict(cfg="yolov6n", N=8, H=384, W=640, u8=True),
    "yolov6m_640_b2": dict(cfg="yolov6m", N=2, H=640, W=640),
    "yolov6l6_1280_b2": dict(cfg="yolov6l6", N=2, H=1280, W=1280),
    "yolov6s_mbla_256_b2": dict(cfg="yolov6s_mbla", N=2, H=256, W=256),
    "yolov6lite_s_128": dict(cfg="yolov6lite_s", N=2, H=128, W=128),
    "yolov6lite_l_192x320": dict(cfg="yolov6lite_l", N=2, H=192, W=320),
}


@pytest.fixture
def fp16_harness(monkeypatch):
    """tests/test_gpu_forward_launches.py with fp16 as its 16-bit activation dtype (restored after the test)."""
    monkeypatch.setattr(fl, "BF16", F16)
    monkeypatch.setattr(fl, "BF16_ULP", F16_ULP)
    monkeypatch.setattr(fl, "SENTINEL", 2.0 ** 14)
    monkeypatch.setattr(fl, "TANH_APPROX", 0.0)          # fp16 outputs take the ex2 / rcp SiLU
    monkeypatch.setattr(fl.Ctx.planes, "__defaults__", (F16,))
    ratio = bwd.ratio                                     # fp16 subnormals: one rounding is off by up to 2^-25 absolute
    monkeypatch.setattr(bwd, "ratio", lambda got, ref, bar: ratio(got, ref, bar + F16_SUBNORMAL))
    return fl


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_fp16_launch_record_matches_float64(config, fp16_harness):
    c = CONFIGS[config]
    m, eng = fl.build_engine(c["cfg"], "fp16")
    ctx = fl.Ctx(eng, c["N"], c["H"], c["W"], c.get("u8", False))
    assert all(t.dtype == F16 for t in ctx.plan.bufs)
    gen = torch.Generator(device="cuda").manual_seed(20261017)
    seen, worst = set(), {}
    for r in ctx.plan.launches:
        sig = fl.launch_signature(ctx, r)
        if sig in seen:
            continue
        seen.add(sig)
        if r.kind == "conv":
            assert r.desc.reserved0 == 3 and r.desc.y_dtype in (1, 3), r.name
        ratio = fl.check_launch(ctx, r, gen)
        assert ratio <= 1.0, f"{config}: {r.kind} {r.name}: error {ratio:.3f} x the bar"
        key = fl.conv_form(r) if r.kind == "conv" else r.kind
        worst[key] = max(worst.get(key, 0.0), ratio)
    print(f"\n{config} fp16: {len(seen)} distinct launches, worst error / bar: "
          + ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst.items())))
    del ctx, eng, m
    torch.cuda.empty_cache()


# (N, H, W, Cin, Cout, k, stride, force, residual, fp32 output): the mainloops and epilogues, CTA pairs included
DIRECT = [
    (2, 40, 40, 64, 128, 3, 1, {}, False, False),
    (2, 40, 40, 64, 128, 3, 1, {"pair": 1}, True, False),
    (2, 40, 40, 128, 64, 3, 1, {"halo": 1}, False, False),
    (2, 40, 40, 128, 64, 3, 1, {"halo": 1, "pair": 1}, False, True),
    (2, 40, 40, 64, 96, 3, 1, {"halo": -1}, True, False),
    (2, 36, 52, 32, 64, 3, 2, {}, False, False),
    (4, 20, 20, 256, 128, 1, 1, {"pair": 1}, True, False),
    (4, 20, 20, 256, 80, 1, 1, {}, False, True),
    (1, 24, 24, 16, 32, 1, 1, {"bn": 32}, False, False),
    (2, 17, 23, 128, 128, 3, 1, {"bw": 8, "bh": 8, "stages": 3}, False, False),
]


@pytest.mark.parametrize("case", DIRECT)
def test_fp16_conv_forms_match_float64(case):
    from yolov6_b200 import ops
    N, H, W, Cin, Cout, k, s, force, use_res, y_f32 = case
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(hash(case[:7]) % (1 << 31))
    x = torch.randn(N, H, W, Cin, generator=g).to(F16)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5).to(F16)
    b = torch.randn(Cout, generator=g)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    res = torch.randn(N, Ho, Wo, Cout, generator=g).to(F16) if use_res else None
    for act in ("silu", "relu", None):
        y = torch.zeros(N, Ho, Wo, Cout, dtype=torch.float32 if y_f32 else F16, device=dev)
        ops.conv_fwd(x.to(dev), w.to(dev), ops.pad_bias(b.to(dev), Cout), y, stride=s, act=act, force=force,
                     res=None if res is None else res.to(dev), alpha=0.5)
        code = {None: fl.ACT_NONE, "relu": fl.ACT_RELU, "silu": fl.ACT_SILU}[act]
        ref, R, z = fl.conv_ref(x.to(dev), w.to(dev), b.to(dev), s, k // 2, code, None if res is None else res.to(dev), 0.5)
        acc = fl.SLOPE[code] * fl.F32_SUM * R + fl.EPI32 * (4 + z.abs()) * ref.abs()
        if res is not None:
            acc = acc + fl.EPS32 * (0.5 * res.to(dev).double()).abs()
        bar = acc if y_f32 else acc + F16_ULP * (ref.abs() + acc)
        ratio = bwd.ratio(y.double(), ref, bar)
        assert ratio <= 1.0, f"{case} {act}: error {ratio:.3f} x the bar"


def _heads(m, x, precision):
    m.set_precision(precision)
    with torch.no_grad():
        cls, reg, _ = m.engine().forward(x, decode=False)
    return cls.clone(), reg.clone()


@pytest.mark.parametrize("name", NAMES)
def test_fp16_deviation_from_fp32_is_at_most_a_quarter_of_bf16s(name):
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = randomize_(build_model(name, 80, dev), seed=0).eval()
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(1)).to(dev)
    ref = _heads(m, x, "fp32")
    dev_of = {}
    for p in ("bf16", "fp16"):
        got = _heads(m, x, p)
        assert all(bool(torch.isfinite(t).all()) for t in got), f"{name} {p}: non-finite head outputs"
        dev_of[p] = max(float(((a - b).abs() / (1 + b.abs())).max()) for a, b in zip(got, ref))
    print(f"\n{name}: max deviation from fp32: bf16 {dev_of['bf16']:.3e}, fp16 {dev_of['fp16']:.3e} "
          f"(ratio {dev_of['fp16'] / max(dev_of['bf16'], 1e-30):.3f})")
    assert dev_of["fp16"] <= 0.25 * dev_of["bf16"], dev_of


KW = dict(conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300)


def test_fp16_detect_pipeline_matches_eager_model_plus_nms():
    from yolov6_b200.model import build_model
    from yolov6_b200.nms import non_max_suppression
    from yolov6_b200.pipeline import DetectPipeline
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = randomize_(build_model("yolov6n", 80, dev), seed=3).eval().set_precision("fp16")
    B, S = 3, 192
    pipe = DetectPipeline(m, B, S, S, host_input=True, **KW)
    g = torch.Generator().manual_seed(9)
    for _ in range(2):
        img = (torch.rand(B, 3, S, S, generator=g) * 255).to(torch.uint8)
        dets = pipe(img)
        with torch.no_grad():
            ref = non_max_suppression(m(img.to(dev))[0], **KW)
        assert sum(len(d) for d in dets) > 0
        for d, r in zip(dets, ref):
            assert torch.equal(d, r.cpu())


def test_fp16_detect_farm_matches_eager_model_plus_nms():
    from yolov6_b200.model import build_model
    from yolov6_b200.nms import non_max_suppression
    from yolov6_b200.pipeline import DetectFarm
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    m = randomize_(build_model("yolov6lite_s", 80, dev), seed=5).eval().set_precision("fp16")
    B, S = 2, 192
    farm = DetectFarm(m, B, S, S, lanes=2, host_input=True, **KW)
    g = torch.Generator().manual_seed(11)
    imgs = [(torch.rand(B, 3, S, S, generator=g) * 255).to(torch.uint8) for _ in range(6)]
    outs, nxt = {}, [0, 1]
    for j, x in enumerate(imgs):
        farm.submit(x)
        r = farm.lanes[j % 2].collect()
        if r is not None:
            outs[nxt[j % 2]] = r
            nxt[j % 2] += 2
    for ln, lane in enumerate(farm.lanes):
        with torch.cuda.stream(farm.streams[ln]):
            lane.drain()
        torch.cuda.synchronize()
        outs[nxt[ln]] = lane.collect()
    assert sorted(outs) == list(range(len(imgs)))
    total = 0
    for j, x in enumerate(imgs):
        with torch.no_grad():
            ref = non_max_suppression(m(x.to(dev))[0], **KW)
        for d, r in zip(outs[j], ref):
            total += len(r)
            assert torch.equal(d, r.cpu())
    assert total > 0


def test_switching_to_fp16_and_back_leaves_bf16_unchanged():
    from yolov6_b200.model import build_model
    from yolov6_b200.synth import randomize_
    dev = torch.device("cuda:0")
    x = torch.rand(2, 3, 192, 192, generator=torch.Generator().manual_seed(2)).to(dev)
    a = randomize_(build_model("yolov6s", 80, dev), seed=4).eval()
    b = randomize_(build_model("yolov6s", 80, dev), seed=4).eval()
    with torch.no_grad():
        ya = a(x)[0]
        b.set_precision("fp16")
        y16 = b(x)[0]
        b.set_precision("bf16")
        yb = b(x)[0]
    assert torch.isfinite(y16).all() and not torch.equal(y16, ya)
    assert torch.equal(ya.view(torch.int32), yb.view(torch.int32))
