"""CPU replay of the inference engine's forward (engine.py): every library call, tensor copy / clear, stream, event record and
event wait of a decoded forward, of the serving pipeline's forward (no decode, head set 1, a hook at the fork index) and of a
decoded forward that switches the head set back, recorded against stand-ins for the library and for torch's CUDA streams and
events (tests/launch_log.py), and compared with a fixture (tests/golden/infer_plan.json.gz, written by
tests/golden/make_golden_infer_plan.py).  Also pins launch_count, conv_bytes_per_launch, profile_convs' (FLOPs, launches) and
the (kind, name) rows of profile_calls, whose timings are zero here.

The conv tile planner runs on the host (yv6_conv_plan_host) with the H100 SXM's properties of tests/test_conv_planner.py: it
decides where the column-pair view of the 64- and 128-channel stride-2 convs is kept."""
import contextlib
import ctypes as C
import json
import os

import pytest
import torch

from launch_log import FakeLib, Recorder, dump, first_difference, load  # noqa: F401  (dump: make_golden_infer_plan.py)
from yolov6_b200 import _lib, configs, ops
from yolov6_b200.engine import InferEngine
from yolov6_b200.model import build_model
from yolov6_b200.synth import randomize_

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "infer_plan.json.gz")
BATCH = 2
H100 = (132, 232448, 66)
# name -> config, model options, precision, image size (H, W), input dtype, launch lanes
CASES = {
    "yolov6n": dict(cfg="yolov6n"),
    "yolov6n_u8": dict(cfg="yolov6n", dtype=torch.uint8),
    "yolov6s_fp32": dict(cfg="yolov6s", precision="fp32"),
    "yolov6s_one_lane": dict(cfg="yolov6s", lanes=1),
    "yolov6m": dict(cfg="yolov6m"),
    "yolov6l6_128": dict(cfg="yolov6l6", size=(128, 128)),
    "yolov6s_mbla": dict(cfg="yolov6s_mbla"),
    "yolov6n_qa": dict(cfg="yolov6n_qa"),
    "yolov6lite_s_128": dict(cfg="yolov6lite_s", size=(128, 128)),
    "yolov6lite_l_192x320": dict(cfg="yolov6lite_l", size=(192, 320)),
    "yolov6n_fuse_ab": dict(cfg="yolov6n", fuse_ab=True),
    "yolov6n_distill_ns": dict(cfg="yolov6n", distill_ns=True),
}


def host_plan(d, device=0):
    out = (C.c_int32 * 12)()
    rc = _lib.lib().yv6_conv_plan_host(*H100, C.byref(d), out)
    assert rc == 0, _lib.lib().yv6_last_error().decode()
    return dict(zip(ops.PLAN_KEYS, out))


@contextlib.contextmanager
def host_planner():
    saved, ops.plan_of = ops.plan_of, host_plan
    try:
        yield
    finally:
        ops.plan_of = saved


def dry_engine(case):
    """An InferEngine over a CPU model with seeded weights whose library, handle and streams are the recorder's stand-ins.
    `case` names one of CASES or is a dict of the same form (tests/test_serving_plan.py)."""
    c = CASES[case] if isinstance(case, str) else case
    cfg = configs.get_config(c["cfg"])
    if c.get("distill_ns"):       # the N / S distillation student needs the DFL head
        cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
    m = build_model(cfg, 80, torch.device("cpu"), fuse_ab=c.get("fuse_ab", False), distill_ns=c.get("distill_ns", False))
    m = randomize_(m, seed=0).eval()
    precision = c.get("precision", "bf16")
    eng = InferEngine.__new__(InferEngine)
    eng.g, eng.device, eng.precision = m.graph, torch.device("cpu"), precision
    eng.nsplit = 3 if precision == "fp32" else 1
    eng.n_lanes, eng._side = c.get("lanes", 4), None
    eng.weights, eng._plans, eng.max_plans, eng._pinned = {}, {}, 4, set()
    eng._pack(m.state_dict())
    rec = Recorder(eng)
    eng.lib, eng.handle = FakeLib(rec), rec.handle
    return eng, rec


def replay(case):
    c = CASES[case]
    eng, rec = dry_engine(case)
    H, W = c.get("size", (64, 64))
    dtype = c.get("dtype", torch.float32)
    x = torch.zeros(BATCH, 3, H, W, dtype=dtype)
    with host_planner(), rec.fakes():
        eng.head_outputs(BATCH, H, W, dtype, head_set=1)     # allocates the alternate head set, so that its pointers are known
        fork = eng.neck_start(BATCH, H, W, dtype)
        rec.collect_storages(x)
        rec.log.append({"fn": "forward"})
        eng.forward(x)
        rec.log.append({"fn": "forward", "decode": False, "head_set": 1})
        eng.forward(x, decode=False, head_set=1, hook=(fork, lambda: rec.log.append({"fn": "hook"})))
        rec.log.append({"fn": "forward"})
        eng.forward(x)
        log, streams, events = list(rec.log), len(rec.streams), len(rec.events)
        out = {"log": log, "streams": streams, "events": events, "fork": fork}
        if dtype == torch.float32:
            _, flops, n_conv = eng.profile_convs(x, steps=1)
            out.update(launch_count=eng.launch_count(BATCH, H, W), conv_bytes_per_launch=eng.conv_bytes_per_launch(BATCH, H, W),
                       profile_convs=[flops, n_conv], profile_calls=[[kind, name] for kind, name, _ in eng.profile_calls(x, steps=1)])
    return out


@pytest.fixture(scope="module")
def fixture():
    return load(FIXTURE)


@pytest.mark.parametrize("case", list(CASES))
def test_inference_forward_replays_the_pinned_launches(case, fixture):
    want, got = fixture[case], json.loads(json.dumps(replay(case)))
    for key in sorted((set(want) | set(got)) - {"log"}):
        assert got.get(key) == want.get(key), f"{case}: {key}: want {want.get(key)}, got {got.get(key)}"
    first_difference(case, want["log"], got["log"])
