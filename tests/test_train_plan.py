"""CPU replay of the training engine's step (train.py): every library call, tensor copy / clear, stream and event of
`begin_step`, `run_forward` and a `backward` cut into the segments TrainStep captures, recorded against stand-ins for the
library and for torch's CUDA streams and events, and compared with a fixture (tests/golden/train_plan.json.gz, written by
tests/golden/make_golden_train_plan.py).  How calls are recorded: tests/launch_log.py."""
import json
import os
import types

import pytest
import torch

from launch_log import FakeLib, Recorder, dump, first_difference, load  # noqa: F401  (dump: make_golden_train_plan.py)
from yolov6_b200 import _lib, configs
from yolov6_b200.model import build_model
from yolov6_b200.step import TrainStep
from yolov6_b200.train import TrainEngine

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_plan.json.gz")
BATCH, N_BUCKETS = 2, 3
# name -> config, model options, image size, input dtype, neck outputs as differentiable outputs, second step with accumulate=True
CASES = {
    "yolov6n": dict(cfg="yolov6n", accumulate_step=True),
    "yolov6n_u8": dict(cfg="yolov6n", dtype=torch.uint8),
    "yolov6m": dict(cfg="yolov6m"),
    "yolov6l6_128": dict(cfg="yolov6l6", size=128),
    "yolov6s_mbla": dict(cfg="yolov6s_mbla"),
    "yolov6n_qa": dict(cfg="yolov6n_qa"),
    "yolov6m_qa": dict(cfg="yolov6m_qa"),
    "yolov6n_fuse_ab": dict(cfg="yolov6n", fuse_ab=True),
    "yolov6n_distill_ns": dict(cfg="yolov6n", distill_ns=True, external_feat_grads=True),
}


def dry_engine(case):
    """A TrainEngine over a CPU model whose library, handle and streams are the recorder's stand-ins."""
    c = CASES[case]
    return dry_engine_of(c["cfg"], N_BUCKETS, fuse_ab=c.get("fuse_ab", False), distill_ns=c.get("distill_ns", False),
                         external_feat_grads=bool(c.get("external_feat_grads")))


def dry_engine_of(cfg_name, n_buckets, fuse_ab=False, distill_ns=False, external_feat_grads=False):
    cfg = configs.get_config(cfg_name)
    if distill_ns:                # the N / S distillation student needs the DFL head
        cfg["head"]["use_dfl"], cfg["head"]["reg_max"] = True, 16
    m = build_model(cfg, 80, torch.device("cpu"), fuse_ab=fuse_ab, distill_ns=distill_ns).train()
    eng = TrainEngine.__new__(TrainEngine)
    eng.model, eng.g, eng.dev = m, m.graph, torch.device("cpu")
    eng.n_buckets = n_buckets
    eng.debug, eng.dbg, eng._shape, eng.bucket_hook = False, {}, None, None
    eng.overlap_wgrad, eng._wg_stream = True, None
    eng.external_feat_grads, eng._feat_grads = external_feat_grads, None
    eng._build_state()
    rec = Recorder(eng)
    eng.lib, eng.h = FakeLib(rec), rec.handle
    return eng, rec


def replay(case):
    c = CASES[case]
    eng, rec = dry_engine(case)
    size = c.get("size", 64)
    eng._plan(BATCH, size, size, c.get("dtype", torch.float32))
    rec.collect_storages()
    firsts, lasts = TrainStep._segments(types.SimpleNamespace(eng=eng))
    steps = [False, True] if c.get("accumulate_step") else [False]
    with rec.fakes():
        for accumulate in steps:
            eng.debug = accumulate            # the second step also snapshots every op's incoming gradient
            sp = _lib.stream_ptr()
            rec.log.append({"fn": "step", "accumulate": accumulate})
            eng.begin_step(sp)
            eng.run_forward(sp)
            for first, last in zip(firsts, lasts):
                rec.log.append({"fn": "segment"})
                eng.backward(None, None, accumulate=accumulate, first=first, last=last)
    zero = [rec.ptr(t.data_ptr(), "zero_gbufs") for t in eng.zero_gbufs]
    return {"log": rec.log, "launch_counts": list(eng.launch_counts()), "zero_gbufs": zero, "streams": len(rec.streams),
            "events": len(rec.events), "debug_ops": sorted(eng.dbg)}


@pytest.fixture(scope="module")
def fixture():
    return load(FIXTURE)


@pytest.mark.parametrize("case", list(CASES))
def test_training_step_replays_the_pinned_launches(case, fixture):
    want, got = fixture[case], json.loads(json.dumps(replay(case)))
    for key in ("launch_counts", "zero_gbufs", "streams", "events", "debug_ops"):
        assert got[key] == want[key], f"{case}: {key}: want {want[key]}, got {got[key]}"
    first_difference(case, want["log"], got["log"])
