"""CPU checks of the training engine's multi-shape plan (TrainEngine.plan_shapes): every shape's launches stay inside the
shared buffers, and those buffers are exactly as large as the largest shape's single plan.  Launches are recorded by the
stand-ins of tests/launch_log.py."""
import types

import pytest
import torch

from launch_log import FakeLib, Recorder
from test_train_plan import dry_engine_of
from yolov6_b200 import _lib
from yolov6_b200.step import TrainStep
from yolov6_b200.train import _Arena

BATCH = 2
# config -> square img_size and the rect canvases planned with it (stride 32 for P5 models, 64 for P6)
CASES = {
    "yolov6n": (640, [(384, 640), (640, 384), (480, 640), (640, 640)]),
    "yolov6s": (640, [(384, 640), (640, 384)]),
    "yolov6m": (320, [(192, 320), (320, 192), (320, 320)]),
    "yolov6l6": (256, [(128, 256), (256, 128), (192, 256)]),
}


def single_plan_bytes(cfg, H, W):
    """Bytes of the per-shape tensors of one fresh single-shape plan, each rounded up as the caching allocator does."""
    eng, _ = dry_engine_of(cfg, 1)
    sizes = []
    new = eng._new

    def counting(shape, dtype=torch.bfloat16, zero=True):
        t = new(shape, dtype, zero)
        sizes.append(t.numel() * t.element_size())
        return t
    eng._new = counting
    eng._plan(BATCH, H, W, torch.float32)
    return sum((n + _Arena.ALIGN - 1) // _Arena.ALIGN * _Arena.ALIGN for n in sizes)


def replay_shape(eng, H, W):
    """Plans (H, W) into the arena and runs one step's launches against the recorder; returns the storages they touched."""
    eng._plan(BATCH, H, W, torch.float32)
    rec = Recorder(eng)
    eng.lib, eng.h, eng._wg_stream = FakeLib(rec), rec.handle, None
    rec.collect_storages()
    firsts, lasts = TrainStep._segments(types.SimpleNamespace(eng=eng))
    with rec.fakes():
        sp = _lib.stream_ptr()
        eng.begin_step(sp)
        eng.run_forward(sp)
        for first, last in zip(firsts, lasts):
            eng.backward(None, None, first=first, last=last)
    return rec


@pytest.mark.parametrize("cfg", list(CASES))
def test_multi_shape_plan_shares_one_arena(cfg):
    size, rects = CASES[cfg]
    shapes = [(size, size)] + rects
    eng, _ = dry_engine_of(cfg, 1)
    eng.plan_shapes(BATCH, shapes, torch.float32)
    arena, x_store = eng.arena.store, eng.x_store
    assert arena.numel() == single_plan_bytes(cfg, size, size)
    for H, W in rects:
        assert single_plan_bytes(cfg, H, W) <= arena.numel()
    shared = {arena.untyped_storage().data_ptr(), x_store.untyped_storage().data_ptr()}
    state = Recorder([eng.flat, eng.wts, eng.zero_arena, eng.stat_out, eng.coef_out, eng.pack_table, eng.grad_tables])
    state.collect_storages()
    fixed = set(state.lo)                   # the shape-independent state: weights, flat buffers, accumulators, xform tables
    for H, W in shapes + rects[:1]:            # and back to a shape planned before
        rec = replay_shape(eng, H, W)
        assert eng.x_static.shape == (BATCH, 3, H, W) and eng.x_static.untyped_storage().data_ptr() in shared
        for t in [*eng.bufs, *eng.gbufs, eng.cls, eng.reg, eng.grad_cls, eng.grad_reg, *eng.scratch.dc, *eng.scratch.dl]:
            assert t.untyped_storage().data_ptr() == arena.untyped_storage().data_ptr()
        assert eng.arena.off <= arena.numel()
        touched = set(rec.ordinal)          # every storage a launch or tensor op of the step pointed into
        assert touched - fixed == shared, f"{cfg} {H}x{W}: launches outside the shared buffers and the model state"


def test_same_shape_replans_at_the_same_addresses():
    eng, _ = dry_engine_of("yolov6n", 1)
    eng.plan_shapes(BATCH, [(320, 320), (192, 320)], torch.float32)
    eng._plan(BATCH, 192, 320, torch.float32)
    first = [t.data_ptr() for t in eng.bufs + eng.gbufs] + [eng.x_static.data_ptr()]
    eng._plan(BATCH, 320, 320, torch.float32)
    eng._plan(BATCH, 192, 320, torch.float32)
    assert [t.data_ptr() for t in eng.bufs + eng.gbufs] + [eng.x_static.data_ptr()] == first
