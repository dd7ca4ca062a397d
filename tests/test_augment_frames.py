"""CPU checks of training from frames in GPU memory: the FrameCache arena (load sizes, offsets, exact byte count) for the
square, specific and rect targets, the record and first-pass job AugmentFeed builds for a device frame, and the C
declaration of yv6_aug_resize_frames against its ctypes binding and the yv6_lb_src mirror.  Device frames are stood in
for by meta tensors, which carry sizes, strides and a device but no memory."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from yolov6_b200 import _lib
from yolov6_b200.augment import (HYP_YOLOV6S, JOB, FrameCache, Sampler, as_source, batch_tables, cache_layout,
                                 frame_records, resized_shape)
from yolov6_b200.preprocess import REC, check_frame

META = torch.device("meta")
SHAPES = [(480, 640), (640, 480), (333, 517), (1, 1), (17, 1000), (720, 1280), (640, 640), (200, 30)]


@pytest.mark.parametrize("target,H,W", [(None, 640, 640), ("specific", 384, 640), ("specific", 640, 384), ("rect", 640, 640)])
def test_cache_layout_is_exact(target, H, W):
    s = Sampler(len(SHAPES), H, W, HYP_YOLOV6S, 640, target)
    loaded, offsets, nbytes = cache_layout(SHAPES, s)
    want = [resized_shape(h0, w0, 640, (H, W) if target == "specific" else None) for h0, w0 in SHAPES]
    assert [tuple(r) for r in loaded.tolist()] == want
    size = [h * w * 3 for h, w in want]
    assert offsets.tolist() == np.concatenate([[0], np.cumsum(size)[:-1]]).tolist()
    assert nbytes == sum(size)
    if target == "specific":
        assert loaded[5].tolist() == [int(720 * min(W / 1280, H / 720)), int(1280 * min(W / 1280, H / 720))]
    else:
        assert loaded[5].tolist() == [360, 640] and loaded[6].tolist() == [640, 640]       # ratio 1: as decoded


def test_cache_over_max_bytes_raises_with_the_count():
    s = Sampler(len(SHAPES), 640, 640, HYP_YOLOV6S)
    nbytes = cache_layout(SHAPES, s)[2]
    with pytest.raises(RuntimeError, match=f"need {nbytes} bytes"):
        FrameCache(SHAPES, s, nbytes - 1)
    with pytest.raises(RuntimeError, match="shapes"):
        FrameCache(SHAPES[:-1], s, nbytes)


def test_geometry_names_what_decides_the_load_size():
    assert Sampler(10, 640, 640, HYP_YOLOV6S).geometry() == (10, None, 640, None)
    assert Sampler(10, 640, 640, HYP_YOLOV6S, target="rect").geometry() == (10, "rect", 640, None)
    assert Sampler(10, 384, 640, HYP_YOLOV6S, target="specific").geometry() == (10, "specific", 640, (384, 640))


def letterbox_plan(sampler, indices):
    import random
    random.seed(0)
    np.random.seed(0)
    return sampler.draw(indices)


def test_device_source_record_and_first_pass_job():
    """A CUDA frame is addressed in place with its own pitches and always gets a first-pass job -- the copy branch when
    already at its load size -- while a host BGR HWC frame at its load size is read from the arena without one."""
    s = Sampler(4, 640, 640, dict(HYP_YOLOV6S, mosaic=0.0))
    big = torch.empty(700, 900, 3, dtype=torch.uint8, device=META)
    crop = big[10:490, 20:660]                                          # 480 x 640: at its load size, rows of 2700 bytes
    chw = torch.empty(3, 333, 517, dtype=torch.uint8, device=META)
    host_at_size = np.zeros((640, 640, 3), np.uint8)
    host_small = np.zeros((100, 60, 3), np.uint8)
    srcs = {0: as_source(check_frame(crop, "bgr_hwc", META), "bgr_hwc"),
            1: as_source(check_frame(chw, "rgb_chw", META), "rgb_chw"),
            2: as_source(check_frame(host_at_size, "bgr_hwc", META), "bgr_hwc"),
            3: as_source(check_frame(host_small, "bgr_hwc", META), "bgr_hwc")}
    plan = letterbox_plan(s, [0, 1, 2, 3])
    used, total, shapes, loc, jobs1, recs1, jobs2, smp = batch_tables(s, 4, plan, srcs)
    assert used == 640 * 640 * 3 + 100 * 60 * 3 and loc == {2: 0, 3: 640 * 640 * 3}
    assert shapes == {0: (480, 640), 1: (333, 517), 2: (640, 640), 3: (100, 60)}
    assert plan.sources == [0, 1, 2, 3] and len(jobs1) == len(recs1) == 3        # nothing for source 2
    jobs, rec = dict(zip([0, 1, 3], jobs1)), dict(zip([0, 1, 3], recs1))
    assert jobs[0][1:3] == jobs[0][4:6] == [480, 640]                   # copy job
    assert rec[0] == (False, crop.data_ptr(), 2700, 0, _lib.LB_BGR_HWC)
    assert jobs[1][4:6] == list(resized_shape(333, 517, 640))
    assert rec[1] == (False, chw.data_ptr(), 517, 333 * 517, _lib.LB_RGB_CHW)
    assert rec[3] == (True, 640 * 640 * 3, 180, 0, _lib.LB_BGR_HWC)      # staged: an arena offset
    assert min(j[3] for j in jobs1) == used and total > used
    table = frame_records(recs1, 0x1000)
    assert C.sizeof(table) == 3 * REC
    staged = [t for t in table if t.row_pitch == 180][0]
    assert staged.base == 0x1000 + 640 * 640 * 3


def test_cache_source_is_a_bgr_record_at_the_load_size():
    s = Sampler(len(SHAPES), 640, 640, HYP_YOLOV6S)
    loaded, offsets, _ = cache_layout(SHAPES, s)
    cache = FrameCache.__new__(FrameCache)                             # the arena's address stands in for device memory
    cache.shapes_hw, cache.loaded, cache.offsets = np.array(SHAPES), loaded, offsets
    cache.arena = torch.empty(16, dtype=torch.uint8)
    src = cache.source(5)
    assert (src.t, src.staged, src.h0, src.w0, src.ph, src.pw) == (None, False, 720, 1280, 360, 640)
    assert (src.base, src.row_pitch, src.plane_pitch, src.layout) == (cache.arena.data_ptr() + int(offsets[5]), 1920, 0,
                                                                      _lib.LB_BGR_HWC)


def test_resize_frames_declaration_matches_binding_and_record(tmp_path):
    """The header declares yv6_aug_resize_frames with the yv6_lb_src table first and the arena last, as bound; the
    yv6_lb_src mirror still matches the header."""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    decl = tmp_path / "decl.c"                          # -Werror: a declaration of another type does not compile
    decl.write_text('#include "yv6.h"\n'
                    "typedef int (*fn)(yv6_handle*, const yv6_lb_src*, const int64_t*, int32_t, int64_t, uint8_t*, void*);\n"
                    "fn resize_frames = yv6_aug_resize_frames;\n")
    subprocess.run(["gcc", "-Werror", "-I", inc, "-c", str(decl), "-o", str(tmp_path / "decl.o")], check=True)
    fields = [f for f, _ in _lib.LbSrc._fields_]
    src = tmp_path / "rec.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yv6.h"\nint main(void){printf("%zu %zu'
                   + " %zu" * len(fields) + '\\n", sizeof(yv6_lb_src), sizeof(int64_t) * YV6_AUG_JOB, '
                   + ", ".join(f"offsetof(yv6_lb_src, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "rec"
    subprocess.run(["gcc", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.LbSrc), JOB * 8] + [getattr(_lib.LbSrc, f).offset for f in fields]
    _, args = _lib._SIGNATURES["yv6_aug_resize_frames"]
    assert len(args) == 7 and args[4] is C.c_int64 and args[3] is C.c_int32
    assert REC == C.sizeof(_lib.LbSrc) == 32
