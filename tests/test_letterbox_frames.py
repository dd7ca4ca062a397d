"""CPU checks of the frame-source side of yv6_letterbox_frames: the yv6_lb_src ctypes mirror against the header, the
records and pitches the host derives from tensor shapes and strides, and the checks that reject a frame before anything
is written or enqueued.  Device frames are stood in for by meta tensors, which carry sizes, strides and a device but no
memory."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from yolov6_b200 import _lib
from yolov6_b200.preprocess import GEO, REC, check_frames, letterbox_geometry, pack_sources, source_pitches

META = torch.device("meta")


def test_lb_src_mirror_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = [f for f, _ in _lib.LbSrc._fields_]
    src = tmp_path / "lb.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yv6.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + ' %d %d\\n", sizeof(yv6_lb_src), '
                   + "".join(f"offsetof(yv6_lb_src, {f}), " for f in fields) + "YV6_LB_BGR_HWC, YV6_LB_RGB_CHW);return 0;}\n")
    exe = tmp_path / "lb"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    want = [C.sizeof(_lib.LbSrc)] + [getattr(_lib.LbSrc, f).offset for f in fields] + [_lib.LB_BGR_HWC, _lib.LB_RGB_CHW]
    assert got == want, (got, want)
    assert REC == C.sizeof(_lib.LbSrc) == 32


def test_pitches_from_shapes_and_strides():
    hwc = torch.zeros(100, 200, 3, dtype=torch.uint8)
    assert source_pitches(hwc.shape, hwc.stride(), "bgr_hwc") == (100, 200, 600, 0)
    crop = hwc[10:50, 20:80]                                       # rows padded to the full frame's 600 bytes
    assert source_pitches(crop.shape, crop.stride(), "bgr_hwc") == (40, 60, 600, 0)
    chw = torch.zeros(3, 100, 200, dtype=torch.uint8)
    assert source_pitches(chw.shape, chw.stride(), "rgb_chw") == (100, 200, 200, 20000)
    crop = chw[:, 10:50, 20:80]
    assert source_pitches(crop.shape, crop.stride(), "rgb_chw") == (40, 60, 200, 20000)
    planes = torch.zeros(4, 100, 200, dtype=torch.uint8)[1:]      # three planes of a four-plane buffer
    assert source_pitches(planes.shape, planes.stride(), "rgb_chw") == (100, 200, 200, 20000)


def records(rec_host, B):
    return [_lib.LbSrc.from_buffer_copy(bytes(rec_host[i * REC:(i + 1) * REC].tolist())) for i in range(B)]


def test_pack_sources_host_and_device_frames():
    """Host frames (numpy HWC, CPU tensor views) are staged contiguously and their records point into the device staging
    buffer; a device frame's record points at the frame with its own pitches and takes no staging bytes."""
    B, H, W, ptr = 4, 32, 64, 0x10000
    host_np = np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3)
    host_view = torch.arange(6 * 4 * 3, dtype=torch.uint8).reshape(6, 4, 3)[1:6, 1:2]        # a crop: staged contiguous
    dev = torch.empty(50, 60, 3, dtype=torch.uint8, device=META)[5:45, 7:57]                  # 6000 bytes, none staged
    srcs = check_frames([host_np, dev, host_view], B, "bgr_hwc", META)
    src, geo, rec = torch.zeros(40, dtype=torch.uint8), torch.zeros(B, GEO, dtype=torch.int32), torch.zeros(B * REC, dtype=torch.uint8)
    used, shapes, devs = pack_sources(srcs, B, H, W, True, "bgr_hwc", src, geo, rec, ptr)
    assert used == 18 + 15 and len(devs) == 1 and devs[0] is srcs[1][0]
    assert src[:18].tolist() == list(range(18)) and src[18:33].tolist() == host_view.reshape(-1).tolist()
    r = records(rec, B)
    assert (r[0].base, r[0].row_pitch, r[0].plane_pitch, r[0].layout) == (ptr, 9, 0, _lib.LB_BGR_HWC)
    assert (r[1].base or 0, r[1].row_pitch, r[1].plane_pitch, r[1].layout) == (dev.data_ptr(), 180, 0, _lib.LB_BGR_HWC)
    assert (r[2].base, r[2].row_pitch) == (ptr + 18, 3)
    assert r[3].base is None                                       # unused slot: null record, all border
    _, (nw, nh), top, left = letterbox_geometry(40, 50, H, W, True)
    assert geo[1].tolist() == [0, 40, 50, nh, nw, top, left, 0]
    assert geo[2].tolist()[:3] == [18, 5, 1] and geo[3].tolist() == [0, H, W, 0, 0, 0, 0, 0]
    assert shapes[1][0] == (40, 50)

    chw_np = np.arange(3 * 2 * 5, dtype=np.uint8).reshape(3, 2, 5)
    chw_dev = torch.empty(3, 70, 90, dtype=torch.uint8, device=META)[:, 10:60, 20:80]
    srcs = check_frames([chw_dev, chw_np], B, "rgb_chw", META)
    used, _, _ = pack_sources(srcs, B, H, W, True, "rgb_chw", src, geo, rec, ptr)
    r = records(rec, B)
    assert used == 30 and src[:30].tolist() == list(range(30))
    assert (r[0].row_pitch, r[0].plane_pitch, r[0].layout) == (90, 6300, _lib.LB_RGB_CHW)
    assert (r[1].base, r[1].row_pitch, r[1].plane_pitch, r[1].layout) == (ptr, 5, 10, _lib.LB_RGB_CHW)
    assert geo[0].tolist()[:3] == [0, 50, 60] and geo[1].tolist()[:3] == [0, 2, 5]


def test_staging_capacity_counts_host_frames_only():
    big_dev = torch.empty(1000, 1000, 3, dtype=torch.uint8, device=META)
    srcs = check_frames([big_dev, np.zeros((2, 2, 3), np.uint8)], 2, "bgr_hwc", META)
    src, geo, rec = torch.zeros(12, dtype=torch.uint8), torch.zeros(2, GEO, dtype=torch.int32), torch.zeros(2 * REC, dtype=torch.uint8)
    assert pack_sources(srcs, 2, 32, 32, True, "bgr_hwc", src, geo, rec, 0)[0] == 12
    srcs = check_frames([np.zeros((3, 2, 3), np.uint8)], 2, "bgr_hwc", META)
    before = (src.clone(), geo.clone(), rec.clone())
    with pytest.raises(RuntimeError, match="max_src_bytes"):
        pack_sources(srcs, 2, 32, 32, True, "bgr_hwc", src, geo, rec, 0)
    assert all(torch.equal(a, b) for a, b in zip((src, geo, rec), before))


def meta(*shape, dtype=torch.uint8):
    return torch.empty(*shape, dtype=dtype, device=META)


@pytest.mark.parametrize("case", [
    "other_device", "dtype", "host_dtype", "dims", "hwc_channels", "chw_channels", "host_channels", "innermost", "pixel_stride",
    "layout", "not_a_frame", "too_many", "none"])
def test_frame_rejections(case):
    """Each malformed frame raises RuntimeError from the checks, which run before any table is written or work enqueued."""
    dev, layout, B = META, "bgr_hwc", 2
    frames = {
        "other_device": ([meta(8, 8, 3)], torch.device("cuda", 0)),              # a device frame on another device
        "dtype": ([meta(8, 8, 3, dtype=torch.float32)], dev),
        "host_dtype": ([np.zeros((8, 8, 3), np.float32)], dev),
        "dims": ([meta(8, 24)], dev),
        "hwc_channels": ([meta(3, 8, 8)], dev),                                     # CHW given as bgr_hwc
        "host_channels": ([np.zeros((8, 8, 4), np.uint8)], dev),
        "innermost": ([meta(3, 8, 8).permute(1, 2, 0)], dev),                       # HWC view of CHW planes: unit stride on W
        "pixel_stride": ([meta(8, 8, 4)[:, :, :3]], dev),                           # BGRA with the alpha left out
        "layout": ([meta(8, 8, 3)], dev),
        "not_a_frame": ([[[1, 2, 3]]], dev),
        "too_many": ([meta(8, 8, 3)] * 3, dev),
        "none": ([], dev),
    }
    if case == "chw_channels":
        frs, dev, layout = [meta(8, 8, 3)], dev, "rgb_chw"                         # HWC given as rgb_chw
    else:
        frs, dev = frames[case]
    if case == "layout":
        layout = "rgb_hwc"
    with pytest.raises(RuntimeError):
        check_frames(frs, B, layout, dev)
    assert check_frames([meta(8, 8, 3), np.zeros((2, 2, 3), np.uint8)], B, "bgr_hwc", META)[0][1]      # the valid form passes
