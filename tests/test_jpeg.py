"""CPU checks of the JPEG decoder's host side and of its numpy oracle against cv2.imread's bytes (tests/golden/jpeg*)."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import jpeg as oj
from yolov6_b200 import jpeg

GOLD = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLD, "jpeg_cases.json")) as f:
    META = json.load(f)
BLOBS = dict(np.load(os.path.join(GOLD, "jpeg.npz")))
CASES, REFUSED = META["cases"], META["refused"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_parse_shape_sampling_restart(name):
    c = CASES[name]
    info = jpeg.parse(BLOBS[name].tobytes())
    assert list(info.shape) == c["shape"]
    assert info.sampling == c["sampling"]
    assert info.restart == c["restart"]
    assert info.orientation == c.get("orientation", 1)


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_with_reason(name):
    with pytest.raises(ValueError, match=REFUSED[name]["reason"]):
        jpeg.parse(BLOBS["refused_" + name].tobytes())


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_cv2(name):
    got = oj.decode(BLOBS[name].tobytes())
    assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == CASES[name]["sha256"]


def test_exif_orientation_transposes_5_to_8():
    """cv2.imread transposes for orientations 5-8 (the reference's check_image swaps the shape for 6 and 8 only)."""
    for o in range(1, 9):
        for order in ("II", "MM"):
            h, w, _ = jpeg.parse(BLOBS[f"exif{o}_{order}"].tobytes()).shape
            assert (h, w) == ((53, 37) if o >= 5 else (37, 53))


def test_huffman_tables_decode_every_code():
    """huff_table's lookahead and long-code arrays give back every symbol of a table with codes of 1..16 bits."""
    bits = [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2]
    vals = list(range(17))
    t = jpeg.huff_table(bits, vals)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            v = code << (16 - l)
            e = t.lut[v >> 7]
            if l <= 9:
                assert e == (l << 8) | vals[k]
            else:
                assert e == 0 and code <= t.maxcode[l] and t.vals[code + t.valoff[l]] == vals[k]
            code += 1
            k += 1
        code <<= 1


def test_ctypes_mirrors_match_the_jpeg_struct_sizes(tmp_path):
    """yolov6_b200._lib's JpegHuff / JpegComp / JpegImage have the sizes a C compiler gives the structs of include/yv6.h."""
    import ctypes as C
    import shutil
    import subprocess
    from yolov6_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "yv6.h"\nint main(){printf("%zu %zu %zu\\n", sizeof(yv6_jpeg_huff), '
                   'sizeof(yv6_jpeg_comp), sizeof(yv6_jpeg_image));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.JpegHuff), C.sizeof(_lib.JpegComp), C.sizeof(_lib.JpegImage)]


def _segments(b):
    out, p = [], 2
    while True:
        m = b[p + 1]
        L = int.from_bytes(b[p + 2:p + 4], "big")
        out.append((m, b[p + 4:p + 2 + L]))
        p += 2 + L
        if m == 0xDA:
            return out, b[p:]


@pytest.mark.parametrize("marker,keep", [(0xC0, 4), (0xC0, 8), (0xC4, 10), (0xC4, 20), (0xDB, 30), (0xDA, 0), (0xDA, 3), (0xDD, 1)])
def test_truncated_header_segment_raises_value_error(marker, keep):
    """A header segment shorter than its fields need is a ValueError naming it, never an IndexError or a short table."""
    b = BLOBS["rst7_333x500"].tobytes()
    segs, rest = _segments(b)
    assert any(m == marker for m, _ in segs)
    body = b"".join(b"\xff" + bytes([m]) + (len(s if m != marker else s[:keep]) + 2).to_bytes(2, "big") + (s if m != marker else s[:keep])
                    for m, s in segs)
    with pytest.raises(ValueError, match="truncated"):
        jpeg.parse(b"\xff\xd8" + body + rest)
