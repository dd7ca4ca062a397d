"""Writes tests/golden/jpeg_cases.json and tests/golden/jpeg.npz: JPEG streams and the SHA-256 of what cv2.imread returns
for each (cv2 4.13 / libjpeg-turbo 3.1.2), plus one crafted stream of each kind the device decoder refuses.

    python tests/golden/make_golden_jpeg.py

Sources are the seeded synthetic photographs of tools/bench_augment_frames.py (smooth waves, blobs and grain) and uniform
noise, JPEG's worst case.  Each case is decoded by cv2.imdecode, which is cv2.imread on the same bytes."""
import hashlib
import json
import os
import struct
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
from bench_augment_frames import photo  # noqa: E402

SAMP = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
        "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420,
        "411": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411}


def enc(img, q=90, samp="420", rst=0, opt=0, prog=0):
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMP[samp],
                                       cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_OPTIMIZE, opt,
                                       cv2.IMWRITE_JPEG_PROGRESSIVE, prog])
    assert ok
    return b.tobytes()


def segments(b):
    """[(marker, payload)] of the header up to and including SOS, and the rest (entropy data + EOI)."""
    out, p = [], 2
    while True:
        m = b[p + 1]
        L = struct.unpack(">H", b[p + 2:p + 4])[0]
        out.append((m, b[p + 4:p + 2 + L]))
        p += 2 + L
        if m == 0xDA:
            return out, b[p:]


def join(segs, rest):
    return b"\xff\xd8" + b"".join(b"\xff" + bytes([m]) + struct.pack(">H", len(s) + 2) + s for m, s in segs) + rest


def with_dqt16(b):
    segs, rest = segments(b)
    new = []
    for m, s in segs:
        if m == 0xDB:
            t, q = b"", 0
            while q < len(s):
                t += bytes([0x10 | (s[q] & 15)]) + b"".join(struct.pack(">H", v) for v in s[q + 1:q + 65])
                q += 65
            s = t
        new.append((m, s))
    return join(new, rest)


def with_exif(b, orientation, order):
    bo = "<" if order == "II" else ">"
    tiff = order.encode() + struct.pack(bo + "HI", 42, 8) + struct.pack(bo + "H", 1)
    tiff += struct.pack(bo + "HHI", 0x0112, 3, 1) + struct.pack(bo + "HH", orientation, 0) + struct.pack(bo + "I", 0)
    app1 = b"Exif\x00\x00" + tiff
    return b[:2] + b"\xff\xe1" + struct.pack(">H", len(app1) + 2) + app1 + b[2:]


def app1(payload):
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def tiff(order="II", entries=((0x0112, 3, 6),), magic=42, ifd=8, count=None, trunc=None):
    """A TIFF header and IFD0 of (tag, type, value) entries, the value stored as that type would store it."""
    bo = "<" if order == "II" else ">"
    t = order.encode() + struct.pack(bo + "HI", magic, ifd) + b"\0" * (ifd - 8)
    t += struct.pack(bo + "H", len(entries) if count is None else count)
    for tag, typ, v in entries:
        t += struct.pack(bo + "HHI", tag, typ, 1)
        t += struct.pack(bo + "HH", v, 0) if typ == 3 else struct.pack(bo + "I", v) if typ == 4 else bytes([v, 0, 0, 0])
    t += b"\0\0\0\0"
    return t if trunc is None else t[:trunc]


def exif_app1(**kw):
    return app1(b"Exif\0\0" + tiff(**kw))


# APP1 payloads cv2.imread may meet, well-formed or not: which orientation it applies is what the golden records
MALFORMED_EXIF = {
    "xmp_then_exif6": [app1(b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta/>"), exif_app1()],
    "long_II_6": [exif_app1(entries=((0x0112, 4, 6),))],
    "long_MM_6": [exif_app1(order="MM", entries=((0x0112, 4, 6),))],
    "byte_II_6": [exif_app1(entries=((0x0112, 1, 6),))],
    "byte_MM_6": [exif_app1(order="MM", entries=((0x0112, 1, 6),))],
    "undefined_II_6": [exif_app1(entries=((0x0112, 7, 6),))],
    "two_exif_1_then_6": [exif_app1(entries=((0x0112, 3, 1),)), exif_app1()],
    "two_exif_none_then_6": [exif_app1(entries=((0x010F, 3, 1),)), exif_app1()],
    "two_exif_6_then_3": [exif_app1(), exif_app1(entries=((0x0112, 3, 3),))],
    "bad_magic": [exif_app1(magic=43)],
    "bad_magic_then_exif6": [exif_app1(magic=43), exif_app1()],
    "bad_byte_order": [app1(b"Exif\0\0XX" + tiff()[2:])],
    "not_exif_header": [app1(b"Exif\0X" + tiff())],
    "value_9": [exif_app1(entries=((0x0112, 3, 9),))],
    "value_0": [exif_app1(entries=((0x0112, 3, 0),))],
    "value_9_then_exif6": [exif_app1(entries=((0x0112, 3, 9),)), exif_app1()],
    "entry_cut_in_value": [app1(b"Exif\0\0" + tiff(trunc=8 + 2 + 9))],
    "entry_cut_after_value": [app1(b"Exif\0\0" + tiff(trunc=8 + 2 + 10))],
    "entry_cut_then_exif6": [app1(b"Exif\0\0" + tiff(trunc=8 + 2 + 9)), exif_app1()],
    "count_past_end": [exif_app1(count=5)],
    "ifd0_past_end": [app1(b"Exif\0\0II" + struct.pack("<HI", 42, 4000) + b"\0" * 20)],
    "ifd0_at_16": [exif_app1(ifd=16)],
    "second_entry_6": [exif_app1(entries=((0x010F, 3, 1), (0x0112, 3, 6)))],
    "duplicate_tag_6_then_3": [exif_app1(entries=((0x0112, 3, 6), (0x0112, 3, 3)))],
}


def applied_orientation(im, plain):
    from oracle.jpeg import orient
    hits = [o for o in range(1, 9) if orient(plain, o).shape == im.shape and np.array_equal(orient(plain, o), im)]
    assert len(hits) >= 1
    return hits[0]


def refused(base, gray):
    segs, rest = segments(base)
    out = {}
    def patch(m_from, fn):
        return join([(fn(m, s) if m == m_from else (m, s)) for m, s in segs], rest)
    out["progressive"] = (None, "progressive")
    out["arithmetic"] = (join([((0xC9, s) if m == 0xC0 else (m, s)) for m, s in segs], rest), "arithmetic")
    out["lossless"] = (join([((0xC3, s) if m == 0xC0 else (m, s)) for m, s in segs], rest), "lossless")
    out["12bit"] = (join([((0xC1, bytes([12]) + s[1:]) if m == 0xC0 else (m, s)) for m, s in segs], rest), "12-bit")
    sof = [s for m, s in segs if m == 0xC0][0]
    cmyk = bytes([8]) + sof[1:5] + bytes([4]) + sof[6:] + bytes([4, 0x11, 0])
    out["cmyk"] = (join([((0xC0, cmyk) if m == 0xC0 else (m, s)) for m, s in segs], rest), "4 components")
    adobe = b"Adobe" + struct.pack(">HHHB", 100, 0, 0, 0)
    out["adobe_rgb"] = (join([(0xEE, adobe)] + segs, rest), "not YCbCr")
    sos = [s for m, s in segs if m == 0xDA][0]
    one = bytes([1]) + sos[1:3] + sos[-3:]
    out["multiscan"] = (join([((m, one) if m == 0xDA else (m, s)) for m, s in segs], rest), "multi-scan")
    out["no_dht"] = (join([(m, s) for m, s in segs if m != 0xC4], rest), "missing Huffman table")
    return out


def main():
    rng = np.random.default_rng(20261018)
    cases = {}

    def add(name, b, **kw):
        im = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        cases[name] = dict(bytes=b, shape=list(im.shape), sha256=hashlib.sha256(np.ascontiguousarray(im).tobytes()).hexdigest(), **kw)

    p33, p333 = photo(33, 65, rng), photo(333, 500, rng)
    for s in SAMP:
        add(f"samp{s}_33x65", enc(p33, samp=s), sampling=s, restart=0)
        add(f"samp{s}_17x9", enc(photo(17, 9, rng), samp=s), sampling=s, restart=0)
    for q in (50, 75, 90, 100):
        for opt in (0, 1):
            add(f"q{q}_opt{opt}_333x500", enc(p333, q=q, opt=opt), sampling="420", restart=0)
    for rst in (1, 7):
        add(f"rst{rst}_333x500", enc(p333, rst=rst), sampling="420", restart=rst)
        add(f"rst{rst}_444_33x65", enc(p33, samp="444", rst=rst), sampling="444", restart=rst)
    add("gray_333x500", enc(cv2.cvtColor(p333, cv2.COLOR_BGR2GRAY)), sampling="gray", restart=0)
    add("gray_rst7_33x65", enc(cv2.cvtColor(p33, cv2.COLOR_BGR2GRAY), rst=7), sampling="gray", restart=7)
    add("dqt16_333x500", with_dqt16(enc(p333, q=75)), sampling="420", restart=0)
    for h, w in ((1, 1), (8, 8), (2, 3), (481, 640)):
        add(f"size_{h}x{w}", enc(photo(h, w, rng) if h > 4 else rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), sampling="420", restart=0)
    add("noise_q90_96x128", enc(rng.integers(0, 256, (96, 128, 3), dtype=np.uint8)), sampling="420", restart=0)
    add("noise_q100_444_64x64", enc(rng.integers(0, 256, (64, 64, 3), dtype=np.uint8), q=100, samp="444"), sampling="444", restart=0)
    big = photo(1080, 1920, rng)
    add("size_1080x1920", enc(big, q=75), sampling="420", restart=0)
    add("size_1080x1920_rst_row", enc(big, q=75, rst=1920 // 16), sampling="420", restart=120)
    p37 = photo(37, 53, rng)
    for o in range(1, 9):
        for order in ("II", "MM"):
            add(f"exif{o}_{order}", with_exif(enc(p37, samp="422"), o, order), sampling="422", restart=0, orientation=o)
    import torch
    from torchvision.io import encode_jpeg
    tv = encode_jpeg(torch.from_numpy(np.ascontiguousarray(p333[..., ::-1].transpose(2, 0, 1))), quality=85).numpy().tobytes()
    add("torchvision_333x500", tv, sampling="420", restart=0)
    b37 = enc(p37, samp="422")
    plain = cv2.imdecode(np.frombuffer(b37, np.uint8), cv2.IMREAD_COLOR)
    for name, segs in MALFORMED_EXIF.items():
        b = b37[:2] + b"".join(segs) + b37[2:]
        o = applied_orientation(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), plain)
        add(f"exifx_{name}", b, sampling="422", restart=0, orientation=o)

    ref = {}
    for name, (b, reason) in refused(enc(p33), True).items():
        ref[name] = dict(bytes=b if b is not None else enc(p33, prog=1), reason=reason)

    blobs = {k: np.frombuffer(v.pop("bytes"), np.uint8) for k, v in list(cases.items())}
    blobs.update({"refused_" + k: np.frombuffer(v.pop("bytes"), np.uint8) for k, v in ref.items()})
    np.savez_compressed(os.path.join(HERE, "jpeg.npz"), **blobs)
    with open(os.path.join(HERE, "jpeg_cases.json"), "w") as f:
        json.dump(dict(cv2=cv2.__version__, cases=cases, refused=ref), f, indent=1, sort_keys=True)
    print(len(cases), "cases,", len(ref), "refused,", os.path.getsize(os.path.join(HERE, "jpeg.npz")), "bytes")


if __name__ == "__main__":
    main()
