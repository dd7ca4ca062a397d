"""JPEG decoding on the device, byte-identical to `cv2.imread(path)` (IMREAD_COLOR, libjpeg-turbo's defaults).

The reference decodes every image with cv2.imread in `load_image` (yolov6/data/datasets.py:272).  Here the header is
parsed on the host (`parse`, once per file: a dataset does it at start-up, as the reference's `check_image` opens every
image) and the pixels are produced by three kernels per batch (csrc/yv6_jpeg.cu):

  - entropy decode, one CTA per image: the scan is unstuffed (FF 00 -> FF, RSTn markers removed and their positions
    kept), then split into one bit range per thread.  Every thread decodes its range from a guessed state, records the
    state in which it leaves the range, and decodes again whenever the state it was handed changes, until every boundary
    agrees (self-synchronising Huffman decoding, Weissenberger & Schmidt); restart markers are exact sync points.  A last
    pass places each block and turns DC differences into DC values;
  - dequantisation and libjpeg's integer ("ISLOW") IDCT into component sample planes;
  - libjpeg-turbo's fancy (triangle) upsampling for h2v1, h2v2 and h1v2 chroma (replication otherwise, and for chroma at
    most two samples wide), its fixed-point YCbCr -> BGR tables, and the EXIF orientation cv2.imread applies, into one
    uint8 BGR HWC frame per image.

Supported: baseline / extended sequential Huffman (SOF0 / SOF1), 8-bit samples, 1 or 3 components in one interleaved scan,
luma sampling 1x1, 2x1, 1x2, 2x2 or 4x1 with chroma 1x1, 8- or 16-bit DQT, any DHT, any restart interval.  Every other
stream is refused by `parse` with a ValueError naming the reason; such files are decoded on the host by the caller and
passed to the feeds as host frames.  Frames of a corrupt stream are flagged in a per-image status word the decode writes
on the device; `JpegDecoder.check()` raises for them.  libjpeg's warn-and-continue recovery is not reproduced.
"""
import ctypes as C
import struct
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63], np.int64)     # zigzag index -> natural (row-major) index
SAMPLINGS = {(1, 1): "444", (2, 1): "422", (1, 2): "440", (2, 2): "420", (4, 1): "411"}
STATUS = {0: "ok", 1: "entropy data ran out", 2: "invalid Huffman code", 3: "AC run-length past coefficient 63"}

_SOF_REFUSED = {0xC2: "progressive (SOF2)", 0xC3: "lossless (SOF3)", 0xC5: "differential sequential (SOF5)",
                0xC6: "differential progressive (SOF6)", 0xC7: "differential lossless (SOF7)"}
_SOF_REFUSED.update({m: f"arithmetic coding (SOF{m - 0xC0})" for m in (0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF)})


@dataclass
class Info:
    """What `parse` finds in one JPEG.  height, width: the frame as coded; shape: what cv2.imread returns (after the EXIF
    orientation: 5-8 transpose); comps: per component (h, v, quant natural-order uint16[64], dc (bits, vals), ac (bits,
    vals)); scan: [start, end) byte offsets of the entropy-coded segment; restart: MCUs per restart interval (0: none);
    tables: per component the keys of its DC and AC tables' device form (`huff_table`, built once per distinct table)."""
    height: int
    width: int
    orientation: int
    shape: tuple
    sampling: str
    restart: int
    comps: list
    scan: tuple
    tables: tuple


def _exif_orientation(seg):
    """The Orientation (0x0112) of IFD0 in one APP1 payload, as cv2 reads it: only a payload that starts with
    "Exif\\0\\0", a TIFF header in either byte order with magic 42, and IFD0 inside the payload; the entries are walked
    while their first 10 bytes are there, and the first Orientation entry gives the 16-bit value at its value field in
    the file's byte order, whatever its type and count say.  None when the payload has no such entry (cv2 then looks at
    the next APP1).  tests/golden/make_golden_jpeg.py pins these rules against cv2.imread, malformed payloads included."""
    if seg[:6] != b"Exif\x00\x00":
        return None
    t = seg[6:]
    bo = {b"II": "<", b"MM": ">"}.get(t[:2])
    if bo is None or len(t) < 8 or struct.unpack(bo + "H", t[2:4])[0] != 42:
        return None
    ifd = struct.unpack(bo + "I", t[4:8])[0]
    if ifd + 2 > len(t):
        return None
    n = struct.unpack(bo + "H", t[ifd:ifd + 2])[0]
    for e in range(n):
        p = ifd + 2 + 12 * e
        if p + 10 > len(t):
            return None
        if struct.unpack(bo + "H", t[p:p + 2])[0] == 0x0112:
            return struct.unpack(bo + "H", t[p + 8:p + 10])[0]
    return None


def _need(seg, n, what):
    if len(seg) < n:
        raise ValueError(f"JPEG: {what} segment is truncated ({len(seg)} bytes, needs {n})")


def _scan_end(a, start):
    """Offset of the first marker after `start` that is not a stuffed FF 00, an RSTn or a fill FF: the end of the
    entropy-coded segment (len(a) for a truncated stream)."""
    s = a[start:]
    ff = np.flatnonzero(s[:-1] == 0xFF)
    nxt = s[ff + 1]
    stop = ff[(nxt != 0) & (nxt != 0xFF) & ((nxt < 0xD0) | (nxt > 0xD7))]
    return start + int(stop[0]) if len(stop) else len(a)


def parse(buf):
    """Parse one JPEG (bytes-like or uint8 array) -> `Info`.  ValueError naming the reason for every stream the device
    decoder does not take (see the module docstring) and for malformed headers."""
    a = np.frombuffer(bytes(buf) if not isinstance(buf, np.ndarray) else buf.tobytes(), np.uint8)
    b = a.tobytes()
    if len(b) < 4 or b[:2] != b"\xff\xd8":
        raise ValueError("JPEG: no SOI marker")
    qt, dht, frame, restart, orient, adobe = {}, {}, None, 0, None, None
    p = 2
    while True:
        while p < len(b) and b[p] != 0xFF:
            p += 1
        while p < len(b) and b[p] == 0xFF:
            p += 1
        if p + 2 >= len(b):
            raise ValueError("JPEG: no scan (SOS) before the end of the data")
        m = b[p]
        p += 1
        if m in (0x01,) or 0xD0 <= m <= 0xD7:
            continue
        if m == 0xD9:
            raise ValueError("JPEG: no scan (SOS) before EOI")
        L = (b[p] << 8) | b[p + 1]
        seg = b[p + 2:p + L]
        if L < 2 or len(seg) != L - 2:
            raise ValueError(f"JPEG: marker FF{m:02X} runs past the end of the data")
        p += L
        if m in _SOF_REFUSED:
            raise ValueError(f"JPEG: {_SOF_REFUSED[m]} is not supported")
        if m in (0xC0, 0xC1):
            _need(seg, 6, "SOF")
            _need(seg, 6 + 3 * seg[5], "SOF")
            P, H, W, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if P != 8:
                raise ValueError(f"JPEG: {P}-bit samples are not supported (8-bit only)")
            if nf not in (1, 3):
                raise ValueError(f"JPEG: {nf} components (CMYK / YCCK) are not supported")
            if H == 0 or W == 0:
                raise ValueError("JPEG: zero image height or width (DNL) is not supported")
            frame = dict(H=H, W=W, comps=[(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)])
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                tc, th = seg[q] >> 4, seg[q] & 15
                _need(seg, q + 17, "DHT")
                bits = list(seg[q + 1:q + 17])
                n = sum(bits)
                _need(seg, q + 17 + n, "DHT")
                dht[(tc, th)] = (bits, list(seg[q + 17:q + 17 + n]))
                _check_table(*dht[(tc, th)], "DC" if tc == 0 else "AC")
                q += 17 + n
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                _need(seg, q + (129 if pq else 65), "DQT")
                if pq:
                    vals = np.frombuffer(seg[q + 1:q + 129], ">u2").astype(np.uint16)
                    q += 129
                else:
                    vals = np.frombuffer(seg[q + 1:q + 65], np.uint8).astype(np.uint16)
                    q += 65
                nat = np.zeros(64, np.uint16)
                nat[ZIGZAG] = vals
                qt[tq] = nat
        elif m == 0xDD:
            _need(seg, 2, "DRI")
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE1 and orient is None:
            orient = _exif_orientation(seg)
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xCC:
            raise ValueError("JPEG: arithmetic coding (DAC) is not supported")
        elif m == 0xDA:
            break
    if frame is None:
        raise ValueError("JPEG: no SOF0 / SOF1 frame header before the scan")
    _need(seg, 1, "SOS")
    ns = seg[0]
    _need(seg, 4 + 2 * ns, "SOS")
    sc = {seg[1 + 2 * i]: (seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)}
    ss, se, ahl = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    fc = frame["comps"]
    if ns != len(fc) or set(sc) != {c[0] for c in fc}:
        raise ValueError("JPEG: multi-scan sequential (a scan without every component) is not supported")
    if ss != 0 or se != 63 or ahl != 0:
        raise ValueError("JPEG: a sequential scan must cover coefficients 0..63 without successive approximation")
    if len(fc) == 3:
        ids = tuple(c[0] for c in fc)
        if adobe == 0 or (adobe is None and ids == (82, 71, 66)):
            raise ValueError("JPEG: the Adobe transform / component ids say RGB, not YCbCr, which is not supported")
        if [(c[1], c[2]) for c in fc[1:]] != [(1, 1), (1, 1)] or (fc[0][1], fc[0][2]) not in SAMPLINGS:
            raise ValueError(f"JPEG: sampling {[(c[1], c[2]) for c in fc]} is not supported (luma 1x1, 2x1, 1x2, 2x2 or 4x1, chroma 1x1)")
    comps = []
    for cid, h, v, tq in fc:
        td, ta = sc[cid]
        if tq not in qt:
            raise ValueError(f"JPEG: missing quantisation table {tq}")
        for cls, t in ((0, td), (1, ta)):
            if (cls, t) not in dht:
                raise ValueError(f"JPEG: missing Huffman table ({'DC' if cls == 0 else 'AC'} {t})")
        comps.append((h, v) if len(fc) == 3 else (1, 1))
        comps[-1] = (*comps[-1], qt[tq], dht[(0, td)], dht[(1, ta)])
    start = p
    end = _scan_end(a, start)
    q = end
    while q + 1 < len(b):                        # what follows the scan: EOI, or another scan (refused)
        if b[q] == 0xFF and b[q + 1] == 0xDA:
            raise ValueError("JPEG: multi-scan sequential (more than one scan) is not supported")
        if b[q] == 0xFF and b[q + 1] == 0xD9:
            break
        if b[q] == 0xFF and b[q + 1] not in (0x00, 0xFF, 0x01) and not 0xD0 <= b[q + 1] <= 0xD7 and q + 3 < len(b):
            q += 2 + ((b[q + 2] << 8) | b[q + 3])
        else:
            q += 1
    orient = orient if orient is not None and 1 <= orient <= 8 else 1
    H, W = frame["H"], frame["W"]
    shape = (W, H, 3) if orient >= 5 else (H, W, 3)
    samp = "gray" if len(fc) == 1 else SAMPLINGS[(fc[0][1], fc[0][2])]
    tables = tuple((_device_table(dc), _device_table(ac)) for _, _, _, dc, ac in comps)
    return Info(H, W, orient, shape, samp, restart, comps, (start, end), tables)


_TABLES = {}     # key -> JpegHuff: the device form of every distinct Huffman table parsed so far


def _device_table(t):
    """Key of table t = (bits, vals) in _TABLES, building its device form the first time it is seen (a dataset written
    by one encoder repeats a few tables)."""
    key = bytes(t[0]) + bytes(t[1])
    if key not in _TABLES:
        _TABLES[key] = huff_table(*t)
    return key


def huff_table(bits, vals):
    """The device form of one Huffman table (`yv6_jpeg_huff`): a 9-bit lookahead (length << 8 | symbol, 0 for longer
    codes), and per length l the largest code maxcode[l] (-1: none; maxcode[17] is a sentinel) and valoff[l] such that
    vals[code + valoff[l]] is the symbol of an l-bit code."""
    t = _lib.JpegHuff()
    maxcode, valoff = [-1] * 18, [0] * 18
    maxcode[17] = 0x7FFFFFFF
    code = k = 0
    for l in range(1, 17):
        n = bits[l - 1]
        if n:
            valoff[l] = k - code
            for _ in range(n):
                if l <= 9:
                    for x in range(code << (9 - l), (code + 1) << (9 - l)):
                        t.lut[x] = (l << 8) | vals[k]
                code += 1
                k += 1
            maxcode[l] = code - 1
        code <<= 1
    t.maxcode[:] = maxcode
    t.valoff[:] = valoff
    t.vals[:len(vals)] = vals[:256]
    return t


def _check_table(bits, vals, what):
    """ValueError for a DHT that is not a Huffman code (libjpeg's 'Bogus Huffman table definition')."""
    code = 0
    for l in range(1, 17):
        code += bits[l - 1]
        if code >= (1 << l):        # no code may be all ones
            raise ValueError(f"JPEG: {what} Huffman table is not a prefix code")
        code <<= 1
    if sum(bits) > 256 or len(vals) != sum(bits):
        raise ValueError(f"JPEG: {what} Huffman table has {sum(bits)} codes")


class JpegStore:
    """The compressed bytes of a dataset resident in device memory, with their parsed `Info`s: what keeps a whole
    compressed training set on the card (COCO train2017: about 19 GB as JPEG).  `files` is any iterable of JPEG files
    (bytes-like), read once in order, so a generator that reads each file from disk holds no more than one chunk on the
    host.  Files are packed into device chunks of about `chunk_bytes` (a larger file gets a chunk of its own), each
    uploaded through one pinned staging buffer of that size.  ValueError naming the index of a file `parse` refuses or
    finds malformed (decode those on the host)."""

    def __init__(self, files, device=None, chunk_bytes=256 << 20):
        self.dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.infos, self.where, self.chunks = [], [], []
        self._stage = None
        pending, size = [], 0
        for i, b in enumerate(files):
            try:
                self.infos.append(parse(b))
            except ValueError as e:
                raise ValueError(f"JpegStore: file {i}: {e}") from None
            b = np.frombuffer(b, np.uint8) if not isinstance(b, np.ndarray) else b.reshape(-1).view(np.uint8)
            if pending and size + len(b) > chunk_bytes:
                self._upload(pending, size, chunk_bytes)
                pending, size = [], 0
            self.where.append((len(self.chunks), size))
            pending.append(b)
            size += len(b)
        if pending:
            self._upload(pending, size, chunk_bytes)
        self._stage = None

    def _upload(self, pending, size, chunk_bytes):
        if self._stage is None or self._stage.numel() < size:
            self._stage = torch.empty(max(size, chunk_bytes), dtype=torch.uint8, pin_memory=True)
        host, o = self._stage.numpy(), 0
        for b in pending:
            host[o:o + len(b)] = b
            o += len(b)
        with torch.cuda.device(self.dev):
            chunk = torch.empty(size, dtype=torch.uint8, device=self.dev)
            chunk.copy_(self._stage[:size], non_blocking=True)
            torch.cuda.current_stream(self.dev).synchronize()      # the staging buffer is refilled next
        self.chunks.append(chunk)

    def address(self, i):
        """Device address of file i's first byte."""
        c, off = self.where[i]
        return self.chunks[c].data_ptr() + off

    def __len__(self):
        return len(self.infos)


class JpegDecoder:
    """Decodes batches of JPEGs on `device` into uint8 BGR HWC frames, byte-identical to cv2.imread.

    `decode(sources, stream=None, store=None)`: `sources` maps a caller's index to a JPEG file (bytes-like, staged through
    pinned memory) or, with `store`, to an index into that `JpegStore`.  Returns ({index: frame}, ready): every frame is a
    CUDA tensor, a slice of one arena per call, written on `stream` (default: the current stream) before the event `ready`.
    Nothing synchronises the host; headers are parsed on the host first (ValueError, before anything is enqueued, naming
    the index of a refused file).  `check()` waits for the decodes since the last check and raises ValueError naming every
    source whose entropy data was corrupt (those frames' pixels are unspecified)."""

    def __init__(self, device=None):
        self.dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.pending = []

    def decode(self, sources, stream=None, store=None):
        keys = list(sources)
        infos, host_bytes = [], []
        for k in keys:
            if store is not None:
                infos.append(store.infos[sources[k]])
            else:
                b = sources[k]
                try:
                    infos.append(parse(b))
                except ValueError as e:
                    raise ValueError(f"JpegDecoder: source {k!r}: {e}") from None
                host_bytes.append(b)
        n = len(keys)
        tables, table_idx = [], {}

        def table(key):
            if key not in table_idx:
                table_idx[key] = len(tables)
                tables.append(_TABLES[key])
            return table_idx[key]

        recs = (_lib.JpegImage * max(n, 1))()
        out_off, out_total = [], 0
        for j, info in enumerate(infos):
            r = recs[j]
            r.height, r.width, r.ncomp, r.orientation, r.restart = info.height, info.width, len(info.comps), info.orientation, info.restart
            r.len = info.scan[1] - info.scan[0]
            for c, ((h, v, q, _, _), (dc, ac)) in enumerate(zip(info.comps, info.tables)):
                r.comp[c].h, r.comp[c].v = h, v
                r.comp[c].dc, r.comp[c].ac = table(dc), table(ac)
                C.memmove(C.addressof(r.comp[c].q), q.ctypes.data, 128)
            out_off.append(out_total)
            out_total += (info.height * info.width * 3 + 15) & ~15
        ws_bytes = _lib.lib().yv6_jpeg_workspace_bytes(recs, n)
        if ws_bytes < 0:
            raise ValueError(f"JpegDecoder: {_lib.lib().yv6_last_error().decode()}")
        seg = [info.scan[1] - info.scan[0] for info in infos]
        rec_b = C.sizeof(recs)
        tab_off = (rec_b + 15) & ~15
        src_off = tab_off + len(tables) * C.sizeof(_lib.JpegHuff)
        staged = sum(seg) if store is None else 0
        s = stream if stream is not None else torch.cuda.current_stream(self.dev)
        with torch.cuda.device(self.dev), torch.cuda.stream(s):
            host = torch.empty(src_off + staged, dtype=torch.uint8, pin_memory=True)
            dev = torch.empty(src_off + staged, dtype=torch.uint8, device=self.dev)
            out = torch.empty(max(out_total, 1), dtype=torch.uint8, device=self.dev)
            ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=self.dev)
            status = torch.empty(max(n, 1), dtype=torch.int32, device=self.dev)
            o, hv = src_off, host.numpy()
            for j, info in enumerate(infos):
                a, e = info.scan
                if store is None:
                    hv[o:o + seg[j]] = np.frombuffer(host_bytes[j], np.uint8)[a:e]
                    recs[j].data = dev.data_ptr() + o
                    o += seg[j]
                else:
                    recs[j].data = store.address(sources[keys[j]]) + a
                recs[j].out = out.data_ptr() + out_off[j]
            C.memmove(host.data_ptr(), recs, rec_b)
            for i, t in enumerate(tables):
                C.memmove(host.data_ptr() + tab_off + i * C.sizeof(t), C.addressof(t), C.sizeof(t))
            dev.copy_(host, non_blocking=True)
            if n:
                _lib.check(_lib.lib().yv6_jpeg_decode(_lib.handle(self.dev.index), dev.data_ptr(), n, dev.data_ptr() + tab_off,
                                                      ws.data_ptr(), status.data_ptr(), _lib.stream_ptr(s)))
            ready = torch.cuda.Event()
            ready.record(s)
        frames = {k: out[out_off[j]:out_off[j] + info.height * info.width * 3].view(*info.shape) for j, (k, info) in enumerate(zip(keys, infos))}
        self.pending.append((keys, status, ready))
        return frames, ready

    def check(self):
        """Synchronise with the decodes since the last check; ValueError naming every source flagged as corrupt."""
        pending, self.pending = self.pending, []
        bad = []
        for keys, status, ready in pending:
            ready.synchronize()
            for k, v in zip(keys, status.cpu().tolist()):
                if v:
                    bad.append(f"{k!r}: {STATUS.get(v, v)}")
        if bad:
            raise ValueError("JpegDecoder: corrupt entropy data in " + "; ".join(bad))
