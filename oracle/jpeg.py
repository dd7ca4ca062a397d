"""A numpy restatement of the JPEG decode cv2.imread performs (libjpeg-turbo with its defaults), written from ITU-T T.81
and libjpeg's documented algorithms; the reference for csrc/yv6_jpeg.cu.

Header parsing is the product's host code (`yolov6_b200.jpeg.parse`: marker walk, tables, EXIF orientation), whose shapes
the goldens pin; everything from the entropy-coded bytes to the BGR frame is restated here:
  - Huffman decoding of the unstuffed scan, restart intervals resetting the DC predictors (T.81 F.2.2);
  - dequantisation and the integer ISLOW IDCT (CONST_BITS 13, PASS1_BITS 2) with libjpeg's post-IDCT range limit, which
    wraps the descaled value modulo 1024 before clamping;
  - chroma upsampling: libjpeg-turbo's fancy (triangle) filters for h2v1 and h2v2 (when the chroma is more than two
    samples wide) and h1v2, replication otherwise; the row above the first and below the last *real* chroma row (not the
    block padding) repeat those rows, and the column beyond each edge repeats the edge column;
  - the fixed-point (16-bit) YCbCr -> RGB tables with range limiting, and gray replicated to three channels;
  - cv2's EXIF orientation: 2 flip x, 3 flip both, 4 flip y, 5 transpose, 6 transpose + flip x, 7 transpose + flip both,
    8 transpose + flip y.
"""
import numpy as np

from yolov6_b200.jpeg import ZIGZAG, parse


def _intervals(a, start, end):
    """Unstuffed byte strings of each restart interval of the segment a[start:end]."""
    out, cur, i = [], bytearray(), start
    while i < end:
        x = a[i]
        if x == 0xFF and i + 1 < end:
            y = a[i + 1]
            if y == 0x00:
                cur.append(0xFF)
                i += 2
                continue
            if 0xD0 <= y <= 0xD7:
                out.append(bytes(cur))
                cur = bytearray()
                i += 2
                continue
            i += 1                      # fill byte
            continue
        cur.append(x)
        i += 1
    out.append(bytes(cur))
    return out


class _Huff:
    def __init__(self, bits, vals):
        self.codes = {}
        code = k = 0
        for l in range(1, 17):
            for _ in range(bits[l - 1]):
                self.codes[(l, code)] = vals[k]
                code += 1
                k += 1
            code <<= 1


class DecodeError(ValueError):
    pass


def _decode_interval(data, comps, nmcu, blocks_per_mcu, coef, blk0, preds):
    """Decode nmcu MCUs of one interval into coef[blk0:], DC as differences added to `preds` (per component)."""
    buf = data + b"\x00" * 8
    nbits = 8 * len(data)
    pos = 0

    def bits(n):
        nonlocal pos
        if n == 0:
            return 0
        v = int.from_bytes(buf[pos >> 3:(pos >> 3) + 4], "big")
        r = (v >> (32 - (pos & 7) - n)) & ((1 << n) - 1)
        pos += n
        return r

    def sym(h):
        code = 0
        for l in range(1, 17):
            code = (code << 1) | bits(1)
            s = h.codes.get((l, code))
            if s is not None:
                return s
        raise DecodeError("invalid Huffman code")

    def extend(v, s):
        return v - (1 << s) + 1 if v < (1 << (s - 1)) else v

    b = blk0
    for _ in range(nmcu):
        for ci in blocks_per_mcu:
            dc, ac = comps[ci][3], comps[ci][4]
            s = sym(dc)
            diff = extend(bits(s), s) if s else 0
            preds[ci] += diff
            blk = coef[b]
            blk[0] = preds[ci]
            k = 1
            while k < 64:
                rs = sym(ac)
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    if k > 63:
                        raise DecodeError("AC run-length past coefficient 63")
                    blk[ZIGZAG[k]] = extend(bits(s), s)
                    k += 1
                elif r == 15:
                    k += 16
                else:
                    break
            b += 1
        if pos > nbits:
            raise DecodeError("entropy data ran out")
    return b


C13 = {k: v for k, v in dict(F0298=2446, F0390=3196, F0541=4433, F0765=6270, F0899=7373, F1175=9633, F1501=12299, F1847=15137,
                              F1961=16069, F2053=16819, F2562=20995, F3072=25172).items()}


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, shift):
    c = C13
    z1 = (x2 + x6) * c["F0541"]
    tmp2 = z1 - x6 * c["F1847"]
    tmp3 = z1 + x2 * c["F0765"]
    tmp0 = (x0 + x4) << 13
    tmp1 = (x0 - x4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = x7, x5, x3, x1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * c["F1175"]
    o0, o1, o2, o3 = o0 * c["F0298"], o1 * c["F2053"], o2 * c["F3072"], o3 * c["F1501"]
    z1, z2 = -z1 * c["F0899"], -z2 * c["F2562"]
    z3, z4 = -z3 * c["F1961"] + z5, -z4 * c["F0390"] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    d = lambda v: (v + (1 << (shift - 1))) >> shift
    return [d(t10 + o3), d(t11 + o2), d(t12 + o1), d(t13 + o0), d(t13 - o0), d(t12 - o1), d(t11 - o2), d(t10 - o3)]


def idct_islow(coef, q):
    """libjpeg's jpeg_idct_islow of blocks coef [N, 64] (natural order) with quant table q [64] -> uint8 [N, 8, 8]."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * q.astype(np.int64).reshape(8, 8)
    ws = np.stack(_idct_1d(*[x[:, r, :] for r in range(8)], 11), 1)           # columns: ws[:, row, col]
    out = np.stack(_idct_1d(*[ws[:, :, c] for c in range(8)], 18), 2)         # rows
    j = out & 1023
    return np.where(j < 128, j + 128, np.where(j < 512, 255, np.where(j < 896, 0, j - 896))).astype(np.uint8)


def _upsample(p, dh, dw, h, v, H, W):
    """Chroma plane p (real part dh x dw) to the luma grid (H x W) as libjpeg-turbo does with fancy upsampling on."""
    p = p[:dh, :dw].astype(np.int64)
    if (h, v) == (1, 1):
        return p[:H, :W]
    if (h, v) == (2, 1) and dw > 2:
        l, r = np.pad(p, ((0, 0), (1, 0)), mode="edge")[:, :-1], np.pad(p, ((0, 0), (0, 1)), mode="edge")[:, 1:]
        o = np.empty((dh, 2 * dw), np.int64)
        o[:, 0::2], o[:, 1::2] = (3 * p + l + 1) >> 2, (3 * p + r + 2) >> 2
        return o[:H, :W]
    if (h, v) == (1, 2):
        u, d = np.pad(p, ((1, 0), (0, 0)), mode="edge")[:-1], np.pad(p, ((0, 1), (0, 0)), mode="edge")[1:]
        o = np.empty((2 * dh, dw), np.int64)
        o[0::2], o[1::2] = (3 * p + u + 1) >> 2, (3 * p + d + 2) >> 2
        return o[:H, :W]
    if (h, v) == (2, 2) and dw > 2:
        u, d = np.pad(p, ((1, 0), (0, 0)), mode="edge")[:-1], np.pad(p, ((0, 1), (0, 0)), mode="edge")[1:]
        o = np.empty((2 * dh, 2 * dw), np.int64)
        for row, nb in ((0, u), (1, d)):
            cs = 3 * p + nb
            l, r = np.pad(cs, ((0, 0), (1, 0)), mode="edge")[:, :-1], np.pad(cs, ((0, 0), (0, 1)), mode="edge")[:, 1:]
            o[row::2, 0::2], o[row::2, 1::2] = (3 * cs + l + 8) >> 4, (3 * cs + r + 7) >> 4
        return o[:H, :W]
    return np.repeat(np.repeat(p, v, 0), h, 1)[:H, :W]


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_bgr(y, cb, cr):
    cb, cr = cb - 128, cr - 128
    r = y + ((_fix(1.40200) * cr + 32768) >> 16)
    g = y + ((-_fix(0.34414) * cb + 32768 - _fix(0.71414) * cr) >> 16)
    b = y + ((_fix(1.77200) * cb + 32768) >> 16)
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def orient(img, o):
    if o >= 5:
        img = img.transpose(1, 0, 2)
    return {1: img, 2: img[:, ::-1], 3: img[::-1, ::-1], 4: img[::-1], 5: img, 6: img[:, ::-1], 7: img[::-1, ::-1],
            8: img[::-1]}[o].copy()


def decode(buf):
    """cv2.imread's uint8 BGR HWC array of one supported JPEG (ValueError from `parse` otherwise, DecodeError on corrupt
    entropy data)."""
    info = parse(buf)
    a = np.frombuffer(bytes(buf), np.uint8)
    H, W, comps = info.height, info.width, info.comps
    hm, vm = max(c[0] for c in comps), max(c[1] for c in comps)
    if len(comps) == 1:
        mx, my = -(-W // 8), -(-H // 8)
    else:
        mx, my = -(-W // (8 * hm)), -(-H // (8 * vm))
    bpm = [ci for ci, c in enumerate(comps) for _ in range(c[0] * c[1])]
    nmcu = mx * my
    ri = info.restart or nmcu
    coef = np.zeros((nmcu * len(bpm), 64), np.int64)
    ivs = _intervals(a, *info.scan)
    huffs = [(None, None, None, _Huff(*c[3]), _Huff(*c[4])) for c in comps]
    b = 0
    for k in range(-(-nmcu // ri)):
        data = ivs[k] if k < len(ivs) else b""
        b = _decode_interval(data, huffs, min(ri, nmcu - k * ri), bpm, coef, b, [0] * len(comps))
    planes = []
    for ci, (h, v, q, _, _) in enumerate(comps):
        sel = np.array([i for i in range(len(bpm)) if bpm[i] == ci])
        blocks = coef.reshape(nmcu, len(bpm), 64)[:, sel].reshape(my, mx, v, h, 64)
        pix = idct_islow(blocks.reshape(-1, 64), q).reshape(my, mx, v, h, 8, 8)
        plane = pix.transpose(0, 2, 4, 1, 3, 5).reshape(my * v * 8, mx * h * 8)
        dh, dw = -(-H * v // vm), -(-W * h // hm)
        planes.append(_upsample(plane, dh, dw, hm // h, vm // v, H, W))
    if len(planes) == 1:
        img = np.repeat(planes[0][..., None], 3, 2).astype(np.uint8)
    else:
        img = ycc_to_bgr(*planes)
    return orient(img, info.orientation)
