"""Oracle for baseline JPEG decoding (TEST INFRASTRUCTURE — see oracle/__init__.py).

What the reference reads: `Image.open(path).convert("RGB")` (dataset/basedataset.py:234-241), i.e. Pillow driving
libjpeg-turbo with its defaults (no draft mode): JDCT_ISLOW, fancy upsampling, out_color_space RGB (3 components) or
GRAYSCALE (1 component, replicated by convert("RGB")).  Restated here for the files the device decoder takes
(visiondk_b200/csrc/jpeg.cu): one SOF0/SOF1 frame of 8-bit samples, one interleaved Huffman scan over all components,
1 component or 3 components in YCbCr, sampling 4:4:4 / 4:2:2 (h2v1) / 4:2:0 (h2v2) / 4:4:0 (h1v2), any restart interval.
Pinned bit for bit against the installed Pillow by tests/test_jpeg_cpu.py.

  * Huffman decode: canonical codes per DHT; DC difference added to the component's predictor (int), stored as the 16-bit
    JCOEF; AC run/size pairs in zig-zag order; a restart resets the predictors and the bit buffer.
  * jidctint.c jpeg_idct_islow: dequantise with the table cast to 16 bits (ISLOW_MULT_TYPE), CONST_BITS 13, PASS1_BITS 2,
    columns then rows, pass-1 results stored as int, outputs through the IDCT range-limit table indexed by x & RANGE_MASK.
    The zero-AC shortcuts of both passes give the same numbers as the full computation, so they are not restated.
  * jdsample.c: h2v1 / h2v2 fancy (triangle) upsampling over downsampled_width when it is > 2, plain replication
    otherwise; h1v2 fancy always.  Vertical context: the row above row 0 is row 0, the row below the last real row is that
    row (jdmainct.c's wraparound and bottom pointers).
  * jdcolor.c ycc_rgb_convert: SCALEBITS 16 tables with ONE_HALF rounding, clamped through the sample range limit.
"""
from __future__ import annotations

import numpy as np

NATURAL_ORDER = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63], np.int64)

# fallback reasons, the same codes as VDK_JPEG_* in include/vdk_b200.h
DEVICE, NOT_JPEG, PROCESS, PRECISION, COLOR, SAMPLING, SCAN, MALFORMED, MPO, RESTART, TOO_LARGE = range(11)


class Unsupported(Exception):
    def __init__(self, reason: int, what: str):
        super().__init__(what)
        self.reason = reason


def _ceil_div(a, b):
    return -(-a // b)


def pillow_reads_app(m: int, s: bytes) -> bool:
    """False for the short application segments on which Pillow's own header reader (JpegImagePlugin.APP, and SOF's ICC
    fix-up) raises before libjpeg runs."""
    if (m == 0xE0 and s.startswith(b"JFIF")) or (m == 0xEE and s.startswith(b"Adobe")):
        return len(s) >= 7
    if m == 0xE2 and s.startswith(b"ICC_PROFILE\0"):
        return len(s) >= 14
    if m == 0xED and s.startswith(b"Photoshop 3.0\x00"):
        off = 14
        while s[off:off + 4] == b"8BIM":
            off += 4
            if off + 2 > len(s):
                return True
            off += 2
            if off >= len(s):
                return False
            off += 1 + s[off]
            off += off & 1
            if off + 4 > len(s):
                return True
            off += 4 + int.from_bytes(s[off:off + 4], "big")
            off += off & 1
    return True


def parse(data: bytes) -> dict:
    """Marker walk -> header dict, or Unsupported(reason) for a file the device path leaves to the host."""
    if len(data) < 3 or data[:3] != b"\xff\xd8\xff":
        raise Unsupported(NOT_JPEG, "no SOI")
    n = len(data)
    pos = 2
    qt, dht = {}, {}
    frame = None
    restart = 0
    jfif = adobe = False
    adobe_transform = -1
    while True:
        while pos < n and data[pos] == 0xFF:  # fill bytes
            pos += 1
        if pos >= n:
            raise Unsupported(MALFORMED, "end of data before SOS")
        m = data[pos]
        pos += 1
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7 or m == 0xD9:
            raise Unsupported(MALFORMED, f"marker {m:02x} before SOS")
        if pos + 2 > n:
            raise Unsupported(MALFORMED, "truncated segment")
        ln = (data[pos] << 8) | data[pos + 1]
        if ln < 2 or pos + ln > n:
            raise Unsupported(MALFORMED, "bad segment length")
        seg = data[pos + 2:pos + ln]
        pos += ln
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise Unsupported(MALFORMED, "two frames")
            if len(seg) < 6:
                raise Unsupported(MALFORMED, "short SOF")
            prec, h, w, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) != 6 + 3 * nf:
                raise Unsupported(MALFORMED, "SOF length")
            if prec != 8:
                raise Unsupported(PRECISION, f"{prec}-bit samples")
            if h == 0 or w == 0:
                raise Unsupported(MALFORMED, "zero size (DNL)")
            if h > 65500 or w > 65500:
                raise Unsupported(TOO_LARGE, "side above JPEG_MAX_DIMENSION")
            comps = [dict(id=seg[6 + 3 * i], h=seg[7 + 3 * i] >> 4, v=seg[7 + 3 * i] & 15, tq=seg[8 + 3 * i]) for i in range(nf)]
            frame = dict(width=w, height=h, comps=comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported(PROCESS, f"SOF{m - 0xC0}")
        elif m == 0xCC:
            raise Unsupported(PROCESS, "arithmetic conditioning")
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise Unsupported(MALFORMED, "short DHT")
                tc, th = seg[i] >> 4, seg[i] & 15
                counts = list(seg[i + 1:i + 17])
                total = sum(counts)
                if tc > 1 or th > 3 or total > 256 or i + 17 + total > len(seg):
                    raise Unsupported(MALFORMED, "bad DHT")
                vals = list(seg[i + 17:i + 17 + total])
                dht[(tc, th)] = (counts, vals)
                i += 17 + total
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + size > len(seg):
                    raise Unsupported(MALFORMED, "bad DQT")
                raw = seg[i + 1:i + 1 + size]
                zz = [(raw[2 * k] << 8) | raw[2 * k + 1] for k in range(64)] if pq else list(raw)
                q = np.zeros(64, np.int64)
                q[NATURAL_ORDER] = zz
                qt[tq] = q
                i += 1 + size
        elif m == 0xDD:
            if len(seg) != 2:
                raise Unsupported(MALFORMED, "DRI length")
            restart = (seg[0] << 8) | seg[1]
        elif 0xE0 <= m <= 0xEF and not pillow_reads_app(m, seg):
            raise Unsupported(MALFORMED, "Image.open refuses this application segment")
        elif m == 0xE0:
            jfif = jfif or (len(seg) >= 14 and seg[:5] == b"JFIF\x00")
        elif m == 0xE2 and seg[:4] == b"MPF\x00":
            raise Unsupported(MPO, "MPO")
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe, adobe_transform = True, seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            return _sos(data, pos, seg, frame, qt, dht, restart, jfif, adobe, adobe_transform)
        else:
            raise Unsupported(MALFORMED, f"marker {m:02x}")


def _sos(data, pos, seg, frame, qt, dht, restart, jfif, adobe, adobe_transform):
    if frame is None:
        raise Unsupported(MALFORMED, "SOS before SOF")
    comps = frame["comps"]
    nf = len(comps)
    if nf not in (1, 3):
        raise Unsupported(COLOR, f"{nf} components")
    if nf == 3:
        ids = [c["id"] for c in comps]
        if jfif:
            pass
        elif adobe:
            if adobe_transform != 1:
                raise Unsupported(COLOR, f"Adobe transform {adobe_transform}")
        elif ids == [82, 71, 66]:
            raise Unsupported(COLOR, "RGB component ids")
        hv = [(c["h"], c["v"]) for c in comps]
        if hv[1:] != [(1, 1), (1, 1)] or hv[0] not in ((1, 1), (2, 1), (2, 2), (1, 2)):
            raise Unsupported(SAMPLING, f"sampling {hv}")
    else:
        if not (1 <= comps[0]["h"] <= 4 and 1 <= comps[0]["v"] <= 4):
            raise Unsupported(MALFORMED, "sampling factor")
    if len(seg) < 1 or len(seg) != 4 + 2 * seg[0]:
        raise Unsupported(MALFORMED, "SOS length")
    ns = seg[0]
    if ns != nf:
        raise Unsupported(SCAN, "scan does not cover every component")
    sel = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
    if [s[0] for s in sel] != [c["id"] for c in comps]:
        raise Unsupported(SCAN, "scan order differs from frame order")
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if ss != 0 or se != 63 or ahal != 0:
        raise Unsupported(MALFORMED, "spectral selection of a sequential scan")
    for c, (_, td, ta) in zip(comps, sel):
        if c["tq"] not in qt or (0, td) not in dht or (1, ta) not in dht:
            raise Unsupported(MALFORMED, "missing table")
        c["q"], c["dc"], c["ac"] = qt[c["tq"]], _huff(*dht[(0, td)], True), _huff(*dht[(1, ta)], False)
    # entropy-coded data: up to the first marker that is not RSTn, which must be EOI (anything else: another scan)
    n = len(data)
    segments, p, start, expect = [], pos, pos, 0
    while True:
        p = data.find(b"\xff", p)
        if p < 0 or p + 1 >= n:
            raise Unsupported(MALFORMED, "end of data inside the scan")
        b = data[p + 1]
        if b == 0x00:
            p += 2
            continue
        if b == 0xFF:  # fill byte before a marker
            p += 1
            continue
        if 0xD0 <= b <= 0xD7:
            if not restart or b != 0xD0 + expect:
                raise Unsupported(RESTART, "unexpected RST")
            expect = (expect + 1) & 7
            segments.append((start, p))
            p += 2
            start = p
            continue
        segments.append((start, p))
        if b != 0xD9:
            raise Unsupported(SCAN, f"marker {b:02x} after the scan")
        break
    hmax, vmax = (max(c["h"] for c in comps), max(c["v"] for c in comps)) if nf == 3 else (1, 1)
    w, h = frame["width"], frame["height"]
    if nf == 1:
        comps[0]["h"] = comps[0]["v"] = 1
    mx, my = _ceil_div(w, 8 * hmax), _ceil_div(h, 8 * vmax)
    if len(segments) != (_ceil_div(mx * my, restart) if restart else 1):
        raise Unsupported(RESTART, "restart count")
    return dict(width=w, height=h, comps=comps, hmax=hmax, vmax=vmax, mcus_x=mx, mcus_y=my, restart=restart,
                segments=segments)


def _huff(counts, vals, is_dc):
    """16-bit lookahead tables (code length, symbol) of one canonical Huffman table (jdhuff.c jpeg_make_d_derived_tbl)."""
    length = np.zeros(1 << 16, np.int64)
    symbol = np.zeros(1 << 16, np.int64)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(counts[l - 1]):
            lo = code << (16 - l)
            length[lo:lo + (1 << (16 - l))] = l
            symbol[lo:lo + (1 << (16 - l))] = vals[k]
            code += 1
            k += 1
        if code >= (1 << l):  # no code may be all ones
            raise Unsupported(MALFORMED, "over-subscribed Huffman table")
        code <<= 1
    if is_dc and any(v > 15 for v in vals):
        raise Unsupported(MALFORMED, "DC symbol > 15")
    return length, symbol


def _windows(seg: bytes) -> np.ndarray:
    """The 16-bit window starting at every bit of an un-stuffed entropy segment (zeros past its end)."""
    raw = np.frombuffer(seg.replace(b"\xff\x00", b"\xff"), np.uint8)
    bits = np.concatenate([np.unpackbits(raw).astype(np.int64), np.zeros(48, np.int64)])
    nb = len(bits) - 32
    win = np.zeros(nb, np.int64)
    for i in range(16):
        win = (win << 1) | bits[i:i + nb]
    return win, 8 * len(raw)


def _extend(r, s):
    return r - (1 << s) + 1 if r < (1 << (s - 1)) else r


def entropy_decode(data: bytes, hdr: dict):
    """-> int16 coefficient arrays [bh, bw, 64] (natural order) per component, or Unsupported for a malformed stream."""
    comps = hdr["comps"]
    mx, my = hdr["mcus_x"], hdr["mcus_y"]
    coef = [np.zeros((my * c["v"], mx * c["h"], 64), np.int64) for c in comps]
    total = mx * my
    per = hdr["restart"] or total
    for sidx, (a, b) in enumerate(hdr["segments"]):
        win, nbits = _windows(data[a:b])
        pos = 0
        pred = [0] * len(comps)
        for m in range(sidx * per, min(total, (sidx + 1) * per)):
            y0, x0 = divmod(m, mx)
            for ci, c in enumerate(comps):
                dl, ds = c["dc"]
                al, asym = c["ac"]
                for by in range(c["v"]):
                    for bx in range(c["h"]):
                        blk = coef[ci][y0 * c["v"] + by, x0 * c["h"] + bx]
                        if pos > nbits:
                            raise Unsupported(MALFORMED, "entropy data ends before the last MCU of its interval")
                        v = int(win[pos])
                        l = int(dl[v])
                        if l == 0:
                            raise Unsupported(MALFORMED, "bad Huffman code")
                        s = int(ds[v])
                        pos += l
                        if s:
                            r = int(win[pos]) >> (16 - s)
                            pos += s
                            pred[ci] += _extend(r, s)
                        blk[0] = ((pred[ci] + 32768) & 0xFFFF) - 32768
                        k = 1
                        while k < 64:
                            if pos > nbits:
                                raise Unsupported(MALFORMED, "entropy data ends before the last MCU of its interval")
                            v = int(win[pos])
                            l = int(al[v])
                            if l == 0:
                                raise Unsupported(MALFORMED, "bad Huffman code")
                            rs = int(asym[v])
                            pos += l
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                if k > 63:
                                    raise Unsupported(MALFORMED, "AC run past coefficient 63")
                                blk[NATURAL_ORDER[k]] = _extend(int(win[pos]) >> (16 - s), s)
                                pos += s
                            elif r == 15:
                                k += 15
                                if k > 63:
                                    raise Unsupported(MALFORMED, "AC run past coefficient 63")
                            else:
                                break
                            k += 1
            if pos > nbits:
                raise Unsupported(MALFORMED, "entropy data ends before the last MCU of its interval")
        if nbits - pos >= 8:
            raise Unsupported(MALFORMED, "extraneous bytes before a marker")
    return [c.astype(np.int16) for c in coef]


CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(c, shift):
    """One jpeg_idct_islow pass over axis 1 of c [N, 8] (int64)."""
    z2, z3 = c[:, 2], c[:, 6]
    z1 = (z2 + z3) * F0541
    tmp2 = z1 + z3 * -F1847
    tmp3 = z1 + z2 * F0765
    tmp0 = (c[:, 0] + c[:, 4]) << CONST_BITS
    tmp1 = (c[:, 0] - c[:, 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = c[:, 7], c[:, 5], c[:, 3], c[:, 1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = z1 * -F0899, z2 * -F2562, z3 * -F1961 + z5, z4 * -F0390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    out = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return np.stack([_descale(v, shift) for v in out], axis=1)


def _idct_range_limit(x):
    t = x & 1023
    return np.where(t < 128, t + 128, np.where(t < 512, 255, np.where(t < 896, 0, t - 896))).astype(np.uint8)


def idct_islow(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """int16 [bh, bw, 64] + quantisation table (natural order) -> uint8 plane [bh * 8, bw * 8]."""
    bh, bw = coef.shape[:2]
    q16 = ((q.astype(np.int64) + 32768) & 0xFFFF) - 32768  # ISLOW_MULT_TYPE is 16-bit
    blocks = (coef.reshape(-1, 64).astype(np.int64) * q16).reshape(-1, 8, 8)  # [N, row u, col]
    cols = blocks.transpose(0, 2, 1).reshape(-1, 8)  # one column per row of `cols`
    ws = _idct_1d(cols, CONST_BITS - PASS1_BITS)  # [N * 8 columns, 8 rows]
    ws = ((ws + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)  # stored as int
    ws = ws.reshape(-1, 8, 8).transpose(0, 2, 1).reshape(-1, 8)  # one row per row
    px = _idct_range_limit(_idct_1d(ws, CONST_BITS + PASS1_BITS + 3))
    return px.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(plane: np.ndarray, dw: int, dh: int, hf: int, vf: int) -> np.ndarray:
    """jdsample.c for a chroma plane cropped to downsampled_width x downsampled_height -> [dh * vf, dw * hf]."""
    p = plane[:dh, :dw].astype(np.int64)
    if vf == 2:
        above = np.concatenate([p[:1], p[:-1]])
        below = np.concatenate([p[1:], p[-1:]])
        if hf == 2 and dw <= 2:
            return np.repeat(np.repeat(p, 2, 0), 2, 1).astype(np.uint8)
        up, down = 3 * p + above, 3 * p + below  # column sums of the two output rows of every input row
        if hf == 1:
            out = np.empty((2 * dh, dw), np.int64)
            out[0::2], out[1::2] = (up + 1) >> 2, (down + 2) >> 2
            return out.astype(np.uint8)
        out = np.empty((2 * dh, 2 * dw), np.int64)
        for r, cs in ((0, up), (1, down)):
            left = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
            right = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
            out[r::2, 0::2] = (3 * cs + left + 8) >> 4
            out[r::2, 1::2] = (3 * cs + right + 7) >> 4
        return out.astype(np.uint8)
    if hf == 2:
        if dw <= 2:
            return np.repeat(p, 2, 1).astype(np.uint8)
        out = np.empty((dh, 2 * dw), np.int64)
        out[:, 0::2] = (3 * p + np.concatenate([p[:, :1], p[:, :-1]], 1) + 1) >> 2
        out[:, 1::2] = (3 * p + np.concatenate([p[:, 1:], p[:, -1:]], 1) + 2) >> 2
        out[:, 0], out[:, -1] = p[:, 0], p[:, -1]
        return out.astype(np.uint8)
    return p.astype(np.uint8)


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
    y, cb, cr = (a.astype(np.int64) for a in (y, cb, cr))
    half = 1 << 15
    r = y + ((91881 * (cr - 128) + half) >> 16)
    g = y + ((-22554 * (cb - 128) + half - 46802 * (cr - 128)) >> 16)
    b = y + ((116130 * (cb - 128) + half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data: bytes) -> np.ndarray:
    """JPEG bytes -> uint8 [h, w, 3], what np.asarray(Image.open(f).convert("RGB")) returns.  Raises Unsupported for
    files outside the device decoder's set and for malformed streams."""
    hdr = parse(data)
    coef = entropy_decode(data, hdr)
    w, h = hdr["width"], hdr["height"]
    planes = [idct_islow(c, comp["q"]) for c, comp in zip(coef, hdr["comps"])]
    if len(planes) == 1:
        return np.repeat(planes[0][:h, :w, None], 3, axis=2)
    hmax, vmax = hdr["hmax"], hdr["vmax"]
    chroma = [upsample(p, _ceil_div(w, hmax), _ceil_div(h, vmax), hmax, vmax)[:h, :w] for p in planes[1:]]
    return ycc_to_rgb(planes[0][:h, :w], *chroma)
