"""Oracle for progressive JPEG decoding (TEST INFRASTRUCTURE — see oracle/__init__.py).

The same call as oracle/jpeg.py (`Image.open(path).convert("RGB")`, libjpeg-turbo with its defaults) on the progressive
files the device decoder takes (visiondk_b200/csrc/jpeg.cu, vdk_jpeg_parse_progressive): one SOF2 frame of 8-bit samples,
the colour spaces and samplings of the baseline set, any restart interval, and any scan script that libjpeg accepts without
a warning and that brings every coefficient of every component to full precision.  The IDCT, upsampling and colour
conversion are oracle/jpeg.py's; restated here are the scan parsing and jdphuff.c's four decoders:

  * scan checks (start_pass_phuff_decoder): a DC scan has Se = 0, an AC scan 1 <= Ss <= Se <= 63 and one component, a
    refinement has Al = Ah - 1, Al <= 13 (else JERR_BAD_PROGRESSION); per component and coefficient, Ah must equal the Al of
    the previous scan (0 if none), and an AC scan needs an earlier DC scan (else JWRN_BOGUS_PROGRESSION).
  * tables: each scan takes the DHT and DRI in force at its SOS; each component's quantisation table is latched at the
    first scan that contains it (jdinput.c latch_quant_tables).
  * geometry: a scan of several components (DC only) runs over the MCU grid; a scan of one component over that component's
    own ceil(width * h / (8 * hmax)) x ceil(height * v / (8 * vmax)) blocks.  Restart intervals count those units.
  * DC first: predictor as int, stored as (JCOEF)(value << Al).  DC refine: the next bit ORed in at Al.
  * AC first: run/size symbols with EOBRUN (2^r + r extra bits, minus the current block).  AC refine: new coefficients of
    magnitude 1 << Al, correction bits for the non-zero ones, ZRL and EOBRUN as in decode_mcu_AC_refine.
  * the dependency level of a scan: 1 + the largest level of the earlier scans that share a component and a coefficient
    with it (0 if none).
"""
from __future__ import annotations

import numpy as np

from . import jpeg as J
from .jpeg import MALFORMED, MPO, NOT_JPEG, PROCESS, RESTART, SCAN, Unsupported

DEVICE_PROGRESSIVE = 11


def _ceil_div(a, b):
    return -(-a // b)


def _colour(comps, jfif, adobe, adobe_transform):
    if len(comps) != 3:
        return
    if not jfif and adobe and adobe_transform != 1:
        raise Unsupported(J.COLOR, f"Adobe transform {adobe_transform}")
    if not jfif and not adobe and [c["id"] for c in comps] == [82, 71, 66]:
        raise Unsupported(J.COLOR, "RGB component ids")
    hv = [(c["h"], c["v"]) for c in comps]
    if hv[1:] != [(1, 1), (1, 1)] or hv[0] not in ((1, 1), (2, 1), (2, 2), (1, 2)):
        raise Unsupported(J.SAMPLING, f"sampling {hv}")


def _extent(data, pos, restart):
    """(segments [(start, end)], position of the marker that ends the scan), as oracle/jpeg.py walks a scan."""
    n = len(data)
    segments, p, start, expect = [], pos, pos, 0
    while True:
        p = data.find(b"\xff", p)
        if p < 0 or p + 1 >= n:
            raise Unsupported(MALFORMED, "end of data inside the scan")
        b = data[p + 1]
        if b == 0x00:
            p += 2
        elif b == 0xFF:
            p += 1
        elif 0xD0 <= b <= 0xD7:
            if not restart or b != 0xD0 + expect:
                raise Unsupported(RESTART, "unexpected RST")
            expect = (expect + 1) & 7
            segments.append((start, p))
            p += 2
            start = p
        else:
            segments.append((start, p))
            return segments, p


def parse(data: bytes) -> dict:
    """Marker walk of a progressive file -> header dict with its scans, or Unsupported(reason)."""
    if len(data) < 3 or data[:3] != b"\xff\xd8\xff":
        raise Unsupported(NOT_JPEG, "no SOI")
    n = len(data)
    pos = 2
    qt, dht = {}, {}
    frame = None
    restart = 0
    jfif = adobe = False
    adobe_transform = -1
    scans = []
    coef_bits = None
    while True:
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise Unsupported(MALFORMED, "end of data before EOI")
        m = data[pos]
        pos += 1
        if m == 0xD9 and scans:
            if (coef_bits != 0).any():
                raise Unsupported(SCAN, "a coefficient is unsent or not fully refined")
            frame.update(scans=scans, levels=1 + max(s["level"] for s in scans))
            return frame
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD9:
            raise Unsupported(MALFORMED, f"marker {m:02x} outside a scan")
        if pos + 2 > n:
            raise Unsupported(MALFORMED, "truncated segment")
        ln = (data[pos] << 8) | data[pos + 1]
        if ln < 2 or pos + ln > n:
            raise Unsupported(MALFORMED, "bad segment length")
        seg = data[pos + 2:pos + ln]
        pos += ln
        if m == 0xC2:
            if frame is not None:
                raise Unsupported(MALFORMED, "two frames")
            if len(seg) < 6:
                raise Unsupported(MALFORMED, "short SOF")
            prec, h, w, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) != 6 + 3 * nf:
                raise Unsupported(MALFORMED, "SOF length")
            if prec != 8:
                raise Unsupported(J.PRECISION, f"{prec}-bit samples")
            if h == 0 or w == 0:
                raise Unsupported(MALFORMED, "zero size (DNL)")
            if h > 65500 or w > 65500:
                raise Unsupported(J.TOO_LARGE, "side above JPEG_MAX_DIMENSION")
            if nf not in (1, 3):
                raise Unsupported(J.COLOR, f"{nf} components")
            comps = [dict(id=seg[6 + 3 * i], h=seg[7 + 3 * i] >> 4, v=seg[7 + 3 * i] & 15, tq=seg[8 + 3 * i]) for i in range(nf)]
            if any(not (1 <= c["h"] <= 4 and 1 <= c["v"] <= 4) or c["tq"] > 3 for c in comps):
                raise Unsupported(MALFORMED, "sampling factor or table")
            frame = dict(width=w, height=h, comps=comps)
            coef_bits = np.full((nf, 64), -1, np.int64)
        elif m in (0xC0, 0xC1):
            raise Unsupported(MALFORMED, "two frames")
        elif 0xC3 <= m <= 0xCF and m not in (0xC4, 0xC8):
            raise Unsupported(PROCESS, f"SOF{m - 0xC0}" if m != 0xCC else "arithmetic conditioning")
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
                dht[(tc, th)] = (counts, list(seg[i + 17:i + 17 + total]))
                i += 17 + total
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + size > len(seg):
                    raise Unsupported(MALFORMED, "bad DQT")
                raw = seg[i + 1:i + 1 + size]
                q = np.zeros(64, np.int64)
                q[J.NATURAL_ORDER] = [(raw[2 * k] << 8) | raw[2 * k + 1] for k in range(64)] if pq else list(raw)
                qt[tq] = q
                i += 1 + size
        elif m == 0xDD:
            if len(seg) != 2:
                raise Unsupported(MALFORMED, "DRI length")
            restart = (seg[0] << 8) | seg[1]
        elif scans and (0xE0 <= m <= 0xEF or m == 0xFE):
            pass  # libjpeg skips these between scans; Pillow's header reader stopped at the first SOS
        elif 0xE0 <= m <= 0xEF and not J.pillow_reads_app(m, seg):
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
            if frame is None:
                raise Unsupported(MALFORMED, "SOS before SOF")
            comps = frame["comps"]
            if not scans:
                _colour(comps, jfif, adobe, adobe_transform)
                nf = len(comps)
                if nf == 1:
                    comps[0]["h"] = comps[0]["v"] = 1
                hmax, vmax = max(c["h"] for c in comps), max(c["v"] for c in comps)
                frame.update(hmax=hmax, vmax=vmax, mcus_x=_ceil_div(frame["width"], 8 * hmax),
                             mcus_y=_ceil_div(frame["height"], 8 * vmax))
            scans.append(_scan(data, pos, seg, frame, qt, dht, restart, coef_bits, scans))
            pos = scans[-1]["end"]
        else:
            raise Unsupported(MALFORMED, f"marker {m:02x}")


def _scan(data, pos, seg, frame, qt, dht, restart, coef_bits, earlier):
    comps = frame["comps"]
    if len(seg) < 1 or len(seg) != 4 + 2 * seg[0] or not 1 <= seg[0] <= 4:
        raise Unsupported(MALFORMED, "SOS length")
    ns = seg[0]
    idx = []
    for i in range(ns):
        found = [c for c, comp in enumerate(comps) if comp["id"] == seg[1 + 2 * i]]
        if not found or found[-1] in idx:
            raise Unsupported(MALFORMED, "bad component id")
        if idx and found[-1] < idx[-1]:
            raise Unsupported(SCAN, "scan order differs from frame order")
        idx.append(found[-1])
    ss, se, ah, al = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15
    dc = ss == 0
    bad = se != 0 if dc else (ss > se or se > 63 or ns != 1)
    if (ah != 0 and al != ah - 1) or al > 13 or bad:
        raise Unsupported(MALFORMED, "bad progression parameters")
    for c in idx:
        cb = coef_bits[c]
        if not dc and cb[0] < 0:
            raise Unsupported(SCAN, "AC scan before the component's DC")
        for k in range(ss, se + 1):
            if ah != max(cb[k], 0):
                raise Unsupported(SCAN, "bogus progression")
            cb[k] = al
        if "q" not in comps[c]:
            if comps[c]["tq"] not in qt:
                raise Unsupported(MALFORMED, "missing quantisation table")
            comps[c]["q"] = qt[comps[c]["tq"]].copy()
    tables = []
    for i in range(ns):
        td, ta = seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15
        if dc and ah == 0:
            if (0, td) not in dht:
                raise Unsupported(MALFORMED, "missing table")
            tables.append(J._huff(*dht[(0, td)], True))
        elif not dc:
            if (1, ta) not in dht:
                raise Unsupported(MALFORMED, "missing table")
            tables.append(J._huff(*dht[(1, ta)], False))
    if ns == 1:
        c = comps[idx[0]]
        ux = _ceil_div(frame["width"] * c["h"], 8 * frame["hmax"])
        uy = _ceil_div(frame["height"] * c["v"], 8 * frame["vmax"])
    else:
        ux, uy = frame["mcus_x"], frame["mcus_y"]
    segments, end = _extent(data, pos, restart)
    if len(segments) != (_ceil_div(ux * uy, restart) if restart else 1):
        raise Unsupported(RESTART, "restart count")
    level = 0
    for e in earlier:
        if set(e["comps"]) & set(idx) and e["ss"] <= se and ss <= e["se"]:
            level = max(level, e["level"] + 1)
    return dict(comps=idx, ss=ss, se=se, ah=ah, al=al, tables=tables, restart=restart, units_x=ux, units_y=uy,
                segments=segments, end=end, level=level)


class _Bits:
    """Bit reader over one un-stuffed restart interval (zeros past its end, as libjpeg feeds them)."""

    def __init__(self, seg: bytes):
        self.win, self.nbits = J._windows(seg)
        self.pos = 0

    def get(self, s):
        if s == 0:
            return 0
        v = int(self.win[self.pos]) >> (16 - s) if self.pos < len(self.win) else 0
        self.pos += s
        return v

    def huff(self, table):
        length, symbol = table
        v = int(self.win[self.pos]) if self.pos < len(self.win) else 0
        if length[v] == 0:
            raise Unsupported(MALFORMED, "bad Huffman code")
        self.pos += int(length[v])
        return int(symbol[v])


def _wrap16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def _block(br, sc, i, blk, state):
    ss, se, ah, al = sc["ss"], sc["se"], sc["ah"], sc["al"]
    nat = J.NATURAL_ORDER
    if ss == 0:
        if ah == 0:
            s = br.huff(sc["tables"][i])
            if s:
                state["pred"][i] += J._extend(br.get(s), s)
            if not -(1 << 31) <= state["pred"][i] < (1 << 31):
                raise Unsupported(MALFORMED, "DC predictor overflow")
            blk[0] = _wrap16(state["pred"][i] << al)
        elif br.get(1):
            blk[0] = _wrap16(int(blk[0]) | (1 << al))
        return
    table = sc["tables"][0]
    if ah == 0:
        if state["eobrun"] > 0:
            state["eobrun"] -= 1
            return
        k = ss
        while k <= se:
            rs = br.huff(table)
            r, s = rs >> 4, rs & 15
            if s:
                k += r
                if k > se:
                    raise Unsupported(MALFORMED, "AC run past the band")
                blk[nat[k]] = _wrap16(J._extend(br.get(s), s) << al)
            elif r == 15:
                k += 15
            else:
                state["eobrun"] = (1 << r) - 1 + br.get(r)
                break
            k += 1
        return
    p1, m1 = 1 << al, -(1 << al)

    def correct(pos):
        if br.get(1) and (int(blk[pos]) & p1) == 0:
            blk[pos] = _wrap16(int(blk[pos]) + (p1 if blk[pos] >= 0 else m1))

    k = ss
    if state["eobrun"] == 0:
        while k <= se:
            rs = br.huff(table)
            r, s = rs >> 4, rs & 15
            if s:
                if s != 1:
                    raise Unsupported(MALFORMED, "refinement coefficient of size other than 1")
                s = p1 if br.get(1) else m1
            elif r != 15:
                state["eobrun"] = (1 << r) + br.get(r)
                break
            while True:
                pos = nat[k]
                if blk[pos] != 0:
                    correct(pos)
                else:
                    r -= 1
                    if r < 0:
                        break
                k += 1
                if k > se:
                    break
            if s:
                if k > se:
                    raise Unsupported(MALFORMED, "AC run past the band")
                blk[nat[k]] = s
            k += 1
    if state["eobrun"] > 0:
        for kk in range(k, se + 1):
            if blk[nat[kk]] != 0:
                correct(nat[kk])
        state["eobrun"] -= 1


def entropy_decode(data: bytes, hdr: dict):
    """-> int16 coefficient arrays [bh, bw, 64] (natural order, MCU-padded) per component, or Unsupported for a malformed
    stream.  Scans run in file order."""
    comps = hdr["comps"]
    mx, my = hdr["mcus_x"], hdr["mcus_y"]
    coef = [np.zeros((my * c["v"], mx * c["h"], 64), np.int64) for c in comps]
    for sc in hdr["scans"]:
        units = sc["units_x"] * sc["units_y"]
        per = sc["restart"] or units
        for sidx, (a, b) in enumerate(sc["segments"]):
            br = _Bits(data[a:b])
            state = dict(pred=[0] * len(sc["comps"]), eobrun=0)
            for u in range(sidx * per, min(units, (sidx + 1) * per)):
                uy, ux = divmod(u, sc["units_x"])
                if len(sc["comps"]) == 1:
                    _block(br, sc, 0, coef[sc["comps"][0]][uy, ux], state)
                else:
                    for i, c in enumerate(sc["comps"]):
                        for by in range(comps[c]["v"]):
                            for bx in range(comps[c]["h"]):
                                _block(br, sc, i, coef[c][uy * comps[c]["v"] + by, ux * comps[c]["h"] + bx], state)
                if br.pos > br.nbits:
                    raise Unsupported(MALFORMED, "entropy data ends before the last block of its interval")
            if br.nbits - br.pos >= 8:
                raise Unsupported(MALFORMED, "extraneous bytes before a marker")
    return [c.astype(np.int16) for c in coef]


def decode(data: bytes) -> np.ndarray:
    """Progressive JPEG bytes -> uint8 [h, w, 3], what np.asarray(Image.open(f).convert("RGB")) returns.  Raises
    Unsupported for files outside the device decoder's set and for malformed streams."""
    hdr = parse(data)
    coef = entropy_decode(data, hdr)
    w, h = hdr["width"], hdr["height"]
    planes = [J.idct_islow(c, comp["q"]) for c, comp in zip(coef, hdr["comps"])]
    if len(planes) == 1:
        return np.repeat(planes[0][:h, :w, None], 3, axis=2)
    hmax, vmax = hdr["hmax"], hdr["vmax"]
    chroma = [J.upsample(p, _ceil_div(w, hmax), _ceil_div(h, vmax), hmax, vmax)[:h, :w] for p in planes[1:]]
    return J.ycc_to_rgb(planes[0][:h, :w], *chroma)
