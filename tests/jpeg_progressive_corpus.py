"""Seeded progressive JPEG corpus of the progressive decoder tests (tests/test_jpeg_progressive_cpu.py,
tests/test_jpeg_progressive_gpu.py): Pillow's `progressive=True` and cv2's IMWRITE_JPEG_PROGRESSIVE over the baseline
corpus's sizes, subsamplings, contents, qualities, custom tables and restart intervals, plus files written by a small
progressive re-encoder with scan scripts no library encoder writes by default."""
from __future__ import annotations

import io
import itertools

import numpy as np
from PIL import Image

from jpeg_corpus import CONTENTS, QUALITIES, SIZES, SUBSAMPLINGS, content
from oracle import jpeg as J

RESTARTS = [None, "blocks", "rows", "cv2", "cv2_none"]


def encode_progressive(a: np.ndarray, sub, quality, restart) -> bytes:
    """Progressive JPEG bytes of RGB `a`: cv2 for 4:4:0 and the cv2 restart cases, Pillow otherwise."""
    q = 90 if isinstance(quality, str) else quality
    if sub == "440" or restart in ("cv2", "cv2_none"):
        import cv2
        params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
        if sub != "gray":
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, {0: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 1: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                                                          2: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420,
                                                          "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440}[sub]]
        if restart == "cv2":
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, 3]
        img = a[:, :, 0] if sub == "gray" else cv2.cvtColor(a, cv2.COLOR_RGB2BGR)
        ok, buf = cv2.imencode(".jpg", img, params)
        assert ok
        return buf.tobytes()
    im = Image.fromarray(a[:, :, 0]) if sub == "gray" else Image.fromarray(a)
    kw = dict(quality=q, progressive=True)
    if sub != "gray":
        kw["subsampling"] = sub
    if quality == "qtables":
        kw["qtables"] = [list(range(1, 65)), [max(1, 255 - 3 * i) for i in range(64)]]
        del kw["quality"]
    if quality == "optimize":
        kw["optimize"] = True
    if restart == "blocks":
        kw["restart_marker_blocks"] = 5
    if restart == "rows":
        kw["restart_marker_rows"] = 1
    if "quality" in kw and kw["quality"] < 95 and a.size >= 3 * 500 * 375 and (a % 255 == 0).all():
        kw["quality"] = 95  # Pillow's progressive buffer holds w * h bytes below quality 95: too few for saturated noise
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


# ---------------------------------------------------------------------------------------------------- progressive re-encoder
def _optimal_table(freq: dict):
    """(counts[16], symbols) of the length-limited optimal code for symbol frequencies `freq` (jchuff.c
    jpeg_gen_optimal_table: a reserved code point keeps every code from being all ones)."""
    f = [0] * 257
    for s, c in freq.items():
        f[s] = c
    f[256] = 1
    size, others = [0] * 257, [-1] * 257
    while True:
        c1 = c2 = -1
        v = 1 << 60
        for i in range(257):
            if f[i] and f[i] <= v:
                v, c1 = f[i], i
        v = 1 << 60
        for i in range(257):
            if f[i] and f[i] <= v and i != c1:
                v, c2 = f[i], i
        if c2 < 0:
            break
        f[c1] += f[c2]
        f[c2] = 0
        size[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            size[c1] += 1
        others[c1] = c2
        size[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            size[c2] += 1
    bits = [0] * 33
    for i in range(257):
        if size[i]:
            bits[size[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1  # the reserved code point
    symbols = [s for length in range(1, 33) for s in range(256) if size[s] == length]
    return bits[1:17], symbols


def _codes(counts, symbols):
    code, k, out = 0, 0, {}
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            out[symbols[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def _nbits(v):
    return int(v).bit_length()


class _Scan:
    """Symbols and raw bits of one scan, recorded per restart interval; encoded once the scan's optimal table is known."""

    def __init__(self):
        self.intervals = []
        self.freq = {}

    def start(self):
        self.intervals.append([])

    def sym(self, table, s):
        self.intervals[-1].append(("s", table, s))
        self.freq.setdefault(table, {})
        self.freq[table][s] = self.freq[table].get(s, 0) + 1

    def bits(self, v, n):
        if n:
            self.intervals[-1].append(("b", v & ((1 << n) - 1), n))


def _blocks(comps, idx, mx, my, w, h, hmax, vmax):
    """Block coordinates of every unit of a scan (lists per unit), in coding order."""
    if len(idx) == 1:
        c = comps[idx[0]]
        ux, uy = -(-w * c["h"] // (8 * hmax)), -(-h * c["v"] // (8 * vmax))
        return [[(0, idx[0], y, x)] for y in range(uy) for x in range(ux)]
    return [[(i, c, y * comps[c]["v"] + by, x * comps[c]["h"] + bx) for i, c in enumerate(idx)
             for by in range(comps[c]["v"]) for bx in range(comps[c]["h"])] for y in range(my) for x in range(mx)]


def _encode_scan(coef, units, idx, ss, se, ah, al, restart):
    sc = _Scan()
    nat = J.NATURAL_ORDER
    per = restart or len(units)
    for u0 in range(0, len(units), per):
        sc.start()
        pred = [0] * len(idx)
        eobrun, be = 0, []

        def flush_eob():
            nonlocal eobrun, be
            if eobrun:
                n = _nbits(eobrun) - 1
                sc.sym(0, n << 4)
                sc.bits(eobrun, n)
                eobrun = 0
            for b in be:
                sc.bits(b, 1)
            be = []

        for unit in units[u0:u0 + per]:
            for i, c, y, x in unit:
                blk = [int(v) for v in coef[c][y, x]]
                if ss == 0:
                    if ah == 0:
                        v = blk[0] >> al
                        d = v - pred[i]
                        pred[i] = v
                        n = _nbits(abs(d))
                        sc.sym(i, n)
                        sc.bits(d if d >= 0 else d - 1, n)
                    else:
                        sc.bits((blk[0] >> al) & 1, 1)
                    continue
                if ah == 0:
                    r = 0
                    for k in range(ss, se + 1):
                        t = blk[nat[k]]
                        m = (-t if t < 0 else t) >> al
                        if m == 0:
                            r += 1
                            continue
                        flush_eob()
                        while r > 15:
                            sc.sym(0, 0xF0)
                            r -= 16
                        n = _nbits(m)
                        sc.sym(0, (r << 4) + n)
                        sc.bits(m if t >= 0 else ~m, n)
                        r = 0
                    if r:
                        eobrun += 1
                        if eobrun == 0x7FFF:
                            flush_eob()
                    continue
                absv = [abs(blk[nat[k]]) >> al for k in range(64)]
                eob = max([k for k in range(ss, se + 1) if absv[k] == 1], default=-1)
                r, br = 0, []
                for k in range(ss, se + 1):
                    t = absv[k]
                    if t == 0:
                        r += 1
                        continue
                    while r > 15 and k <= eob:
                        flush_eob()
                        sc.sym(0, 0xF0)
                        r -= 16
                        for b in br:
                            sc.bits(b, 1)
                        br = []
                    if t > 1:
                        br.append(t & 1)
                        continue
                    flush_eob()
                    sc.sym(0, (r << 4) + 1)
                    sc.bits(0 if blk[nat[k]] < 0 else 1, 1)
                    for b in br:
                        sc.bits(b, 1)
                    br, r = [], 0
                if r > 0 or br:
                    eobrun += 1
                    be += br
                    if eobrun == 0x7FFF or len(be) > 900:
                        flush_eob()
        flush_eob()
    return sc


def _segment(marker, payload: bytes) -> bytes:
    return bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + payload


def _entropy_bytes(items, codes) -> bytes:
    bits = []
    for kind, a, b in items:
        if kind == "s":
            code, n = codes[a][b]
            bits.append(format(code, f"0{n}b"))
        else:
            bits.append(format(a, f"0{b}b"))
    s = "".join(bits)
    s += "1" * (-len(s) % 8)
    raw = int(s, 2).to_bytes(len(s) // 8, "big") if s else b""
    return raw.replace(b"\xff", b"\xff\x00")


def reencode(baseline: bytes, script, restart: int = 0, dri_per_scan=None) -> bytes:
    """A progressive file with the quantised coefficients of `baseline` (oracle/jpeg.py's entropy_decode) and the scan
    script `script` ([(component indexes, Ss, Se, Ah, Al)]), each scan with its own optimal Huffman tables in a DHT right
    before its SOS (every table in slot 0, so each DHT redefines the previous one).  `restart` is the DRI of every scan, or
    `dri_per_scan` gives one per scan (a DRI segment before each)."""
    hdr = J.parse(baseline)
    coef = J.entropy_decode(baseline, hdr)
    comps, w, h = hdr["comps"], hdr["width"], hdr["height"]
    out = bytearray(b"\xff\xd8")
    out += _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    qid = [c["tq"] for c in comps]
    seen = {}
    for c, t in zip(comps, qid):
        if t not in seen:
            seen[t] = c["q"]
            zz = np.asarray(c["q"])[J.NATURAL_ORDER]
            out += _segment(0xDB, bytes([0x10 | t]) + b"".join(int(v).to_bytes(2, "big") for v in zz)
                            if zz.max() > 255 else bytes([t]) + bytes(int(v) for v in zz))
    sof = bytes([8, h >> 8, h & 255, w >> 8, w & 255, len(comps)])
    for i, (c, t) in enumerate(zip(comps, qid)):
        sof += bytes([i + 1, (c["h"] << 4) | c["v"], t])
    out += _segment(0xC2, sof)
    if dri_per_scan is None:
        out += _segment(0xDD, bytes([restart >> 8, restart & 255]))
    for j, (idx, ss, se, ah, al) in enumerate(script):
        ri = restart if dri_per_scan is None else dri_per_scan[j]
        if dri_per_scan is not None:
            out += _segment(0xDD, bytes([ri >> 8, ri & 255]))
        units = _blocks(comps, list(idx), hdr["mcus_x"], hdr["mcus_y"], w, h, hdr["hmax"], hdr["vmax"])
        sc = _encode_scan(coef, units, list(idx), ss, se, ah, al, ri)
        dc = ss == 0
        codes, dht = {}, b""
        for table, freq in sorted(sc.freq.items()):
            counts, symbols = _optimal_table(freq)
            codes[table] = _codes(counts, symbols)
            dht += bytes([(0 if dc else 0x10) | table]) + bytes(counts) + bytes(symbols)
        if dht:
            out += _segment(0xC4, dht)
        sos = bytes([len(idx)])
        for i, c in enumerate(idx):
            sos += bytes([c + 1, (i << 4) if dc else 0])
        out += _segment(0xDA, sos + bytes([ss, se, (ah << 4) | al]))
        for k, items in enumerate(sc.intervals):
            if k:
                out += bytes([0xFF, 0xD0 + ((k - 1) & 7)])
            out += _entropy_bytes(items, codes)
    out += b"\xff\xd9"
    return bytes(out)


def _pillow(a, sub, **kw) -> bytes:
    b = io.BytesIO()
    im = Image.fromarray(a[:, :, 0]) if sub == "gray" else Image.fromarray(a)
    if sub != "gray":
        kw["subsampling"] = sub
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def scripts(ncomp: int) -> dict:
    """Scan scripts no library encoder writes by default."""
    cs = list(range(ncomp))
    dc_all = [(tuple(cs), 0, 0, 0, 0)]
    out = {}
    out["spectral_only"] = dc_all + [((c,), 1, 5, 0, 0) for c in cs] + [((c,), 6, 63, 0, 0) for c in cs]
    out["approx_from_al3"] = ([(tuple(cs), 0, 0, 0, 3)] + [((c,), 1, 63, 0, 3) for c in cs]
                              + [(tuple(cs), 0, 0, a + 1, a) for a in (2, 1, 0)]
                              + [((c,), 1, 63, a + 1, a) for a in (2, 1, 0) for c in cs])
    out["dc_per_component"] = ([((c,), 0, 0, 0, 1) for c in cs] + [((c,), 1, 63, 0, 1) for c in cs]
                               + [((c,), 0, 0, 1, 0) for c in cs] + [((c,), 1, 63, 1, 0) for c in cs])
    out["scan_per_coefficient"] = dc_all + [((c,), k, k, 0, 0) for c in cs for k in range(1, 64)]
    return out


def reencoded(seed: int = 0):
    """(name, bytes): every script on baseline files of sizes off the MCU grid in each subsampling, with and without restart
    intervals (one DRI per scan in one case), EOB runs longer than 32767 blocks, and extreme coefficients."""
    rng = np.random.default_rng(seed)
    out = []
    for (w, h), sub in [((33, 47), 2), ((17, 9), 1), ((15, 17), 0), ((23, 18), "gray")]:
        base = _pillow(content("noise" if w < 30 else "grad", w, h, rng), sub, quality=85)
        ncomp = 1 if sub == "gray" else 3
        for name, script in scripts(ncomp).items():
            for rst in (0, 2):
                out.append((f"re-{w}x{h}-{sub}-{name}-rst{rst}", reencode(base, script, rst)))
        script = scripts(ncomp)["approx_from_al3"]
        out.append((f"re-{w}x{h}-{sub}-dri_per_scan", reencode(base, script, dri_per_scan=[(j % 3) for j in range(len(script))])))
    flat = _pillow(np.full((1400, 1600, 3), 90, np.uint8), "gray", quality=90)  # 35000 blocks: EOB runs past 32767
    out.append(("re-1600x1400-gray-long_eobrun", reencode(flat, scripts(1)["approx_from_al3"])))
    out.append(("re-1600x1400-gray-long_eobrun-rst", reencode(flat, scripts(1)["approx_from_al3"], 4000)))
    sat = content("sat", 40, 24, rng)
    ones = _pillow(sat, 0, qtables=[[1] * 64, [1] * 64])
    for name in ("approx_from_al3", "spectral_only"):
        out.append((f"re-40x24-444-sat-q1tables-{name}", reencode(ones, scripts(3)[name], 3)))
    return out


def corpus(seed: int = 0):
    """(name, bytes): every size x subsampling with content, quality and restart interval cycling through their lists; every
    quality x restart interval at 33 x 47 in 4:2:0 and gray; and the re-encoded files."""
    rng = np.random.default_rng(seed)
    out = []
    for i, ((w, h), sub) in enumerate(itertools.product(SIZES, SUBSAMPLINGS)):
        kind, q, rst = CONTENTS[i % len(CONTENTS)], QUALITIES[i % len(QUALITIES)], RESTARTS[i % len(RESTARTS)]
        out.append((f"{w}x{h}-{sub}-{kind}-q{q}-{rst}", encode_progressive(content(kind, w, h, rng), sub, q, rst)))
    for sub, q, rst in itertools.product([2, "gray"], QUALITIES, RESTARTS):
        out.append((f"33x47-{sub}-noise-q{q}-{rst}", encode_progressive(content("noise", 33, 47, rng), sub, q, rst)))
    return out + reencoded(seed)
