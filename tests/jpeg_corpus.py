"""Seeded JPEG corpus of the decoder tests (tests/test_jpeg_cpu.py, tests/test_jpeg_decode_gpu.py): encoded by Pillow and
cv2 (libjpeg-turbo) across sizes around the MCU edges, every subsampling the device decodes, qualities, custom tables,
optimised Huffman tables, restart intervals and contents that reach the range limits."""
from __future__ import annotations

import io
import itertools

import numpy as np
from PIL import Image

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 16), (33, 47), (15, 15), (17, 17), (15, 7), (17, 9), (7, 15),
         (9, 17), (500, 375)]
SUBSAMPLINGS = [0, 1, 2, "440", "gray"]
QUALITIES = [1, 50, 75, 90, 95, 100, "qtables", "optimize"]
RESTARTS = [None, "blocks", "rows", "cv2"]
CONTENTS = ["flat", "grad", "noise", "sat"]


def content(kind: str, w: int, h: int, rng) -> np.ndarray:
    if kind == "flat":
        return np.full((h, w, 3), (200, 30, 90), np.uint8)
    if kind == "grad":
        x = np.linspace(0, 255, w)[None, :, None]
        y = np.linspace(0, 255, h)[:, None, None]
        return np.broadcast_to(np.concatenate([x + 0 * y, y + 0 * x, (x + y) / 2], 2), (h, w, 3)).astype(np.uint8)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)  # saturated extremes


def encode(a: np.ndarray, sub, quality, restart) -> bytes:
    """JPEG bytes of RGB `a`; cv2 for 4:4:0 and its restart interval, Pillow otherwise."""
    q = 90 if isinstance(quality, str) else quality
    if sub == "440" or restart == "cv2":
        import cv2
        params = [cv2.IMWRITE_JPEG_QUALITY, q]
        if quality == "optimize":
            params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
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
    kw = dict(quality=q)
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
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def corpus(seed: int = 0):
    """(name, bytes): every size x subsampling x content, quality and restart interval cycling through their lists; plus
    every quality x restart interval at 33 x 47 in 4:2:0 and gray."""
    rng = np.random.default_rng(seed)
    out = []
    for i, ((w, h), sub, kind) in enumerate(itertools.product(SIZES, SUBSAMPLINGS, CONTENTS)):
        q, rst = QUALITIES[i % len(QUALITIES)], RESTARTS[i % len(RESTARTS)]
        out.append((f"{w}x{h}-{sub}-{kind}-q{q}-{rst}", encode(content(kind, w, h, rng), sub, q, rst)))
    for sub, q, rst in itertools.product([2, "gray"], QUALITIES, RESTARTS):
        out.append((f"33x47-{sub}-noise-q{q}-{rst}", encode(content("noise", 33, 47, rng), sub, q, rst)))
    return out


def photo(w: int, h: int, seed: int = 0) -> np.ndarray:
    """A smooth photo-like image with texture: low-frequency colour fields plus noise."""
    rng = np.random.default_rng(seed)
    small = rng.integers(0, 256, (max(2, h // 64), max(2, w // 64), 3), dtype=np.uint8)
    base = np.asarray(Image.fromarray(small).resize((w, h), Image.BICUBIC), np.int16)
    return np.clip(base + rng.integers(-12, 13, (h, w, 3)), 0, 255).astype(np.uint8)


def corrupt(data: bytes, how: str) -> bytes:
    """`data` damaged in one way: the first single-byte change of the scan (positions and values in a fixed order) after
    which the oracle refuses the stream for the wanted reason ("flip": an invalid Huffman code, "ac_overrun": an AC run past
    coefficient 63), or "drop_rst": the second RST marker removed, or "early_eoi": EOI a third of the way into the scan."""
    from oracle import jpeg as J
    b = bytearray(data)
    sos = b.index(b"\xff\xda")
    start = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    if how == "drop_rst":
        i = b.index(b"\xff\xd1", start)
        return bytes(b[:i] + b[i + 2:])
    if how == "early_eoi":
        cut = start + (len(b) - start) // 3
        while b[cut - 1] == 0xFF:
            cut -= 1
        return bytes(b[:cut]) + b"\xff\xd9"
    want = {"flip": "bad Huffman code", "ac_overrun": "AC run past coefficient 63"}[how]
    for pos in range(start, len(b) - 2):
        if b[pos] == 0xFF or b[pos - 1] == 0xFF:
            continue
        for v in (0xFE, 0x00, 0x7F, 0xF0, 0x0F, 0xAA, 0x55):
            c = bytearray(b)
            c[pos] = v
            try:
                J.decode(bytes(c))
            except J.Unsupported as e:
                if str(e) == want:
                    return bytes(c)
    raise ValueError(f"no single-byte change gives {want}")


def all_ones_code(data: bytes) -> bytes:
    """`data` with one more DC symbol of length 9 in its first DHT table, which makes 111111111 a code: a table libjpeg
    refuses (JERR_BAD_HUFF_TABLE).  The scan bytes are unchanged."""
    b = bytearray(data)
    i = b.index(b"\xff\xc4")
    assert b[i + 4] >> 4 == 0, "first DHT table is not a DC table"
    counts = b[i + 5:i + 21]
    at = i + 21 + sum(counts[:9])  # after the symbols of lengths 1..9
    counts[8] += 1
    b[i + 5:i + 21] = counts
    b[at:at] = b"\x00"
    ln = (b[i + 2] << 8 | b[i + 3]) + 1
    b[i + 2:i + 4] = bytes([ln >> 8, ln & 255])
    return bytes(b)


def with_size(data: bytes, w: int, h: int) -> bytes:
    """`data` with the frame header's size replaced."""
    b = bytearray(data)
    i = b.index(b"\xff\xc0")
    b[i + 5:i + 9] = bytes([h >> 8, h & 255, w >> 8, w & 255])
    return bytes(b)


def with_segment(data: bytes, marker: int, payload: bytes) -> bytes:
    """`data` with one more marker segment right after SOI."""
    return data[:2] + bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + payload + data[2:]
