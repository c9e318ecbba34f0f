"""CPU checks of the baseline JPEG decoder: the numpy oracle (oracle/jpeg.py) against the installed Pillow, bit for bit, on the
seeded corpus of tests/jpeg_corpus.py, and the host parser of csrc/jpeg.cu (vdk_jpeg_parse: which files the device takes,
and the fallback reason of each one it does not)."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import Image, features

from jpeg_corpus import all_ones_code, corpus, corrupt, encode, photo, with_segment, with_size
from oracle import jpeg as J
from visiondk_b200 import _lib


def test_struct_mirrors(lib):
    sizes = (C.c_size_t * 2)()
    assert lib.vdk_jpeg_struct_sizes(sizes, 2) == 2
    assert list(sizes) == [C.sizeof(_lib.JpegHuff), C.sizeof(_lib.JpegDesc)]


def test_oracle_is_pillow_bit_for_bit():
    print("Pillow", Image.__version__ if hasattr(Image, "__version__") else "", "libjpeg-turbo", features.version("libjpeg_turbo"))
    items = corpus()
    assert len(items) > 300
    for name, data in items:
        ref = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        got = J.decode(data)
        assert np.array_equal(ref, got), name


def parse(lib, blobs):
    offs, off = [], 0
    for b in blobs:
        offs.append(off)
        off += len(b) + 16
    buf = np.zeros(off, np.uint8)
    descs = (_lib.JpegDesc * len(blobs))()
    for i, b in enumerate(blobs):
        buf[offs[i]:offs[i] + len(b)] = np.frombuffer(b, np.uint8)
        descs[i].data_offset, descs[i].data_bytes = offs[i], len(b)
    segs = np.full(1 << 16, -1, np.int64)
    assert lib.vdk_jpeg_parse(buf.ctypes.data, descs, len(blobs), segs.ctypes.data, len(segs)) == 0
    parse.segs = segs
    return descs


def test_parser_takes_the_corpus_and_agrees_with_the_oracle_header(lib):
    items = corpus()
    descs = parse(lib, [d for _, d in items])
    for (name, data), d in zip(items, descs):
        hdr = J.parse(data)
        assert d.reason == _lib.JPEG_DEVICE, name
        assert (d.width, d.height, d.ncomp) == (hdr["width"], hdr["height"], len(hdr["comps"])), name
        assert (d.mcus_x, d.mcus_y, d.restart_interval, d.n_segments) == (hdr["mcus_x"], hdr["mcus_y"], hdr["restart"],
                                                                            len(hdr["segments"])), name
        assert (d.scan_begin, d.scan_end) == (hdr["segments"][0][0], hdr["segments"][-1][1]), name
        starts = parse.segs[d.seg_first:d.seg_first + d.n_segments].tolist()
        assert starts == [a for a, _ in hdr["segments"]], name
        for c, comp in enumerate(hdr["comps"]):
            assert (d.h[c], d.v[c]) == (comp["h"], comp["v"])
            assert list(d.quant[c]) == [int(np.int16(np.uint16(q))) for q in comp["q"]]


def test_parser_fallback_reasons(lib):
    import cv2
    a = photo(64, 48)
    cases = {}
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", progressive=True)
    cases["progressive"] = (b.getvalue(), _lib.JPEG_PROCESS)
    b = io.BytesIO()
    Image.fromarray(a).convert("CMYK").save(b, "JPEG")
    cases["cmyk"] = (b.getvalue(), _lib.JPEG_COLOR)
    ok, buf = cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])
    cases["411"] = (buf.tobytes(), _lib.JPEG_SAMPLING)
    b = io.BytesIO()
    Image.fromarray(a).save(b, "PNG")
    cases["png"] = (b.getvalue(), _lib.JPEG_NOT_JPEG)
    good = encode(a, 2, 90, None)
    cases["jpeg_named_png"] = (good, _lib.JPEG_DEVICE)  # content decides, not the name
    cases["truncated_header"] = (good[:200], _lib.JPEG_MALFORMED)
    cases["truncated_scan"] = (good[:len(good) // 2], _lib.JPEG_MALFORMED)
    rst = encode(a, 2, 90, "blocks")
    cases["dropped_rst"] = (corrupt(rst, "drop_rst"), _lib.JPEG_RESTART)
    cases["early_eoi_with_dri"] = (corrupt(rst, "early_eoi"), _lib.JPEG_RESTART)
    # scan-byte damage is the device's to find: the parser still hands these over
    cases["flipped_scan_byte"] = (corrupt(good, "flip"), _lib.JPEG_DEVICE)
    cases["early_eoi"] = (corrupt(good, "early_eoi"), _lib.JPEG_DEVICE)
    rgb = bytearray(encode(a, 0, 90, None))  # Adobe transform 0 (RGB): rewrite the JFIF APP0 into an APP14 "Adobe" segment
    app0 = rgb.index(b"\xff\xe0")
    ln = (rgb[app0 + 2] << 8) | rgb[app0 + 3]
    rgb[app0:app0 + 2 + ln] = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"
    cases["adobe_rgb"] = (bytes(rgb), _lib.JPEG_COLOR)
    cases["huffman_all_ones_code"] = (all_ones_code(good), _lib.JPEG_MALFORMED)
    cases["width_65501"] = (with_size(good, 65501, 48), _lib.JPEG_TOO_LARGE)
    cases["short_jfif_app0"] = (with_segment(good, 0xE0, b"JFIF\0"), _lib.JPEG_MALFORMED)
    cases["short_adobe_app14"] = (with_segment(good, 0xEE, b"Adobe"), _lib.JPEG_MALFORMED)
    cases["short_icc_app2"] = (with_segment(good, 0xE2, b"ICC_PROFILE\0\x01"), _lib.JPEG_MALFORMED)
    cases["photoshop_cut_after_code"] = (with_segment(good, 0xED, b"Photoshop 3.0\x008BIM\x03\xed"), _lib.JPEG_MALFORMED)
    cases["photoshop_short_size"] = (with_segment(good, 0xED, b"Photoshop 3.0\x008BIM\x04\x04\x00\x00\x00"), _lib.JPEG_DEVICE)
    names = list(cases)
    descs = parse(lib, [cases[k][0] for k in names])
    for k, d in zip(names, descs):
        assert d.reason == cases[k][1], (k, d.reason)
        if cases[k][1] != _lib.JPEG_DEVICE and cases[k][1] != _lib.JPEG_NOT_JPEG:
            with pytest.raises(J.Unsupported) as e:
                J.decode(cases[k][0])
            assert e.value.reason == cases[k][1], k


def test_corrupted_scans_are_refused_by_the_oracle():
    good = encode(photo(96, 80), 2, 90, None)
    for how in ("flip", "ac_overrun", "early_eoi"):
        with pytest.raises(J.Unsupported):
            J.decode(corrupt(good, how))


def test_what_the_parser_refuses_pillow_refuses():
    """The header cases above on which the device path must not decode: Image.open(...).convert("RGB") raises on each."""
    good = encode(photo(64, 48), 2, 90, None)
    for data in (all_ones_code(good), with_segment(good, 0xE0, b"JFIF\0"), with_segment(good, 0xEE, b"Adobe"),
                 with_segment(good, 0xE2, b"ICC_PROFILE\0\x01"), with_segment(good, 0xED, b"Photoshop 3.0\x008BIM\x03\xed")):
        with pytest.raises(Exception):
            Image.open(io.BytesIO(data)).convert("RGB")
    ok = with_segment(good, 0xED, b"Photoshop 3.0\x008BIM\x04\x04\x00\x00\x00")
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(ok)).convert("RGB")), J.decode(ok))
