"""CPU checks of the progressive JPEG decoder: the numpy oracle (oracle/jpeg_progressive.py) against the installed Pillow, bit
for bit, on the seeded corpus of tests/jpeg_progressive_corpus.py, and the second host parser of csrc/jpeg.cu
(vdk_jpeg_parse_progressive: headers, scan tables, dependency levels, restart-interval starts and fallback reasons)."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import Image, features

from jpeg_corpus import corpus as baseline_corpus
from jpeg_corpus import photo
from jpeg_progressive_corpus import corpus, encode_progressive, reencode, scripts
from oracle import jpeg as J
from oracle import jpeg_progressive as JP
from visiondk_b200 import _lib


@pytest.fixture(scope="module")
def items():
    return corpus()


def parse(lib, blobs, scan_capacity=1 << 12):
    offs, off = [], 0
    for b in blobs:
        offs.append(off)
        off += len(b) + 16
    buf = np.zeros(off, np.uint8)
    descs = (_lib.JpegDesc * len(blobs))()
    for i, b in enumerate(blobs):
        buf[offs[i]:offs[i] + len(b)] = np.frombuffer(b, np.uint8)
        descs[i].data_offset, descs[i].data_bytes = offs[i], len(b)
    segs = np.full(1 << 20, -1, np.int64)
    scans = (_lib.JpegScan * scan_capacity)()
    assert lib.vdk_jpeg_parse(buf.ctypes.data, descs, len(blobs), segs.ctypes.data, len(segs)) == 0
    assert lib.vdk_jpeg_parse_progressive(buf.ctypes.data, descs, len(blobs), scans, scan_capacity, segs.ctypes.data,
                                          len(segs)) == 0
    return descs, scans, segs


def test_struct_mirror(lib):
    size = (C.c_size_t * 1)()
    assert lib.vdk_jpeg_progressive_struct_sizes(size, 1) == 1
    assert size[0] == C.sizeof(_lib.JpegScan)


def test_oracle_is_pillow_bit_for_bit(items):
    print("Pillow", Image.__version__ if hasattr(Image, "__version__") else "", "libjpeg-turbo", features.version("libjpeg_turbo"))
    assert len(items) > 150
    for name, data in items:
        with pytest.raises(J.Unsupported) as e:  # the baseline oracle still refuses every one of them
            J.parse(data)
        assert e.value.reason == J.PROCESS, name
        ref = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        assert np.array_equal(ref, JP.decode(data)), name


def test_parser_agrees_with_the_oracle(lib, items):
    descs, scans, segs = parse(lib, [d for _, d in items])
    for (name, data), d in zip(items, descs):
        hdr = JP.parse(data)
        assert d.reason == _lib.JPEG_DEVICE_PROGRESSIVE, (name, d.reason)
        assert (d.width, d.height, d.ncomp, d.mcus_x, d.mcus_y) == (hdr["width"], hdr["height"], len(hdr["comps"]),
                                                                     hdr["mcus_x"], hdr["mcus_y"]), name
        assert (d.n_scans, d.n_levels) == (len(hdr["scans"]), hdr["levels"]), name
        for c, comp in enumerate(hdr["comps"]):
            assert (d.h[c], d.v[c]) == (comp["h"], comp["v"]), name
            assert list(d.quant[c]) == [int(np.int16(np.uint16(q))) for q in comp["q"]], name
        first = d.seg_first
        for j, sh in enumerate(hdr["scans"]):
            s = scans[d.scan_first + j]
            assert (s.ncomp, list(s.comp)[:s.ncomp], s.ss, s.se, s.ah, s.al) == (len(sh["comps"]), sh["comps"], sh["ss"],
                                                                                   sh["se"], sh["ah"], sh["al"]), name
            assert (s.level, s.units_x, s.units_y, s.restart_interval) == (sh["level"], sh["units_x"], sh["units_y"],
                                                                           sh["restart"]), name
            assert s.seg_first == first and s.n_segments == len(sh["segments"]), name
            assert segs[first:first + s.n_segments].tolist() == [a for a, _ in sh["segments"]], name
            assert (s.scan_begin, s.scan_end) == (sh["segments"][0][0], sh["segments"][-1][1]), name
            first += s.n_segments
        assert first == d.seg_first + d.n_segments, name


def test_default_script_levels(lib):
    """Pillow's and cv2's default script (libjpeg's jpeg_simple_progression): levels of 5, 4 and 1 scans."""
    import cv2
    a = photo(64, 48)
    ok, buf = cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    for data in (encode_progressive(a, 2, 90, None), buf.tobytes()):
        descs, scans, _ = parse(lib, [data])
        levels = [scans[descs[0].scan_first + j].level for j in range(descs[0].n_scans)]
        assert [levels.count(k) for k in range(3)] == [5, 4, 1] and descs[0].n_levels == 3


def test_parser_leaves_other_descriptors_alone(lib):
    """Only VDK_JPEG_PROCESS descriptors are re-read: baseline files, PNGs and refused baseline headers keep every byte."""
    blobs = [d for _, d in baseline_corpus()[::40]]
    b = io.BytesIO()
    Image.fromarray(photo(40, 30)).save(b, "PNG")
    blobs += [b.getvalue(), blobs[0][:100], encode_progressive(photo(40, 30), 2, 90, None)]
    offs, off = [], 0
    for x in blobs:
        offs.append(off)
        off += len(x) + 16
    buf = np.zeros(off, np.uint8)
    descs = (_lib.JpegDesc * len(blobs))()
    for i, x in enumerate(blobs):
        buf[offs[i]:offs[i] + len(x)] = np.frombuffer(x, np.uint8)
        descs[i].data_offset, descs[i].data_bytes = offs[i], len(x)
    segs = np.full(1 << 16, -1, np.int64)
    assert lib.vdk_jpeg_parse(buf.ctypes.data, descs, len(blobs), segs.ctypes.data, len(segs)) == 0
    before = [bytes(d) for d in descs]
    segs_before = segs.copy()
    scans = (_lib.JpegScan * 64)()
    assert lib.vdk_jpeg_parse_progressive(buf.ctypes.data, descs, len(blobs), scans, 64, segs.ctypes.data, len(segs)) == 0
    for i, d in enumerate(descs[:-1]):
        assert bytes(d) == before[i], i
    last = descs[len(blobs) - 1]
    assert last.reason == _lib.JPEG_DEVICE_PROGRESSIVE
    used = max(d.seg_first + d.n_segments for d in descs[:-1] if d.reason == _lib.JPEG_DEVICE)
    assert last.seg_first == used  # its restart-interval starts follow the baseline files' ones
    assert np.array_equal(segs[:used], segs_before[:used])


def _patched_sof(data: bytes, marker: int) -> bytes:
    b = bytearray(data)
    b[b.index(b"\xff\xc2") + 1] = marker
    return bytes(b)


def _scan_headers(data: bytes):
    """Positions of the Ss byte of every SOS header."""
    out, p = [], 0
    while True:
        p = data.find(b"\xff\xda", p)
        if p < 0:
            return out
        ns = data[p + 4]
        out.append(p + 5 + 2 * ns)
        p += 2


def refused_cases():
    a = photo(64, 48)
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", quality=90, subsampling=2)
    baseline = b.getvalue()
    good = encode_progressive(a, 2, 90, None)
    full = scripts(3)["spectral_only"]
    cases = {}
    cases["incomplete_script"] = (reencode(baseline, full[:-1]), _lib.JPEG_SCAN)  # Cr 6..63 never sent
    cases["unrefined_script"] = (reencode(baseline, [((0, 1, 2), 0, 0, 0, 1)] + full[1:]), _lib.JPEG_SCAN)  # DC stays at Al 1
    cases["missing_last_scan"] = (good[:good.rindex(b"\xff\xc4")] + b"\xff\xd9", _lib.JPEG_SCAN)
    dc_bogus = [((0, 1, 2), 0, 0, 0, 1), ((0, 1, 2), 0, 0, 2, 1), ((0, 1, 2), 0, 0, 1, 0)]  # Ah 2 where Al was 1
    cases["bogus_progression"] = (reencode(baseline, dc_bogus + full[1:]), _lib.JPEG_SCAN)
    cases["first_scan_sent_twice"] = (reencode(baseline, full + [((0,), 1, 5, 0, 0)]), _lib.JPEG_DEVICE_PROGRESSIVE)
    cases["ac_before_dc"] = (reencode(baseline, [((0,), 1, 63, 0, 0)] + [((0, 1, 2), 0, 0, 0, 0)] + full[2:] + [((0,), 1, 63, 0, 0)]),
                             _lib.JPEG_SCAN)
    cases["refine_without_first"] = (reencode(baseline, full + [((1,), 1, 63, 1, 0)]), _lib.JPEG_SCAN)
    cases["arithmetic_sof10"] = (_patched_sof(good, 0xCA), _lib.JPEG_PROCESS)
    cases["sof6"] = (_patched_sof(good, 0xC6), _lib.JPEG_PROCESS)
    bad = bytearray(good)
    at = _scan_headers(good)[1]  # an AC scan: Se above 63
    bad[at + 1] = 64
    cases["se_above_63"] = (bytes(bad), _lib.JPEG_MALFORMED)
    bad = bytearray(good)
    at = _scan_headers(good)[0]  # the DC scan: Al 14
    bad[at + 2] = 0x0E
    cases["al_14"] = (bytes(bad), _lib.JPEG_MALFORMED)
    bad = bytearray(good)
    at = _scan_headers(good)[-1]  # a refinement scan whose Al is not Ah - 1
    bad[at + 2] = (bad[at + 2] & 0xF0) | ((bad[at + 2] >> 4) + 1)
    cases["refine_al_not_ah_minus_1"] = (bytes(bad), _lib.JPEG_MALFORMED)
    return cases


def test_fallback_reasons_match_the_oracle_and_the_host_gives_pillow(lib):
    cases = refused_cases()
    names = list(cases)
    descs, _, _ = parse(lib, [cases[k][0] for k in names])
    for k, d in zip(names, descs):
        data, want = cases[k]
        assert d.reason == want, (k, d.reason)
        if want == _lib.JPEG_DEVICE_PROGRESSIVE:  # Ah 0 over coefficients already at Al 0: libjpeg accepts it silently
            assert np.array_equal(JP.decode(data), np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))), k
            continue
        with pytest.raises(J.Unsupported) as e:
            JP.decode(data)
        assert e.value.reason == want, k
        try:  # what the host decodes or raises is Pillow's own; make sure the files are what their names say
            Image.open(io.BytesIO(data)).convert("RGB")
            assert want in (_lib.JPEG_SCAN,), k  # incomplete and warned-about scripts still decode on the host
        except Exception:  # noqa: BLE001 - Pillow refuses the bad parameters and the arithmetic frames
            assert want in (_lib.JPEG_MALFORMED, _lib.JPEG_PROCESS), k
