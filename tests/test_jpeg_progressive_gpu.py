"""GPU tests of the progressive JPEG decoder (csrc/jpeg.cu via visiondk_b200.jpeg): bit for bit against Pillow on the seeded
progressive corpus and on photo-sized files with and without restart intervals, mixed batches of baseline, progressive, PNG
and corrupt progressive files equal to decoding each file alone and to read_image (in one launch and under a tiny workspace
budget), corrupted progressive streams flagged by the device and given read_image's result, determinism, and the three
image-folder consumers on folders with progressive files equal to their host-decoded path."""
import io
import os

import numpy as np
import pytest
import torch
import yaml
from PIL import Image, features

from engine.cbir.folder import read_image
from jpeg_corpus import encode, photo
from jpeg_progressive_corpus import corpus, encode_progressive
from oracle import jpeg_progressive as JP
from visiondk_b200 import _lib
from visiondk_b200.jpeg import JpegDecoder

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def write(tmp_path, items):
    paths = []
    for i, (name, data) in enumerate(items):
        p = tmp_path / f"{i:04d}-{name}.jpg"
        p.write_bytes(data)
        paths.append(str(p))
    return paths


def pil(path):
    return np.asarray(Image.open(path).convert("RGB"))


def host_result(path):
    try:
        return read_image(path)
    except Exception as e:  # noqa: BLE001 - the device path must raise the same type
        return type(e)


def test_corpus_bit_exact(tmp_path):
    print("Pillow", Image.__version__ if hasattr(Image, "__version__") else "", "libjpeg-turbo", features.version("libjpeg_turbo"))
    items = corpus()
    paths = write(tmp_path, items)
    batch = JpegDecoder("cuda", read_image)(paths)
    assert batch.reasons == [_lib.JPEG_DEVICE_PROGRESSIVE] * len(paths)
    assert batch.status == [0] * len(paths), [n for (n, _), s in zip(items, batch.status) if s]
    for (name, _), p, got in zip(items, paths, batch.numpy()):
        assert np.array_equal(pil(p), got), name


@pytest.mark.parametrize("w,h", [(2000, 1500), (4032, 3024)])
@pytest.mark.parametrize("restart", [None, "rows", "blocks"])
def test_photos_bit_exact(tmp_path, w, h, restart):
    paths = write(tmp_path, [(f"{sub}", encode_progressive(photo(w, h, seed=w + (sub if isinstance(sub, int) else 7)), sub, 90,
                                                           restart)) for sub in (2, 1, 0)])
    batch = JpegDecoder("cuda", read_image)(paths)
    assert batch.reasons == [_lib.JPEG_DEVICE_PROGRESSIVE] * 3 and batch.status == [0, 0, 0]
    for p, got in zip(paths, batch.numpy()):
        assert np.array_equal(pil(p), got), p


def scan_starts(data: bytes):
    """(start of the entropy-coded data, its end) of every scan, from the oracle's parse."""
    return [(s["segments"][0][0], s["end"]) for s in JP.parse(data)["scans"]]


def flipped(data: bytes, scan: int) -> bytes:
    """`data` with one byte of scan `scan` changed: the first change (positions and values in a fixed order) that the oracle
    refuses as a malformed stream, or the first change at all when every bit string is a valid scan (a DC refinement)."""
    a, b = scan_starts(data)[scan]
    first = None
    for pos in range(a, b - 1):
        if data[pos] == 0xFF or data[pos - 1] == 0xFF:
            continue
        for v in (0xFE, 0x00, 0x7F, 0xF0, 0x0F, 0xAA, 0x55):
            if v == data[pos]:
                continue
            c = bytearray(data)
            c[pos] = v
            first = first or bytes(c)
            try:
                JP.decode(bytes(c))
            except JP.Unsupported as e:
                if e.reason == JP.MALFORMED:
                    return bytes(c)
        if pos > a + 64:
            break
    return first


def corrupted():
    good = encode_progressive(photo(96, 80), 2, 90, None)
    hdr = JP.parse(good)
    kinds = {}
    for j, s in enumerate(hdr["scans"]):  # the first scan of each kind: DC first, AC first, DC refine, AC refine
        kinds.setdefault((s["ss"] == 0, s["ah"] != 0), j)
    items = [(f"flip_scan{j}", flipped(good, j)) for j in sorted(kinds.values())]
    a, b = scan_starts(good)[3]
    items.append(("truncated_mid_scan", good[:(a + b) // 2]))
    items.append(("eoi_mid_scan", good[:(a + b) // 2] + b"\xff\xd9"))
    items.append(("missing_last_scan", good[:good.rindex(b"\xff\xc4")] + b"\xff\xd9"))
    return items


def test_corrupted_streams(tmp_path):
    items = corrupted()
    assert len(items) == 7
    paths = write(tmp_path, items)
    dec = JpegDecoder("cuda", read_image)
    for (name, _), p in zip(items, paths):
        expect = host_result(p)
        if isinstance(expect, type):
            with pytest.raises(expect):
                dec([p])
            continue
        batch = dec([p])
        if name.startswith("flip"):  # the parser hands these over; the device flags what the oracle refuses
            try:
                JP.decode(open(p, "rb").read())
                refused = False
            except JP.Unsupported:
                refused = True
            assert batch.reasons[0] == _lib.JPEG_DEVICE_PROGRESSIVE, name
            assert (batch.status[0] & ~_lib.JPEG_BAD_SKIPPED) if refused else batch.status[0] == 0, name
        else:
            assert batch.status[0] != 0, name
        assert np.array_equal(batch.numpy()[0], expect), name


def mixed(tmp_path):
    items = [(n, d) for n, d in corpus()[::9]]
    items += [("baseline", encode(photo(64, 48), 2, 90, None)), ("baseline_rst", encode(photo(120, 90), 0, 85, "rows"))]
    b = io.BytesIO()
    Image.fromarray(photo(40, 30)).save(b, "PNG")
    items.append(("png", b.getvalue()))
    items.append(("photo", encode_progressive(photo(640, 480), 2, 85, "rows")))
    items += [c for c in corrupted() if c[0].startswith("flip")][:2]
    return write(tmp_path, items)


def test_mixed_batches_equal_single_decodes_and_read_image(tmp_path):
    paths = mixed(tmp_path)
    dec = JpegDecoder("cuda", read_image)
    whole = dec(paths)
    assert {_lib.JPEG_DEVICE, _lib.JPEG_DEVICE_PROGRESSIVE, _lib.JPEG_NOT_JPEG} <= set(whole.reasons)
    split = JpegDecoder("cuda", read_image, workspace_budget=1 << 16)(paths).numpy()  # many launches into one output
    for p, a, b in zip(paths, whole.numpy(), split):
        alone = dec([p]).numpy()[0]
        assert np.array_equal(a, alone) and np.array_equal(b, alone) and np.array_equal(alone, read_image(p)), p


def test_deterministic(tmp_path):
    paths = mixed(tmp_path)
    a = JpegDecoder("cuda", read_image)(paths)
    b = JpegDecoder("cuda", read_image)(paths)
    assert torch.equal(a.data, b.data) or all(np.array_equal(x, y) for x, y in zip(a.numpy(), b.numpy()))


def test_pixel_limit_applies_to_progressive_files(tmp_path, monkeypatch):
    paths = write(tmp_path, [("small", encode_progressive(photo(40, 30), 2, 90, None)),
                             ("mid", encode_progressive(photo(64, 48), 2, 90, None))])
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 2000)
    with pytest.warns(Image.DecompressionBombWarning):
        batch = JpegDecoder("cuda", read_image)(paths)
    assert batch.reasons == [_lib.JPEG_DEVICE_PROGRESSIVE, _lib.JPEG_TOO_LARGE] and batch.status[0] == 0
    for p, got in zip(paths, batch.numpy()):
        assert np.array_equal(got, pil(p))


def folder(tmp_path, splits, ids=3, per=5):
    rng = np.random.default_rng(7)
    for split in splits:
        for i in range(ids):
            d = tmp_path / split / f"id{i}"
            os.makedirs(d)
            for j in range(per):
                w, h = int(rng.integers(60, 300)), int(rng.integers(60, 300))
                sub = [0, 1, 2, "gray"][(i + j) % 4]
                enc = encode_progressive if j % 2 == 0 else encode
                (d / f"{j}.jpg").write_bytes(enc(photo(w, h, seed=100 * i + j), sub, 90, [None, "rows"][(j // 2) % 2]))
            Image.fromarray(photo(50, 40, seed=i)).save(d / "extra.png")


def test_cbir_folder_batches_equal_host_path(tmp_path):
    from engine.cbir.folder import CBIRFolderData
    from visiondk_b200.preprocess import ImagePreprocessor
    folder(tmp_path, ("query", "gallery"))
    aug = [{"resize_and_padding": {"size": 96, "training": False}}, {"to_tensor": "no_params"}, {"normalize": "no_params"}]
    data = CBIRFolderData(str(tmp_path), aug, batch=4, device="cuda", nw=2)
    pre = ImagePreprocessor(96, data.mean, data.std, "cuda")
    for dev, files in ((data.gallery_batches(), data.gallery_files), (data.query_batches(), data.query_files)):
        host = [pre(images) for images in data.decoded_batches(files)]
        dev = list(dev)
        assert len(dev) == len(host)
        for x, y in zip(dev, host):
            assert torch.equal(x, y)


def test_folder_train_batches_equal_host_path(tmp_path):
    from engine.cbir.folder import decode_batches
    from engine.folder_train import FolderTrainData
    import engine.folder_train as FT
    folder(tmp_path, ("train",), ids=3, per=6)
    with open(os.path.join(GOLDEN, "reference_configs", "cbir.yaml")) as f:
        cfg = yaml.safe_load(f)["data"]
    cfg = dict(cfg, nw=2)
    cfg["train"] = dict(cfg["train"], bs=4, aug_epoch=2)
    data = FolderTrainData(str(tmp_path), cfg, 3, "cuda", warm_ep=1, seed=3)
    for epoch in (0, 1):
        dev = list(data.train_batches(epoch))
        orig = FT.device_decode_batches
        FT.device_decode_batches = lambda files, batch, device, nw: decode_batches(files, batch, nw)
        try:
            host = list(data.train_batches(epoch))
        finally:
            FT.device_decode_batches = orig
        assert len(dev) == len(host) > 0
        for (x, y), (hx, hy) in zip(dev, host):
            assert torch.equal(x, hx) and torch.equal(y, hy)


def test_face_image_batches_equal_host_path(tmp_path):
    from engine.cbir.folder import decode_batches
    from engine.faceX.evaluation import image_batches
    from visiondk_b200.preprocess import ImagePreprocessor
    folder(tmp_path, ("val",), ids=2, per=5)
    paths = sorted(str(p) for p in (tmp_path / "val").rglob("*.*"))
    aug = [{"resize_and_padding": {"size": 112, "training": False}}, {"to_tensor": "no_params"}, {"normalize": "no_params"}]
    pre = ImagePreprocessor(112, device="cuda")
    host = [pre(images) for images in decode_batches(paths, 3, 2)]
    dev = list(image_batches(paths, aug, 3, "cuda", nw=2))
    assert len(dev) == len(host)
    for (_, x, names), y in zip(dev, host):
        assert torch.equal(x, y)
