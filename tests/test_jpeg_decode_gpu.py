"""GPU tests of the baseline JPEG decoder (csrc/jpeg.cu via visiondk_b200.jpeg): bit for bit against Pillow on the seeded
corpus and on photo-sized files with and without restart intervals, mixed batches (sizes, subsamplings, host-path files,
a workspace split) equal to decoding each file alone, corrupted streams flagged by the device and given read_image's
result, determinism, and the three image-folder consumers equal to their host-decoded path."""
import io
import os

import numpy as np
import pytest
import torch
import yaml
from PIL import Image, features

from engine.cbir.folder import read_image
from jpeg_corpus import all_ones_code, corpus, corrupt, encode, photo
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


def test_corpus_bit_exact(tmp_path):
    print("Pillow", Image.__version__ if hasattr(Image, "__version__") else "", "libjpeg-turbo", features.version("libjpeg_turbo"))
    items = corpus()
    paths = write(tmp_path, items)
    dec = JpegDecoder("cuda", read_image)
    batch = dec(paths)
    assert batch.status == [0] * len(paths), [n for (n, _), s in zip(items, batch.status) if s]
    for (name, _), p, got in zip(items, paths, batch.numpy()):
        assert np.array_equal(pil(p), got), name


@pytest.mark.parametrize("w,h", [(2000, 1500), (4032, 3024)])
@pytest.mark.parametrize("restart", [None, "rows", "blocks"])
def test_photos_bit_exact(tmp_path, w, h, restart):
    paths = write(tmp_path, [(f"{sub}", encode(photo(w, h, seed=w + (sub if isinstance(sub, int) else 7)), sub, 90, restart))
                             for sub in (2, 1, 0)])
    batch = JpegDecoder("cuda", read_image)(paths)
    assert batch.status == [0, 0, 0]
    for p, got in zip(paths, batch.numpy()):
        assert np.array_equal(pil(p), got), p


def mixed(tmp_path):
    items = corpus()[::7]
    b = io.BytesIO()
    Image.fromarray(photo(40, 30)).save(b, "PNG")
    items.append(("png", b.getvalue()))
    b = io.BytesIO()
    Image.fromarray(photo(64, 48)).save(b, "JPEG", progressive=True)
    items.append(("progressive", b.getvalue()))
    items.append(("photo", encode(photo(640, 480), 2, 85, "rows")))
    items.append(("flipped", corrupt(encode(photo(96, 80), 2, 90, None), "flip")))
    return write(tmp_path, items)


def test_mixed_batches_equal_single_decodes(tmp_path):
    paths = mixed(tmp_path)
    dec = JpegDecoder("cuda", read_image)
    whole = dec(paths).numpy()
    split = JpegDecoder("cuda", read_image, workspace_budget=1 << 16)(paths).numpy()  # many launches into one output
    for p, a, b in zip(paths, whole, split):
        alone = dec([p]).numpy()[0]
        assert np.array_equal(a, alone) and np.array_equal(b, alone) and np.array_equal(alone, read_image(p)), p


def test_corrupted_streams(tmp_path):
    good = encode(photo(96, 80), 2, 90, None)
    rst = encode(photo(96, 80), 2, 90, "blocks")
    items = [("flip", corrupt(good, "flip")), ("ac_overrun", corrupt(good, "ac_overrun")),
             ("early_eoi", corrupt(good, "early_eoi")), ("drop_rst", corrupt(rst, "drop_rst")),
             ("early_eoi_dri", corrupt(rst, "early_eoi")), ("truncated", good[:len(good) // 2])]
    paths = write(tmp_path, items)
    expect = []
    for p in paths:
        try:
            expect.append(read_image(p))
        except Exception as e:  # noqa: BLE001 - the same exception type must come out of the device path
            expect.append(type(e))
    dec = JpegDecoder("cuda", read_image)
    for (name, _), p, e in zip(items, paths, expect):
        if isinstance(e, type):
            with pytest.raises(e):
                dec([p])
            continue
        batch = dec([p])
        assert batch.status[0] != 0, name  # the device did not take the stream as it is
        if name in ("flip", "ac_overrun", "early_eoi"):
            assert batch.reasons[0] == _lib.JPEG_DEVICE and batch.status[0] & ~_lib.JPEG_BAD_SKIPPED, name
        assert np.array_equal(batch.numpy()[0], e), name


def test_deterministic(tmp_path):
    paths = mixed(tmp_path)
    a = JpegDecoder("cuda", read_image)(paths)
    b = JpegDecoder("cuda", read_image)(paths)
    assert torch.equal(a.data, b.data) or all(np.array_equal(x, y) for x, y in zip(a.numpy(), b.numpy()))


def folder(tmp_path, splits, ids=3, per=5):
    rng = np.random.default_rng(5)
    for split in splits:
        for i in range(ids):
            d = tmp_path / split / f"id{i}"
            os.makedirs(d)
            for j in range(per):
                w, h = int(rng.integers(60, 300)), int(rng.integers(60, 300))
                sub = [0, 1, 2, "gray"][(i + j) % 4]
                (d / f"{j}.jpg").write_bytes(encode(photo(w, h, seed=100 * i + j), sub, 90, [None, "rows"][j % 2]))
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
    folder(tmp_path, ("train",), ids=3, per=6)
    with open(os.path.join(GOLDEN, "reference_configs", "cbir.yaml")) as f:
        cfg = yaml.safe_load(f)["data"]
    cfg = dict(cfg, nw=2)
    cfg["train"] = dict(cfg["train"], bs=4, aug_epoch=2)
    data = FolderTrainData(str(tmp_path), cfg, 3, "cuda", warm_ep=1, seed=3)
    for epoch in (0, 1):  # val list, train list
        dev = list(data.train_batches(epoch))
        import engine.folder_train as FT
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


def host_result(path):
    try:
        return read_image(path)
    except Exception as e:  # noqa: BLE001 - the device path must raise the same type
        return type(e)


def test_files_pillow_refuses_raise_what_read_image_raises(tmp_path):
    bad = write(tmp_path, [("all_ones", all_ones_code(encode(photo(96, 80), 2, 90, None)))])[0]
    expect = host_result(bad)
    assert isinstance(expect, type)
    with pytest.raises(expect):
        JpegDecoder("cuda", read_image)([bad])


def test_pixel_limit_follows_pillow(tmp_path, monkeypatch):
    """Above PIL.Image.MAX_IMAGE_PIXELS Image.open warns, above twice that it raises DecompressionBombError: such files take
    the host path, and the limit is read when the batch is decoded."""
    paths = write(tmp_path, [("small", encode(photo(40, 30), 2, 90, None)), ("mid", encode(photo(64, 48), 2, 90, None)),
                             ("big", encode(photo(96, 80), 2, 90, None))])
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 2000)
    dec = JpegDecoder("cuda", read_image)
    with pytest.warns(Image.DecompressionBombWarning):
        batch = dec(paths[:2])
    assert batch.reasons == [_lib.JPEG_DEVICE, _lib.JPEG_TOO_LARGE] and batch.status[0] == 0
    for p, got in zip(paths, batch.numpy()):
        assert np.array_equal(got, pil(p))
    with pytest.raises(Image.DecompressionBombError):
        dec(paths)


def test_batches_raise_with_the_batch_of_the_failing_file(tmp_path):
    """An unreadable file surfaces when its own batch is finished, after the batches before it, like the host path."""
    from engine.cbir.folder import decode_batches, device_decode_batches
    paths = write(tmp_path, [(f"{k}", encode(photo(40, 30, seed=k), 2, 90, None)) for k in range(4)])
    junk = tmp_path / "junk.png"
    junk.write_bytes(b"not an image at all")
    files = paths + [str(junk)]
    seen = []
    for gen in (decode_batches(files, 2, 2), device_decode_batches(files, 2, "cuda", 2)):
        got = []
        with pytest.raises(Exception) as e:
            for b in gen:
                got.append(len(b))
        assert got == [2, 2]
        seen.append(type(e.value))
    assert seen[0] is seen[1]
