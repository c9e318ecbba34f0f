"""Image-folder source of the CBIR evaluation: the reference's local `CBIRDatasets` layout (dataset/basedataset.py:463-596)

    <root>/query/<identity>/*.jpg|png        <root>/gallery/<identity>/*.jpg|png        (query identities must be a subset)

read the way the reference reads it (`Image.open(path).convert('RGB')`, cv2 fallback: basedataset.py:234-241) and fed to the
H100 path: decoded RGB bytes -> visiondk_b200.preprocess (the val transform list on the device, bit-exact with the reference's
PIL / torchvision pipeline) -> embed -> index -> search.  On a CUDA device the baseline JPEGs are decoded there
(visiondk_b200.jpeg, bit-exact with `read_image`) and every other file with `read_image` on host threads (`nw`) inside the
same batch, one batch ahead of the consumer; `decode_batches` / `decoded_batches` are the host path.

Only the deterministic eval list of the reference's configs is built — `resize_and_padding(size, training=False)` ->
`to_tensor` -> `normalize(mean, std)` (configs/faceX/cbir.yaml, data.val.augment); anything else raises with its name.
Relevance is an identity-label comparison: a query's positives (`data['pos']`, basedataset.py:507-511) are exactly the
gallery files of its identity folder."""
from __future__ import annotations

import glob
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch


def parse_val_augment(augment: Sequence[dict]) -> Tuple[int, Tuple[float, ...], Tuple[float, ...]]:
    """data.val.augment (a list of one-key dicts, dataset/transforms.py:530-555) -> (size, mean, std) of the supported list."""
    names = [next(iter(a.keys())) for a in augment]
    if names != ["resize_and_padding", "to_tensor", "normalize"]:
        raise NotImplementedError(f"val.augment {names}: the device pipeline builds resize_and_padding -> to_tensor -> normalize "
                                  "(the eval list of the reference's faceX / cbir configs)")
    rp = augment[0]["resize_and_padding"]
    if not isinstance(rp, dict) or bool(rp.get("training", False)):
        raise NotImplementedError("resize_and_padding(training=True) draws its resampling filter at random: eval list only")
    norm = augment[2]["normalize"]
    mean = (0.485, 0.456, 0.406) if norm == "no_params" else tuple(float(v) for v in norm.get("mean", (0.485, 0.456, 0.406)))
    std = (0.229, 0.224, 0.225) if norm == "no_params" else tuple(float(v) for v in norm.get("std", (0.229, 0.224, 0.225)))
    return int(rp.get("size", 224)), mean, std


def read_image(path: str) -> np.ndarray:
    """basedataset.py:234-241 -> uint8 [h, w, 3] RGB."""
    from PIL import Image
    try:
        img = Image.open(path).convert("RGB")
    except OSError:
        import cv2
        img = Image.fromarray(cv2.cvtColor(cv2.imread(path), cv2.COLOR_BGR2RGB))
    return np.asarray(img, dtype=np.uint8)


def device_decode_batches(files: Sequence[str], batch: int, device, nw: int = 8):
    """visiondk_b200.jpeg.DecodedBatch per `batch` files: what `decode_batches` yields, already on the device."""
    from visiondk_b200.jpeg import JpegDecoder, decode_batches as jpeg_batches
    decoder = JpegDecoder(device, read_image, nw)
    try:
        yield from jpeg_batches(files, batch, decoder)
    finally:
        decoder.close()


def decode_batches(files: Sequence[str], batch: int, nw: int = 8) -> Iterable[List[np.ndarray]]:
    """Lists of decoded images, `batch` files at a time, decoded on `nw` host threads one batch ahead of the consumer."""
    chunks = [files[a:a + batch] for a in range(0, len(files), batch)]
    if not chunks:
        return
    with ThreadPoolExecutor(max(1, int(nw))) as pool:
        pending = [pool.submit(read_image, f) for f in chunks[0]]
        for j in range(len(chunks)):
            nxt = [pool.submit(read_image, f) for f in chunks[j + 1]] if j + 1 < len(chunks) else []
            yield [p.result() for p in pending]
            pending = nxt


class CBIRFolderData:
    """Query / gallery file lists, identity labels and device batches of a local CBIR root (same surface as SyntheticFaceData)."""

    def __init__(self, root: str, augment: Sequence[dict], batch: int, device, nw: int = 8, postfix: Sequence[str] = ("jpg", "png")):
        query_dir, gallery_dir = os.path.join(root, "query"), os.path.join(root, "gallery")
        if not (os.path.isdir(query_dir) and os.path.isdir(gallery_dir)):
            raise ValueError(f"{root}: make sure query dir and gallery dir exists")  # basedataset.py:482
        q_ids = sorted(d for d in os.listdir(query_dir) if not d.startswith("."))
        g_ids = sorted(d for d in os.listdir(gallery_dir) if not d.startswith("."))
        if not set(q_ids).issubset(g_ids):
            raise ValueError("query identity is not subset of gallery identity")  # basedataset.py:497
        self.identities = g_ids
        label_of = {name: i for i, name in enumerate(g_ids)}

        def files(d):  # basedataset.py:503-504: postfix[0] files, then postfix[1] files (sorted here: listing order is the ids)
            return [f for p in postfix for f in sorted(glob.glob(os.path.join(d, f"*.{p}")))]

        self.query_files: List[str] = []
        q_lab: List[int] = []
        for name in q_ids:
            fs = files(os.path.join(query_dir, name))
            self.query_files += fs
            q_lab += [label_of[name]] * len(fs)
        self.gallery_files: List[str] = []
        g_lab: List[int] = []
        for name in g_ids:
            fs = files(os.path.join(gallery_dir, name))
            self.gallery_files += fs
            g_lab += [label_of[name]] * len(fs)
        self._q_label, self._g_label = np.asarray(q_lab, np.int64), np.asarray(g_lab, np.int64)
        self.size, self.mean, self.std = parse_val_augment(augment)
        self.batch, self.device, self.nw = int(batch), torch.device(device), max(1, int(nw))
        self._pre = None

    # ---- labels (order = file order = the ids the search returns) ----
    def gallery_labels(self, limit: Optional[int] = None) -> torch.Tensor:
        return torch.from_numpy(self._g_label[:limit]).to(self.device)

    def query_labels(self, limit: Optional[int] = None) -> torch.Tensor:
        return torch.from_numpy(self._q_label[:limit]).to(self.device)

    def positives(self, limit: Optional[int] = None) -> List[List[str]]:
        """`data['pos']` of the reference: every query's positive gallery files."""
        by_label = {}
        for f, l in zip(self.gallery_files, self._g_label):
            by_label.setdefault(int(l), []).append(f)
        return [by_label.get(int(l), []) for l in self._q_label[:limit]]

    # ---- batches ----
    def decoded_batches(self, files: Sequence[str]) -> Iterable[List[np.ndarray]]:
        return decode_batches(files, self.batch, self.nw)

    def _device_batches(self, files: Sequence[str]) -> Iterable[torch.Tensor]:
        from visiondk_b200.preprocess import ImagePreprocessor
        if self._pre is None:
            self._pre = ImagePreprocessor(self.size, self.mean, self.std, self.device)
        batches = (device_decode_batches(files, self.batch, self.device, self.nw) if self.device.type == "cuda"
                   else self.decoded_batches(files))
        for images in batches:
            yield self._pre(images)

    def gallery_batches(self, limit: Optional[int] = None) -> Iterable[torch.Tensor]:
        return self._device_batches(self.gallery_files[:limit])

    def query_batches(self, limit: Optional[int] = None) -> Iterable[torch.Tensor]:
        return self._device_batches(self.query_files[:limit])
