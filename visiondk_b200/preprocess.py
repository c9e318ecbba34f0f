"""Eval-time image preprocessing on the device (SURVEY.md §8f-3): the reference's `val.augment` list —
`resize_and_padding(size, training=False)` -> `to_tensor` -> `normalize(mean, std)` (dataset/transforms.py:325-365, 466-477;
configs/faceX/cbir.yaml val.augment) — for a batch of decoded RGB images of different sizes.

    batch = resize_pad_normalize([np.uint8 [h, w, 3], ...], size=224, device="cuda")      # fp32 [n, 3, size, size]

Decoded images come either from the host (PIL / cv2; the decoded bytes are packed into one pinned buffer and cross PCIe once) or
already on the device (visiondk_b200.jpeg.DecodedBatch); the two
resampling passes + padding + ToTensor + Normalize run in csrc/preprocess.cu — bit-exact with Pillow's 8-bit BILINEAR resize and
torch's fp32 arithmetic (tests/test_preprocess_gpu.py).  No CPU fallback."""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np
import torch

from . import _lib
from .jpeg import DecodedBatch

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


class ImagePreprocessor:
    """Reusable staging (pinned host buffer, device buffer, workspace) for `resize_pad_normalize` calls of similar size."""

    def __init__(self, size: int, mean: Sequence[float] = IMAGENET_MEAN, std: Sequence[float] = IMAGENET_STD, device="cuda"):
        self.size = int(size)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("visiondk_b200 preprocessing runs on CUDA (sm_90a) only; there is no CPU fallback")
        self.mean = (C.c_float * 3)(*[float(np.float32(m)) for m in mean])
        self.std = (C.c_float * 3)(*[float(np.float32(s)) for s in std])
        self._pinned = None
        self._dev = None
        self._ws = None
        self._copied = None  # event after the last host->device copy out of the pinned buffer

    def __call__(self, images: Sequence[np.ndarray] | DecodedBatch) -> torch.Tensor:
        """`images`: decoded RGB arrays on the host, or a DecodedBatch already on the device."""
        lib = _lib.load()
        n = len(images)
        if n == 0:
            return torch.empty((0, 3, self.size, self.size), dtype=torch.float32, device=self.device)
        packed, descs = self._stage(images)
        with torch.cuda.device(self.device):
            need = lib.vdk_preprocess_workspace_bytes(descs, n, self.size)
            if need == 0:
                raise RuntimeError("vdk_preprocess_workspace_bytes: " + _lib.last_error())
            ws = self._workspace(need)
            out = torch.empty((n, 3, self.size, self.size), dtype=torch.float32, device=self.device)
            _lib.check(lib.vdk_preprocess_resize_pad_normalize(packed, descs, n, self.size, self.mean, self.std,
                                                               out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                               _lib.stream_ptr()), "vdk_preprocess_resize_pad_normalize")
        return out

    def _stage(self, images):
        """(device pointer of the packed RGB images, their descriptors): a DecodedBatch as it is, host arrays uploaded."""
        if isinstance(images, DecodedBatch):
            return images.data.data_ptr(), images.descs
        descs = self._upload(images)
        return self._dev.data_ptr(), descs

    def _upload(self, images: Sequence[np.ndarray]):
        """Packs the images into the pinned buffer and queues its copy to the device buffer; returns their descriptors."""
        n = len(images)
        descs = (_lib.ImageDesc * n)()
        off = 0
        for i, im in enumerate(images):
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"image {i}: expected uint8 [h, w, 3] (RGB), got {im.dtype} {im.shape}")
            descs[i].offset, descs[i].width, descs[i].height = off, im.shape[1], im.shape[0]
            off += (im.shape[0] * im.shape[1] * 3 + 255) // 256 * 256
        if self._copied is not None:  # the previous call's asynchronous copy still reads the pinned buffer refilled below
            self._copied.synchronize()
        if self._pinned is None or self._pinned.numel() < off:
            self._pinned = torch.empty((off,), dtype=torch.uint8, pin_memory=True)
            self._dev = torch.empty((off,), dtype=torch.uint8, device=self.device)
        host = self._pinned.numpy()
        for i, im in enumerate(images):
            o = descs[i].offset
            host[o:o + im.size] = np.ascontiguousarray(im).reshape(-1)
        with torch.cuda.device(self.device):
            self._dev[:off].copy_(self._pinned[:off], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
        return descs

    def _workspace(self, need: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty((need,), dtype=torch.uint8, device=self.device)
        return self._ws


def resize_pad_normalize(images: Sequence[np.ndarray], size: int = 224, mean: Sequence[float] = IMAGENET_MEAN,
                         std: Sequence[float] = IMAGENET_STD, device="cuda") -> torch.Tensor:
    return ImagePreprocessor(size, mean, std, device)(images)
