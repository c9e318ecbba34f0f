"""Baseline and progressive JPEG decoding on the device (csrc/jpeg.cu), bit-exact with `Image.open(path).convert("RGB")` for
the files it takes, with the host decoder inside the same batch for every other file.

    dec = JpegDecoder("cuda", host_decode=read_image)
    batch = dec(paths)              # DecodedBatch: device uint8 RGB buffer + vdk_image_desc array + shapes
    ImagePreprocessor(224)(batch)   # or TrainAugmenter(...)(batch, ...): no host round trip

Per batch, `start`: read the files on host threads, parse their headers (vdk_jpeg_parse, then vdk_jpeg_parse_progressive on
the files the first parser leaves as VDK_JPEG_PROCESS; host), submit every file the device does not take (not a JPEG,
outside the baseline and progressive sets, more pixels than PIL.Image.MAX_IMAGE_PIXELS) to `host_decode` on host threads,
upload only the compressed bytes, descriptors, restart-interval table and scan table (one copy), launch the decode.  `finish`:
read back the per-image status words (one small copy), decode with `host_decode` the streams the device flagged as not well
formed, and upload the host-decoded images into their slots.  An exception `host_decode` raises is raised by `finish`, for
the first failing file of the batch, as a host decoder would raise it for that batch.
The output layout is the packed [h][w][3] at 256-byte aligned offsets that `ImagePreprocessor._upload` produces."""
from __future__ import annotations

import ctypes as C
from concurrent.futures import Future, ThreadPoolExecutor
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import _lib


def _read(path: str) -> bytes:
    with open(path, "rb") as f:
        return f.read()


def _up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class DecodedBatch:
    """Decoded RGB images on the device: `data` (uint8 buffer), `descs` (vdk_image_desc array, one per image, in file order),
    `shapes` ((h, w, 3) per image), `status` (the device status word per image; VDK_JPEG_BAD_SKIPPED for files it did not
    take) and `reasons` (the parser's VDK_JPEG_* per file)."""

    def __init__(self, data: torch.Tensor, descs, shapes, status: List[int], reasons: List[int]):
        self.data, self.descs, self.shapes, self.status, self.reasons = data, descs, shapes, status, reasons

    def __len__(self):
        return len(self.shapes)

    def numpy(self) -> List[np.ndarray]:
        host = self.data.cpu().numpy()
        return [host[d.offset:d.offset + h * w * 3].reshape(h, w, 3).copy() for d, (h, w, _) in zip(self.descs, self.shapes)]


class _Pending:
    """A batch whose device decode is queued: what finish() needs to complete it."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class JpegDecoder:
    """Reusable staging for device JPEG decoding: a pinned buffer for the compressed bytes and descriptors, its device copy,
    the decode workspace, and a pinned buffer for host-decoded images; one event fences each pinned buffer's reuse.  A batch
    whose workspace would exceed `workspace_budget` bytes is decoded in several launches into the same output buffer."""

    def __init__(self, device="cuda", host_decode: Callable[[str], np.ndarray] = None, nw: int = 8,
                 workspace_budget: int = 1 << 30):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("visiondk_b200 JPEG decoding runs on CUDA (sm_90a) only; there is no CPU fallback")
        if host_decode is None:
            raise ValueError("JpegDecoder needs the host decoder of the files the device does not take")
        self.host_decode, self.nw, self.budget = host_decode, max(1, int(nw)), int(workspace_budget)
        self._pool = None
        self._pinned = self._dev = self._ws = None
        self._segs = np.zeros(1 << 12, np.int64)  # restart-interval starts, filled by the parsers
        self._scans = (_lib.JpegScan * 64)()  # scans of the progressive files, filled by vdk_jpeg_parse_progressive
        self._copied = None  # event after the last copy out of _pinned
        self._img_pinned = None
        self._img_copied = None  # event after the last copy out of _img_pinned

    def pool(self) -> ThreadPoolExecutor:
        if self._pool is None:
            self._pool = ThreadPoolExecutor(self.nw)
        return self._pool

    def close(self):
        if self._pool is not None:
            self._pool.shutdown()
            self._pool = None

    def __call__(self, files: Sequence[str]) -> DecodedBatch:
        return self.finish(self.start(files))

    def read(self, files: Sequence[str]) -> List[Future]:
        return [self.pool().submit(_read, f) for f in files]

    # ---- stage 1: read, parse, upload, launch (host-path files are only submitted to the thread pool) ----
    def start(self, files: Sequence[str], reads: Optional[List[Future]] = None) -> _Pending:
        from PIL import Image
        lib = _lib.load()
        files = list(files)
        n = len(files)
        if reads is None:
            reads = self.read(files)
        blobs = []
        for r in reads:  # an unreadable file goes to host_decode, which raises its error when the batch is finished
            try:
                blobs.append(r.result())
            except OSError:
                blobs.append(b"")
        offs, off = [], 0
        for b in blobs:
            offs.append(off)
            off = _up(off + len(b), 16)
        descs = (_lib.JpegDesc * max(n, 1))()
        for i, b in enumerate(blobs):
            descs[i].data_offset, descs[i].data_bytes = offs[i], len(b)
        if self._copied is not None:  # the previous batch's upload still reads the pinned buffer refilled below
            self._copied.synchronize()
        self._reserve(_up(off, 256))
        host = self._pinned.numpy()
        for i, b in enumerate(blobs):
            host[offs[i]:offs[i] + len(b)] = np.frombuffer(b, np.uint8)
        device = (_lib.JPEG_DEVICE, _lib.JPEG_DEVICE_PROGRESSIVE)
        while n:  # parse; again with larger restart-interval and scan tables when these were too small
            _lib.check(lib.vdk_jpeg_parse(self._pinned.data_ptr(), descs, n, self._segs.ctypes.data, len(self._segs)),
                       "vdk_jpeg_parse")
            _lib.check(lib.vdk_jpeg_parse_progressive(self._pinned.data_ptr(), descs, n, self._scans, len(self._scans),
                                                      self._segs.ctypes.data, len(self._segs)), "vdk_jpeg_parse_progressive")
            need = max([descs[i].seg_first + descs[i].n_segments for i in range(n) if descs[i].reason in device], default=0)
            need_scans = max([descs[i].scan_first + descs[i].n_scans for i in range(n)
                              if descs[i].reason == _lib.JPEG_DEVICE_PROGRESSIVE], default=0)
            if need <= len(self._segs) and need_scans <= len(self._scans):
                break
            if need > len(self._segs):
                self._segs = np.zeros(need * 2, np.int64)
            if need_scans > len(self._scans):
                self._scans = (_lib.JpegScan * (need_scans * 2))()
            for i, b in enumerate(blobs):
                descs[i].data_offset, descs[i].data_bytes = offs[i], len(b)
        limit = Image.MAX_IMAGE_PIXELS  # read per call: users set it; above it Image.open warns, above twice it raises
        for i in range(n):
            if descs[i].reason in device and limit is not None and descs[i].width * descs[i].height > limit:
                descs[i].reason = _lib.JPEG_TOO_LARGE
        reasons = [int(descs[i].reason) for i in range(n)]
        on_dev = [i for i in range(n) if reasons[i] in device]
        host_jobs = {i: self.pool().submit(self.host_decode, files[i]) for i in range(n) if reasons[i] not in device}
        shapes: List[Optional[tuple]] = [None] * n
        slots, out_bytes = [0] * n, 0
        for i in on_dev:
            shapes[i] = (int(descs[i].height), int(descs[i].width), 3)
            slots[i] = descs[i].out_offset = out_bytes
            out_bytes += _up(shapes[i][0] * shapes[i][1] * 3, 256)
        # device images in consecutive groups whose workspace fits the budget; every group's descriptors and the restart-
        # interval table are uploaded with the compressed bytes in one copy
        groups, cur, cur_bytes = [], [], 0
        for i in on_dev:
            d = descs[i]
            need = 192 * d.mcus_x * d.mcus_y * (d.h[0] * d.v[0] + (2 if d.ncomp == 3 else 0)) + 512
            if cur and cur_bytes + need > self.budget:
                groups.append(cur)
                cur, cur_bytes = [], 0
            cur.append(i)
            cur_bytes += need
        if cur:
            groups.append(cur)
        launches, at, ws_need = [], _up(off, 256), 0
        for g in groups:
            arr = (_lib.JpegDesc * len(g))(*[descs[i] for i in g])
            need = lib.vdk_jpeg_workspace_bytes(arr, len(g))
            if need == 0:
                raise RuntimeError("vdk_jpeg_workspace_bytes: " + _lib.last_error())
            ws_need = max(ws_need, need)
            launches.append((g, arr, at))
            at += C.sizeof(arr)
        seg_at = _up(at, 256)
        n_segs = max([descs[i].seg_first + descs[i].n_segments for i in on_dev], default=0)
        scan_at = _up(seg_at + 8 * n_segs, 256)
        n_scans = max([descs[i].scan_first + descs[i].n_scans for i in on_dev if reasons[i] == _lib.JPEG_DEVICE_PROGRESSIVE],
                      default=0)
        total = scan_at + C.sizeof(_lib.JpegScan) * n_scans
        self._reserve(total)
        for g, arr, g_at in launches:
            C.memmove(self._pinned.data_ptr() + g_at, C.addressof(arr), C.sizeof(arr))
        C.memmove(self._pinned.data_ptr() + seg_at, self._segs.ctypes.data, 8 * n_segs)
        C.memmove(self._pinned.data_ptr() + scan_at, C.addressof(self._scans), C.sizeof(_lib.JpegScan) * n_scans)
        out = torch.empty((max(out_bytes, 256),), dtype=torch.uint8, device=self.device)
        status = torch.zeros((max(len(on_dev), 1),), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            self._dev[:total].copy_(self._pinned[:total], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
            if ws_need and (self._ws is None or self._ws.numel() < ws_need):
                self._ws = torch.empty((ws_need,), dtype=torch.uint8, device=self.device)
            s = 0
            base = self._dev.data_ptr()
            for g, arr, g_at in launches:
                if n_scans:  # baseline and progressive images
                    _lib.check(lib.vdk_jpeg_decode_ex(base, arr, base + g_at, base + seg_at, C.addressof(self._scans),
                                                      base + scan_at, len(g), out.data_ptr(), status.data_ptr() + 4 * s,
                                                      self._ws.data_ptr(), self._ws.numel(), _lib.stream_ptr()),
                               "vdk_jpeg_decode_ex")
                else:
                    _lib.check(lib.vdk_jpeg_decode(base, arr, base + g_at, base + seg_at, len(g), out.data_ptr(),
                                                   status.data_ptr() + 4 * s, self._ws.data_ptr(), self._ws.numel(),
                                                   _lib.stream_ptr()), "vdk_jpeg_decode")
                s += len(g)
            status_host = status.to("cpu", non_blocking=True) if on_dev else None
            done = torch.cuda.Event()
            done.record()
        return _Pending(files=files, n=n, on_dev=on_dev, reasons=reasons, shapes=shapes, slots=slots, out=out,
                        status_host=status_host, done=done, host_jobs=host_jobs)

    def _reserve(self, nbytes: int) -> None:
        """Grows the pinned staging buffer (keeping its contents) and its device copy to at least `nbytes`."""
        if self._pinned is not None and self._pinned.numel() >= nbytes:
            return
        bigger = torch.empty((nbytes * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        if self._pinned is not None:
            bigger[:self._pinned.numel()].copy_(self._pinned)
        self._pinned = bigger
        self._dev = torch.empty((nbytes * 5 // 4,), dtype=torch.uint8, device=self.device)

    # ---- stage 2: host decodes, status read-back, host decode of what the device flagged ----
    def finish(self, p: _Pending) -> DecodedBatch:
        p.done.synchronize()
        status = [_lib.JPEG_BAD_SKIPPED] * p.n
        if p.on_dev:
            for i, v in zip(p.on_dev, p.status_host.tolist()):
                status[i] = int(v)
        jobs = dict(p.host_jobs)
        jobs.update({i: self.pool().submit(self.host_decode, p.files[i]) for i in p.on_dev if status[i] != 0})
        images = {i: jobs[i].result() for i in sorted(jobs)}  # raises what host_decode raises, first file first
        out, slots, shapes = p.out, list(p.slots), list(p.shapes)
        grow = 0
        for i in sorted(images):
            im = images[i]
            if im.shape != shapes[i]:  # a host-path file, or a corrupt stream that decodes to another size: a new slot
                slots[i] = out.numel() + grow
                grow += _up(im.size, 256)
            shapes[i] = im.shape
        with torch.cuda.device(self.device):
            if grow:
                bigger = torch.empty((out.numel() + grow,), dtype=torch.uint8, device=self.device)
                bigger[:out.numel()].copy_(out)
                out = bigger
            self._put(out, images, slots)
        descs = (_lib.ImageDesc * p.n)()
        for i in range(p.n):
            descs[i].offset, descs[i].width, descs[i].height = slots[i], shapes[i][1], shapes[i][0]
        return DecodedBatch(out, descs, shapes, status, p.reasons)

    def _put(self, out: torch.Tensor, images: dict, slots: List[int]) -> None:
        """Copies host-decoded images into their slots of `out` through the pinned image buffer."""
        if not images:
            return
        sizes = {i: _up(im.size, 256) for i, im in images.items()}
        total = sum(sizes.values())
        if self._img_copied is not None:
            self._img_copied.synchronize()
        if self._img_pinned is None or self._img_pinned.numel() < total:
            self._img_pinned = torch.empty((total,), dtype=torch.uint8, pin_memory=True)
        host = self._img_pinned.numpy()
        at = 0
        for i, im in images.items():
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"{i}: expected uint8 [h, w, 3] (RGB), got {im.dtype} {im.shape}")
            host[at:at + im.size] = np.ascontiguousarray(im).reshape(-1)
            out[slots[i]:slots[i] + im.size].copy_(self._img_pinned[at:at + im.size], non_blocking=True)
            at += sizes[i]
        self._img_copied = torch.cuda.Event()
        self._img_copied.record()


def decode_batches(files: Sequence[str], batch: int, decoder: JpegDecoder):
    """DecodedBatch per `batch` files.  Before the current batch is yielded the next batch's files are read, its device decode
    is queued and its host-path files are submitted to the host threads; a host decoding error surfaces when the batch it
    belongs to is finished, as with engine.cbir.folder.decode_batches."""
    chunks = [list(files[a:a + batch]) for a in range(0, len(files), batch)]
    if not chunks:
        return
    pending = decoder.start(chunks[0])
    for j in range(len(chunks)):
        reads = decoder.read(chunks[j + 1]) if j + 1 < len(chunks) else None
        cur = decoder.finish(pending)
        if reads is not None:
            pending = decoder.start(chunks[j + 1], reads)
        yield cur
