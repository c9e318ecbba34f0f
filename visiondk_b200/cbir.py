"""CBIR eval path on H100: extract -> index -> search (SURVEY.md §8b, Seams 5 and 6).

Mirrors, by name and argument meaning:
  FeatureExtractor.extract_cbir   models/faceX/face_model.py:120-144   (.extract_face :93-118)
  index(...)                      engine/cbir/evaluation.py:106-169   (cbir_eval.py:35-96)
  search(...)                     engine/cbir/evaluation.py:171-200   (cbir_eval.py:98-122)
with the arithmetic on the sm_90a kernels: the backbone's `embed()` fuses F.normalize into the neck epilogue,
embeddings stay in HBM between extraction and search (the reference copies every batch to the host,
face_model.py:140), and the faiss objects are replaced by visiondk_b200.retrieval.FlatIPIndex and visiondk_b200.ivf.IVFIndex.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from .ivf import index_factory as make_index, parse_index_factory
from .retrieval import FlatIPIndex


def _prefetch_to_device(dataloader, device):
    """Yields device batches with the host->device copy of batch i+1 (pinned memory, side stream) overlapping the
    kernels of batch i — what the reference's DataLoader(pin_memory=True) + .to(device, non_blocking=True)
    (engine/vision_engine.py:457-468, face_model.py:136) is meant to achieve."""
    copy_stream = torch.cuda.Stream(device=device)
    main = torch.cuda.current_stream(device)

    def stage(batch):
        if isinstance(batch, (list, tuple)):
            batch = batch[0]
        if batch.device == device:
            return batch, None
        with torch.cuda.stream(copy_stream):
            dev = batch.to(device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return dev, ev

    it = iter(dataloader)
    try:
        nxt = stage(next(it))
    except StopIteration:
        return
    while nxt is not None:
        cur, ev = nxt
        try:
            nxt = stage(next(it))
        except StopIteration:
            nxt = None
        if ev is not None:
            main.wait_event(ev)
            cur.record_stream(main)
        yield cur


class FeatureExtractor:
    """models/faceX/face_model.py:88-144 (CBIR branch)."""

    def __init__(self, model):
        self.model = model

    @torch.no_grad()
    def extract_cbir_device(self, dataloader, device) -> torch.Tensor:
        """Device-resident fp32 [N, feat_dim], rows L2-normalised, dataloader order preserved."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("visiondk_b200 extraction runs on CUDA (sm_90a) only; there is no CPU fallback")
        model = self.model
        model.eval()
        model.to(device)
        feats = []
        for tensors in _prefetch_to_device(dataloader, device):
            feats.append(model.embed(tensors, l2_normalize=True))
        if not feats:
            return torch.empty((0, model.feat_dim), dtype=torch.float32, device=device)
        return torch.cat(feats, dim=0)

    @torch.no_grad()
    def extract_face(self, dataloader, device) -> dict:
        """models/faceX/face_model.py:93-118: `dataloader` yields (images, tensors, file_realpaths) (ImageDatasets.collate_fn,
        dataset/basedataset.py:455-458); returns {"<parent dir>/<file name>": L2-normalised float32 feature} — the
        `image_name2feature` dict the face evaluator (engine/faceX/evaluation.py:34-113) looks pairs up in."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("visiondk_b200 extraction runs on CUDA (sm_90a) only; there is no CPU fallback")
        model = self.model
        model.eval()
        model.to(device)
        names, feats = [], []
        for _, tensors, file_realpaths in dataloader:
            feats.append(model.embed(tensors.to(device, non_blocking=True), l2_normalize=True))
            names += [os.path.join(os.path.basename(os.path.dirname(p)), os.path.basename(p)) for p in file_realpaths]
        if not feats:
            return {}
        host = torch.cat(feats, dim=0).cpu().numpy()  # one device->host copy for the whole set (the reference copies per batch)
        return {name: host[i] for i, name in enumerate(names)}

    @torch.no_grad()
    def extract_cbir(self, dataloader, device) -> np.ndarray:
        """Reference signature: numpy float32 [N, feat_dim].  Every batch's embeddings are copied to pinned host
        memory asynchronously (the reference blocks on `.cpu().numpy()` per batch, face_model.py:140)."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("visiondk_b200 extraction runs on CUDA (sm_90a) only; there is no CPU fallback")
        model = self.model
        model.eval()
        model.to(device)
        host_chunks = []
        pool = self.__dict__.setdefault("_pinned_pool", [])  # pinned staging buffers are reused across calls: allocating
        for j, tensors in enumerate(_prefetch_to_device(dataloader, device)):  # page-locked memory synchronises with the device
            emb = model.embed(tensors, l2_normalize=True)
            if j < len(pool) and pool[j].shape == emb.shape:
                host = pool[j]
            else:
                host = torch.empty(emb.shape, dtype=torch.float32, pin_memory=True)
                if j < len(pool):
                    pool[j] = host
                elif len(pool) < 4096:
                    pool.append(host)
            host.copy_(emb, non_blocking=True)
            host_chunks.append(host)
        torch.cuda.current_stream(device).synchronize()
        if not host_chunks:
            return np.zeros((0, model.feat_dim), np.float32)
        return np.concatenate([h.numpy() for h in host_chunks], axis=0)


def memmap_shard(path: str, feat_dim: int, dtype=np.float16, rank: int = 0, world: int = 1):
    """Rows of the reference's raw embedding store (engine/cbir/evaluation.py:124-152: `[N, feat_dim]`, no header) that belong to
    `rank` of `world` under the sharded search's contiguous row split -> (np.memmap view [n_local, feat_dim], first_row, N).
    Only this rank's byte range of the file is ever touched (a 1 M x 512 fp16 store: 128 MB per rank on 8 GPUs instead of 1 GB)."""
    from .sharding import shard_bounds
    item = np.dtype(dtype).itemsize
    size = os.path.getsize(path)
    if feat_dim <= 0 or size % (item * feat_dim) != 0:
        raise ValueError(f"{path}: {size} bytes is not a whole number of {feat_dim}-wide {np.dtype(dtype).name} rows")
    n = size // (item * feat_dim)
    lo, hi = shard_bounds(n, world, rank)
    view = np.memmap(path, mode="r", dtype=dtype, offset=lo * feat_dim * item, shape=(hi - lo, feat_dim))
    return view, lo, n


def index(extractor: FeatureExtractor, gallery_dataloader, device, logger=None, index_factory: str = "Flat",
          memmap_feat_dim: Optional[int] = None, memmap_dtype=np.float16, memmap_save_path: Optional[str] = None,
          memmap_load_embedding: bool = False, shard: Optional[tuple] = None):
    """engine/cbir/evaluation.py:106-169: encode the gallery, build the inner-product index named by `index_factory`
    ("Flat" -> FlatIPIndex, "IVF<nlist>,Flat" / "IVF<nlist>,PQ<M>[x8]" -> visiondk_b200.ivf.IVFIndex; resident on `device`),
    optionally save / load the embeddings as a raw np.memmap (:124-152).  An IVF index trains on the sampled rows of a loaded
    store and adds it chunk by chunk, so the store is never uploaded whole.
    shard=(rank, world) with memmap_load_embedding: this rank loads only ITS rows of the store and the index carries their
    global ids (`id_offset`) — the per-rank index visiondk_b200.retrieval.sharded_flat_search expects (BASELINE config 4)."""
    flat = parse_index_factory(index_factory) is None  # refuses unknown strings before anything runs
    if shard is not None and not flat:
        raise ValueError(f"shard=(rank, world) builds per-rank Flat indexes; index_factory {index_factory!r} is not sharded")
    device = torch.device(device)
    id_offset = 0
    if shard is not None and not memmap_load_embedding:
        raise ValueError("shard=(rank, world) selects rows of a saved embedding store: it needs memmap_load_embedding=True")
    if memmap_load_embedding:
        if shard is not None:
            emb, id_offset, _ = memmap_shard(memmap_save_path, memmap_feat_dim, memmap_dtype, shard[0], shard[1])
        else:
            emb = np.memmap(memmap_save_path, mode="r", dtype=memmap_dtype).reshape(-1, memmap_feat_dim)
        if flat:
            emb = torch.from_numpy(np.ascontiguousarray(emb, dtype=np.float32)).to(device)
    else:
        emb = extractor.extract_cbir_device(gallery_dataloader, device)
        if memmap_save_path is not None:
            if logger is not None:
                logger.console(f"saving embeddings at {memmap_save_path}...")
            host = emb.cpu().numpy()
            mm = np.memmap(memmap_save_path, shape=host.shape, mode="w+", dtype=host.dtype)
            mm[:] = host
            mm.flush()
    faiss_index = make_index(emb.shape[-1], index_factory, device, id_offset=id_offset)
    if logger is not None:
        logger.console("Adding embeddings...")
    faiss_index.train(emb)
    faiss_index.add(emb)
    return faiss_index


def search(extractor: FeatureExtractor, query_dataloader, faiss_index, device, logger=None, k: int = 100,
           batch_size: int = 256):
    """engine/cbir/evaluation.py:171-200.  The reference searches in `batch_size` slices because faiss wants host
    arrays per call; here the whole query block is scored in one pass (each gallery tile is read once for all
    queries), so `batch_size` is accepted and ignored.  Returns numpy (scores [n,k] desc, ids [n,k], -1 padded)."""
    q = extractor.extract_cbir_device(query_dataloader, device)
    if logger is not None:
        logger.console("Searching ...")
    scores, ids = faiss_index.search_device(q, k, resolve_overflow=True)
    return scores.cpu().numpy(), ids.cpu().numpy()
