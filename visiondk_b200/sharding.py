"""Host-side plumbing of the sharded CBIR search (SURVEY.md §8e): one process per GPU, gallery rows sharded
contiguously, two small exchanges over torch.distributed (NCCL on GPUs; the same code runs over gloo in the CPU
tests and in the single-GPU two-rank parity test).  The reference only replicates the index
(`faiss.index_cpu_to_all_gpus`, engine/cbir/evaluation.py:159-162); sharding is BASELINE config 4.  No arithmetic
happens here: scoring, packing and merging are the CUDA kernels' job.

Exchange 1: all-gather of the query embeddings every rank extracted.
Between gallery ranges (visiondk_b200.retrieval._Exchange): all-gather of each shard's RANK SKETCH (lower bounds of its scores at
ranks k, k/2, k/4, ...: 4 floats per query on 8 GPUs) from which every shard derives a lower bound of the global k-th score.
Last exchange: ONE all-gather of the per-shard top-k lists, each entry packed into a 64-bit word (score bits << 32 | id).

The collectives sit behind a small `comm` object: DistComm (torch.distributed; the product path) or LocalShardGroup (W shards on
one device, one host thread each; the single-GPU harness of the W-shard protocol).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous rows [lo, hi) of rank `rank`; sizes differ by at most one and cover [0, n) exactly."""
    return n * rank // world, n * (rank + 1) // world


def shard_sizes(n: int, world: int) -> List[int]:
    return [shard_bounds(n, world, r)[1] - shard_bounds(n, world, r)[0] for r in range(world)]


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _active() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def _all_gather_into(out: torch.Tensor, src: torch.Tensor) -> None:
    """all_gather_into_tensor; over gloo, device tensors are staged through the host (gloo gathers host memory only —
    that backend is the test harness, NCCL is the product path)."""
    world = dist.get_world_size()
    flat = (world * src.shape[0],) + tuple(src.shape[1:])  # the concatenated form every backend accepts
    if src.is_cuda and dist.get_backend() != "nccl":
        host = torch.empty(flat, dtype=out.dtype)
        dist.all_gather_into_tensor(host, src.cpu())
        out.view(flat).copy_(host)
    else:
        dist.all_gather_into_tensor(out.view(flat), src)


def all_reduce_max_(t: torch.Tensor) -> None:
    """In-place element-wise maximum over the ranks (the per-query k-th score bounds of the sharded search: 4 bytes / query)."""
    if not _active():
        return
    if t.is_cuda and dist.get_backend() != "nccl":
        host = t.cpu()
        dist.all_reduce(host, op=dist.ReduceOp.MAX)
        t.copy_(host)
    else:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)


def all_reduce_sum_(t: torch.Tensor) -> None:
    """In-place element-wise sum over the ranks (the class-sharded head's label cosines and feature-gradient partials).  NCCL
    reduces device memory; gloo (the test harness) reduces host memory, so device tensors are staged through the host."""
    if not _active():
        return
    if t.is_cuda and dist.get_backend() != "nccl":
        host = t.cpu()
        dist.all_reduce(host, op=dist.ReduceOp.SUM)
        t.copy_(host)
    else:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)


class DistComm:
    """The shards' collectives over torch.distributed (NCCL between GPUs): the product path."""

    @property
    def world(self) -> int:
        return world_size()

    @property
    def rank(self) -> int:
        return dist.get_rank() if _active() else 0

    def all_gather(self, src: torch.Tensor) -> torch.Tensor:
        """Equal-shaped `src` of every shard -> [world, *src.shape] on every shard."""
        if not _active():
            return src.unsqueeze(0)
        out = torch.empty((dist.get_world_size(),) + tuple(src.shape), dtype=src.dtype, device=src.device)
        _all_gather_into(out, src.contiguous())
        return out

    def __deepcopy__(self, memo):  # a handle on the process group: copies of a module holding it share it
        return self

    def all_reduce_max_(self, t: torch.Tensor) -> None:
        all_reduce_max_(t)

    def all_reduce_sum_(self, t: torch.Tensor) -> None:
        all_reduce_sum_(t)


class LocalShardGroup:
    """W shards living on ONE device, one host thread each: the same protocol with the collectives replaced by a barrier and a
    `torch.stack` (all threads launch on the device's default stream, so stream order = launch order).  Test / measurement
    harness only: it checks the W-shard protocol (and times a shard's share of the work) where a single GPU is available.
    A shard that waits more than `timeout` seconds for the others fails with threading.BrokenBarrierError, so that a protocol
    bug (one shard skipping a collective) fails its test instead of hanging it."""

    def __init__(self, world: int, timeout: float = 120.0):
        import threading
        self.world, self.timeout = world, timeout
        self._slots = [None] * world
        self._barrier = threading.Barrier(world, timeout=timeout)

    def comm(self, rank: int) -> "LocalShardGroup._Comm":
        return LocalShardGroup._Comm(self, rank)

    def run(self, fn: Callable, device=None) -> list:
        """fn(comm) on one thread per shard; returns the per-shard results in rank order (re-raises the first failure)."""
        import threading
        results, errors = [None] * self.world, []
        self._barrier = threading.Barrier(self.world, timeout=self.timeout)  # a failed run leaves the old one broken

        def work(rank: int) -> None:
            try:
                if device is not None:
                    torch.cuda.set_device(device)
                results[rank] = fn(self.comm(rank))
            except BaseException as e:  # noqa: BLE001 — reported to the caller below
                errors.append(e)
                self._barrier.abort()  # release the shards waiting for this one

        threads = [threading.Thread(target=work, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            first = [e for e in errors if not isinstance(e, threading.BrokenBarrierError)] or errors
            raise first[0]
        return results

    class _Comm:
        def __init__(self, group: "LocalShardGroup", rank: int):
            self.g, self.rank, self.world = group, rank, group.world

        def __deepcopy__(self, memo):  # a handle on the group: copies of a module holding it share it
            return self

        def all_gather(self, src: torch.Tensor) -> torch.Tensor:
            self.g._slots[self.rank] = src
            self.g._barrier.wait()
            out = torch.stack(list(self.g._slots))
            self.g._barrier.wait()  # nobody overwrites a slot before every thread has read it
            return out

        def all_reduce_max_(self, t: torch.Tensor) -> None:
            t.copy_(self.all_gather(t).amax(dim=0))

        def all_reduce_sum_(self, t: torch.Tensor) -> None:
            """Sum in rank order (every shard gets the same bits)."""
            parts = self.all_gather(t)
            acc = parts[0].clone()
            for p in parts[1:]:
                acc += p
            t.copy_(acc)


def all_gather_rows(local: torch.Tensor, sizes: List[int]) -> torch.Tensor:
    """Exchange 1: every rank extracted `sizes[rank]` query embeddings; returns all of them in rank order."""
    if not _active():
        return local
    # ranks may hold one row more or less: pad to the largest shard so every backend sees equal shapes
    m = max(sizes)
    padded = local.contiguous()
    if padded.shape[0] < m:
        pad = torch.zeros((m - padded.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        padded = torch.cat([padded, pad], dim=0)
    out = torch.empty((len(sizes) * m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    _all_gather_into(out, padded)
    if all(n == m for n in sizes):
        return out
    return torch.cat([out[r * m:r * m + n] for r, n in enumerate(sizes)], dim=0)


def all_gather_packed(packed: torch.Tensor) -> torch.Tensor:
    """Exchange 2: per-shard packed top-k lists [nq,k] int64 -> [world, nq, k] on every rank (one collective, 8 MB per rank
    at 10k x 100)."""
    if not _active():
        return packed.unsqueeze(0)
    world = dist.get_world_size()
    out = torch.empty((world,) + tuple(packed.shape), dtype=packed.dtype, device=packed.device)
    _all_gather_into(out, packed.contiguous())
    return out


def all_gather_topk(scores: torch.Tensor, ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Unpacked variant (two collectives): per-shard lists [nq,k] -> stacked [world, nq, k].  Kept for callers whose global
    ids do not fit the packed format (>= 2^32 - 1 gallery rows)."""
    if not _active():
        return scores.unsqueeze(0), ids.unsqueeze(0)
    world = dist.get_world_size()
    ss = torch.empty((world,) + tuple(scores.shape), dtype=scores.dtype, device=scores.device)
    ii = torch.empty((world,) + tuple(ids.shape), dtype=ids.dtype, device=ids.device)
    _all_gather_into(ss, scores.contiguous())
    _all_gather_into(ii, ids.contiguous())
    return ss, ii


def sharded_search(q_local: torch.Tensor, q_sizes: List[int], local_search: Callable, merge: Callable, k: int,
                   pack: Optional[Callable] = None, merge_packed: Optional[Callable] = None):
    """all-gather queries -> local_search(q_all, k) on this rank's shard -> all-gather lists -> merge.

    `local_search` must return COMPLETE lists (FlatIPIndex.search_device(..., resolve_overflow=True)): an overflowed query
    resolved on one rank only would silently lose candidates in the merge.  With `pack` / `merge_packed`
    (visiondk_b200.retrieval.pack_topk / merge_topk_packed) the lists travel in one collective."""
    q_all = all_gather_rows(q_local, q_sizes)
    s, i = local_search(q_all, k)
    if not _active():
        return s, i
    if pack is not None and merge_packed is not None:
        return merge_packed(all_gather_packed(pack(s, i)), k)
    ss, ii = all_gather_topk(s, i)
    return merge(ss, ii, k)
