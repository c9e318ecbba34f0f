"""Flat inner-product index on H100: the drop-in for the faiss objects of the reference's CBIR path.

Seam (SURVEY.md §8b, Seam 6): engine/cbir/evaluation.py:155-168 builds
`faiss.index_factory(dim, "Flat", faiss.METRIC_INNER_PRODUCT)`, clones it to the GPUs, then calls
`.train(x)`, `.add(x)` and (evaluation.py:193) `.search(x, k) -> (scores float32 [n,k] desc, ids int64 [n,k])`.
FlatIPIndex answers exactly those calls with numpy in / numpy out, and adds `search_device` for callers that
keep embeddings on the GPU (what extract -> search should do on an H100; the reference's per-batch
`.cpu().numpy()` at face_model.py:140 is a host round trip the hot path does not need).

Results are EXACT inner-product top-k under the canonical score / tie rule of oracle/retrieval.py
(score desc, id asc), independent of how the gallery is sharded.  The fp16 tensor-core pass only nominates
candidates; every returned score is re-computed from the fp32 rows.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib

FLT_LOWEST = -3.4028234663852886e38


def _dev(device) -> torch.device:
    d = torch.device(device if device is not None else "cuda")
    if d.type != "cuda":
        raise RuntimeError("visiondk_b200 runs on CUDA (sm_90a) devices only; there is no CPU path")
    return d


class PreparedRows:
    """fp32 rows + fp16 copy + norm / rounding-error bounds, all resident in HBM."""

    def __init__(self, x: torch.Tensor, normalize: bool):
        lib = _lib.load()
        if x.dim() != 2:
            raise ValueError(f"expected [n, dim] rows, got shape {tuple(x.shape)}")
        x = x.contiguous().float()
        n, dim = x.shape
        self.n, self.dim = n, dim
        self.x32 = x if not normalize else torch.empty_like(x)
        self.xh = torch.empty((n, dim), dtype=torch.float16, device=x.device)
        self.norm = torch.empty((n,), dtype=torch.float32, device=x.device)
        self.err = torch.empty((n,), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(lib.vdk_rows_prepare(_lib.ptr(x), n, dim, int(normalize), _lib.ptr(self.x32), _lib.ptr(self.xh),
                                            _lib.ptr(self.norm), _lib.ptr(self.err), _lib.stream_ptr()),
                       "vdk_rows_prepare")

    def maxima(self) -> Tuple[torch.Tensor, torch.Tensor]:
        lib = _lib.load()
        out = torch.zeros((2,), dtype=torch.float32, device=self.x32.device)
        with torch.cuda.device(self.x32.device):
            _lib.check(lib.vdk_reduce_max(_lib.ptr(self.norm), self.n, out.data_ptr(), _lib.stream_ptr()),
                       "vdk_reduce_max")
            _lib.check(lib.vdk_reduce_max(_lib.ptr(self.err), self.n, out.data_ptr() + 4, _lib.stream_ptr()),
                       "vdk_reduce_max")
        return out[0:1], out[1:2]


class FlatIPIndex:
    """Exact inner-product index (faiss "Flat", METRIC_INNER_PRODUCT) with the gallery resident on one GPU.

    normalize=True fuses F.normalize (face_model.py:139) into add()/search(), i.e. cosine similarity.
    id_offset shifts returned ids (a shard's first global row under multi-GPU sharding).
    """

    def __init__(self, dim: int, device=None, normalize: bool = False, id_offset: int = 0):
        _lib.load()
        self.d = int(dim)
        self.device = _dev(device)
        self.normalize = bool(normalize)
        self.id_offset = int(id_offset)
        self.is_trained = True
        self._chunks = []
        self._rows: Optional[PreparedRows] = None
        self._gmax = None
        self._ws = None
        self.last_status = None
        self.last_plan = None
        self.stage_ends = None  # optional override of the gallery range schedule (tuning / tests)
        self.wide_path_rows = 0
        self.exhaustive_rows = 0

    # ---- faiss-shaped surface -------------------------------------------------------------------
    @property
    def ntotal(self) -> int:
        return sum(c.shape[0] for c in self._chunks) + (self._rows.n if self._rows is not None else 0)

    def train(self, x) -> None:  # Flat indexes need no training (evaluation.py:167)
        return None

    def add(self, x) -> None:
        t = self._to_device(x)
        if t.shape[1] != self.d:
            raise ValueError(f"index dimension is {self.d}, got rows of width {t.shape[1]}")
        if self._rows is not None:  # re-open: keep the fp32 rows, re-prepare on next search
            self._chunks.insert(0, self._rows.x32)
            self._rows = None
        self._chunks.append(t)

    def reset(self) -> None:
        self._chunks, self._rows, self._gmax = [], None, None

    def search(self, x, k: int):
        """numpy float32 [n, d] -> (scores float32 [n, k], ids int64 [n, k]); the faiss call of evaluation.py:193."""
        s, i = self.search_device(self._to_device(x), k, resolve_overflow=True)
        return s.cpu().numpy(), i.cpu().numpy()

    def search_l2(self, x, k: int):
        """Squared-L2 top-k for a cosine index (`normalize=True`): for unit vectors ||q - g||^2 = 2 - 2 q.g, so the k nearest in
        L2 are the k largest inner products.  Returns (distances float32 [n, k] ascending = fl(2 - 2 * canonical score), ids int64
        [n, k], -1 / +inf padded), ordered by the canonical cosine score (ties broken by id like `search`)."""
        if not self.normalize:
            raise ValueError("search_l2 needs a cosine index (normalize=True): un-normalised L2 ranks differently from inner product")
        s, i = self.search_device(self._to_device(x), k, resolve_overflow=True)
        d = torch.where(i >= 0, 2.0 - 2.0 * s, torch.full_like(s, float("inf")))
        return d.cpu().numpy(), i.cpu().numpy()

    # ---- device-resident path ----------------------------------------------------------------------
    def _run_topk(self, qp: "PreparedRows", rows, g_lo: int, g_hi: int, k: int, dense_all: bool, exchange=None):
        """One vdk_ip_topk call: queries `rows` of qp (None = all) against gallery rows [g_lo, g_hi).  With `exchange` (the
        sharded search) the call is split: per gallery range vdk_ip_topk_filter_stages -> exchange(bound, sketch) (raises the
        lower bound of the global k-th score from what all shards publish, in place), then vdk_ip_topk_rerank of the candidates
        that can still reach the global top-k."""
        lib = _lib.load()
        g = self._rows
        q32, qh, qn, qe = qp.x32, qp.xh, qp.norm, qp.err
        if rows is not None:
            q32, qh, qn, qe = q32[rows].contiguous(), qh[rows].contiguous(), qn[rows].contiguous(), qe[rows].contiguous()
        nq, ng = q32.shape[0], g_hi - g_lo
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        status = torch.zeros((4,), dtype=torch.int32, device=self.device)
        plan = _lib.TopkPlan()
        _lib.check(lib.vdk_topk_plan_default(C.byref(plan), nq, ng, self.d, k), "vdk_topk_plan_default")
        ends = None
        if dense_all:  # wide path: every range scored densely -> no admission threshold, no segment can overflow
            cap = plan.cand_capacity
            ends = list(range(cap, ng, cap))
            plan.dense_mask = 0xFF
        elif self.stage_ends is not None:
            ends = [int(e) for e in self.stage_ends if int(e) < ng]
        elif exchange is not None and exchange.schedule is not None:
            ends = [min(int(e), ng) for e in exchange.schedule]  # the SAME number of ranges on every shard (clamped to its rows)
            while ends and ends[-1] >= ng:
                ends.pop()
            ends = ends + [ng] * (len(exchange.schedule) - len(ends))  # empty trailing ranges keep the exchange count equal
            ends = ends[:len(exchange.schedule)]
        if ends is not None and ng > 0:
            ends = ends + [ng]
            assert len(ends) <= 8, "at most 8 gallery ranges"
            plan.n_stages = len(ends)
            for j in range(8):
                plan.stage_end[j] = ends[min(j, len(ends) - 1)]
        need = lib.vdk_topk_workspace_bytes(C.byref(plan))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty((need,), dtype=torch.uint8, device=self.device)
        gn, ge = self._gmax if self._gmax is not None else (None, None)
        esz32, esz16 = 4 * self.d, 2 * self.d
        g32_ptr = (g.x32.data_ptr() + g_lo * esz32) if g else 0
        gh_ptr = (g.xh.data_ptr() + g_lo * esz16) if g else 0
        with torch.cuda.device(self.device):
            if exchange is None:
                rc = lib.vdk_ip_topk(C.byref(plan), q32.data_ptr(), qh.data_ptr(), qn.data_ptr(), qe.data_ptr(), g32_ptr, gh_ptr,
                                     _lib.ptr(gn), _lib.ptr(ge), self.id_offset + g_lo, out_s.data_ptr(), out_i.data_ptr(),
                                     status.data_ptr(), self._ws.data_ptr(), self._ws.numel(), _lib.stream_ptr())
                _lib.check(rc, "vdk_ip_topk")
            else:
                # sharded search: the shards exchange their k-th score bounds after EVERY gallery range, so each of them
                # filters the next range as if it had scanned the union of all shards' prefixes
                kth_lb = torch.full((nq,), float("-inf"), dtype=torch.float32, device=self.device)
                n_ex = plan.n_stages if exchange.schedule is None else len(exchange.schedule) + 1
                for st in range(n_ex):  # every shard runs the same number of exchanges, whatever its row count
                    if ng > 0 and st < plan.n_stages:
                        rc = lib.vdk_ip_topk_filter_stages(C.byref(plan), qh.data_ptr(), qn.data_ptr(), qe.data_ptr(), gh_ptr,
                                                           _lib.ptr(gn), _lib.ptr(ge), st, st + 1, kth_lb.data_ptr() if st > 0 else 0,
                                                           kth_lb.data_ptr(), status.data_ptr(), self._ws.data_ptr(), self._ws.numel(),
                                                           _lib.stream_ptr())
                        _lib.check(rc, "vdk_ip_topk_filter_stages")
                    done = min(st + 1, plan.n_stages)

                    def sketch(ranks, done=done):
                        sk = torch.full((nq, len(ranks)), float("-inf"), dtype=torch.float32, device=self.device)
                        if ng > 0:  # an empty shard has nothing to report
                            arr = (C.c_int32 * len(ranks))(*[int(r) for r in ranks])
                            _lib.check(lib.vdk_ip_topk_rank_sketch(C.byref(plan), done, arr, len(ranks), sk.data_ptr(),
                                                                   self._ws.data_ptr(), self._ws.numel(), _lib.stream_ptr()),
                                       "vdk_ip_topk_rank_sketch")
                        return sk

                    exchange(kth_lb, sketch)
                rc = lib.vdk_ip_topk_rerank(C.byref(plan), q32.data_ptr(), g32_ptr, self.id_offset + g_lo, kth_lb.data_ptr(),
                                            out_s.data_ptr(), out_i.data_ptr(), self._ws.data_ptr(), self._ws.numel(),
                                            _lib.stream_ptr())
                _lib.check(rc, "vdk_ip_topk_rerank")
        return out_s, out_i, status, plan

    def search_device(self, q: torch.Tensor, k: int, resolve_overflow: bool = False, exchange=None):
        """Device tensors in/out.  With resolve_overflow=True the call synchronises, and queries whose candidate
        lists overflowed (massive near-ties, adversarially ordered galleries) are recomputed on the wide path.
        `exchange` (sharded search only, see _Exchange): called after every gallery range as exchange(bound, sketch) — it raises the
        device float32 [n] `bound` (lower bound of the GLOBAL k-th canonical score) in place from what all shards publish;
        sketch(ranks) returns this shard's rank sketch.  The returned lists are then this shard's contribution to the GLOBAL
        top-k (entries that cannot reach it are dropped before the canonical re-rank) and must be merged with the other shards'."""
        _lib.load()
        _lib.require_device()
        self._finalize()
        k = int(k)
        if not (1 <= k <= 1024):
            raise ValueError("k must be in [1, 1024]")
        q = self._to_device(q)
        if q.shape[1] != self.d:
            raise ValueError(f"index dimension is {self.d}, got queries of width {q.shape[1]}")
        nq = q.shape[0]
        if nq == 0:
            return (torch.empty((0, k), dtype=torch.float32, device=self.device),
                    torch.empty((0, k), dtype=torch.int64, device=self.device))
        qp = PreparedRows(q, self.normalize)
        ng = self._rows.n if self._rows is not None else 0
        out_s, out_i, status, plan = self._run_topk(qp, None, 0, ng, k, dense_all=False, exchange=exchange)
        self.last_status, self.last_plan = status, plan
        if resolve_overflow and int(status[0].item()) > 0:
            self._wide_path(qp, out_s, out_i, plan, k)
        return out_s, out_i

    def _wide_path(self, qp: "PreparedRows", out_s: torch.Tensor, out_i: torch.Tensor, plan, k: int) -> None:
        """Recomputes the flagged queries with all-dense plans over gallery slices, merged like shards."""
        lib = _lib.load()
        flags_ptr = C.c_void_p()
        _lib.check(lib.vdk_topk_row_flags(C.byref(plan), self._ws.data_ptr(), self._ws.numel(), C.byref(flags_ptr)),
                   "vdk_topk_row_flags")
        off = flags_ptr.value - self._ws.data_ptr()
        flags = self._ws[off:off + 4 * plan.n_query].view(torch.int32)
        rows = torch.nonzero(flags).flatten()
        ng = self._rows.n
        slice_rows = 8 * plan.cand_capacity
        lists_s, lists_i = [], []
        still = torch.zeros((rows.numel(),), dtype=torch.bool, device=self.device)
        for a in range(0, ng, slice_rows):
            s_, i_, st, p_ = self._run_topk(qp, rows, a, min(ng, a + slice_rows), k, dense_all=True)
            if int(st[0].item()) > 0:  # more near-ties than a carry list holds: those rows go to the exhaustive path
                fp = C.c_void_p()
                _lib.check(lib.vdk_topk_row_flags(C.byref(p_), self._ws.data_ptr(), self._ws.numel(), C.byref(fp)),
                           "vdk_topk_row_flags")
                o = fp.value - self._ws.data_ptr()
                still |= self._ws[o:o + 4 * p_.n_query].view(torch.int32) != 0
            lists_s.append(s_)
            lists_i.append(i_)
        while len(lists_s) > 1:  # merge up to 32 lists at a time
            ms, mi = merge_topk(torch.stack(lists_s[:32]), torch.stack(lists_i[:32]), k)
            lists_s, lists_i = [ms] + lists_s[32:], [mi] + lists_i[32:]
        out_s[rows] = lists_s[0]
        out_i[rows] = lists_i[0]
        self.wide_path_rows = int(rows.numel())
        self.exhaustive_rows = 0
        if bool(still.any().item()):
            ex = rows[still]
            es, ei = self._exhaustive(qp.x32[ex].contiguous(), k)
            out_s[ex] = es
            out_i[ex] = ei
            self.exhaustive_rows = int(ex.numel())
        self.last_status = torch.zeros_like(self.last_status)

    def _exhaustive(self, q32: torch.Tensor, k: int):
        """Canonical scores of the given (already normalised) queries against every gallery row + exact selection
        (vdk_ip_topk_exhaustive): cannot overflow, whatever the number of duplicates."""
        lib = _lib.load()
        nq, ng = q32.shape[0], self._rows.n
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        ws = torch.empty((lib.vdk_ip_topk_exhaustive_workspace_bytes(ng),), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.vdk_ip_topk_exhaustive(q32.data_ptr(), nq, self._rows.x32.data_ptr(), ng, self.d, k, self.id_offset,
                                                  out_s.data_ptr(), out_i.data_ptr(), ws.data_ptr(), ws.numel(),
                                                  _lib.stream_ptr()), "vdk_ip_topk_exhaustive")
        return out_s, out_i

    def check_status(self, all_ranks: bool = False) -> dict:
        """Synchronises and raises if any query overflowed its candidate lists (results would be incomplete; the
        numpy `search()` resolves such rows on the wide path by itself).  all_ranks=True (sharded search): the status is
        first max-reduced over the process group, so every rank raises when any shard overflowed."""
        st_t = self.last_status
        if all_ranks and torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            st_t = st_t.clone()
            if torch.distributed.get_backend() != "nccl" and st_t.is_cuda:
                host = st_t.cpu()
                torch.distributed.all_reduce(host, op=torch.distributed.ReduceOp.MAX)
                st_t = host
            else:
                torch.distributed.all_reduce(st_t, op=torch.distributed.ReduceOp.MAX)
        st = st_t.cpu().tolist()
        info = {"overflow_rows": st[0], "max_candidates": st[1], "max_survivors": st[2]}
        if st[0] != 0:
            raise RuntimeError(f"vdk_ip_topk: {st[0]} query rows overflowed their candidate lists {info}; "
                               "call search_device(..., resolve_overflow=True) or search() to recompute them")
        return info

    # ---- internals -----------------------------------------------------------------------------
    def _to_device(self, x) -> torch.Tensor:
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        if not isinstance(x, torch.Tensor):
            raise TypeError("expected a numpy array or torch tensor")
        if x.dim() != 2:
            raise ValueError(f"expected [n, dim], got shape {tuple(x.shape)}")
        return x.to(self.device, torch.float32, non_blocking=True).contiguous()

    def _finalize(self) -> None:
        if not self._chunks:
            return
        rows = self._chunks[0] if len(self._chunks) == 1 else torch.cat(self._chunks, dim=0)
        self._chunks = []
        if rows.shape[0] == 0:
            self._rows, self._gmax = None, None
            return
        self._rows = PreparedRows(rows, self.normalize)
        self._gmax = self._rows.maxima()


def merge_topk(scores: torch.Tensor, ids: torch.Tensor, k: int):
    """Merge per-shard lists [n_lists, n_query, k] -> global [n_query, k] (score desc, id asc)."""
    lib = _lib.load()
    n_lists, nq, kk = scores.shape
    assert kk == k and ids.shape == scores.shape
    scores = scores.contiguous().float()
    ids = ids.contiguous().long()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=scores.device)
    with torch.cuda.device(scores.device):
        _lib.check(lib.vdk_topk_merge(scores.data_ptr(), ids.data_ptr(), n_lists, nq, k, out_s.data_ptr(),
                                      out_i.data_ptr(), _lib.stream_ptr()), "vdk_topk_merge")
    return out_s, out_i


def pack_topk(scores: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """(scores, ids) [n_query, k] -> int64 words (score bits << 32 | uint32 id): the sharded search's exchange format."""
    lib = _lib.load()
    if ids.numel() and int(ids.shape[0]) and scores.shape != ids.shape:
        raise ValueError("scores and ids must have the same shape")
    scores = scores.contiguous().float()
    ids = ids.contiguous().long()
    out = torch.empty(scores.shape, dtype=torch.int64, device=scores.device)
    with torch.cuda.device(scores.device):
        _lib.check(lib.vdk_topk_pack(scores.data_ptr(), ids.data_ptr(), scores.numel(), out.data_ptr(), _lib.stream_ptr()),
                   "vdk_topk_pack")
    return out


def merge_topk_packed(packed: torch.Tensor, k: int):
    """Packed per-shard lists [n_lists, n_query, k] (pack_topk words) -> global (scores, ids) [n_query, k]."""
    lib = _lib.load()
    n_lists, nq, kk = packed.shape
    assert kk == k and packed.dtype == torch.int64
    packed = packed.contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=packed.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=packed.device)
    with torch.cuda.device(packed.device):
        _lib.check(lib.vdk_topk_merge_packed(packed.data_ptr(), n_lists, nq, k, out_s.data_ptr(), out_i.data_ptr(),
                                             _lib.stream_ptr()), "vdk_topk_merge_packed")
    return out_s, out_i


def bound_from_sketches(sketches: torch.Tensor, ranks, k: int, bound: torch.Tensor) -> None:
    """sketches [n_shards, n_query, n_ranks] (every shard's vdk_ip_topk_rank_sketch) -> bound[n_query] = max(bound, the largest
    reported score the union provably holds k rows above): a lower bound of the global k-th canonical score, in place."""
    lib = _lib.load()
    n_shards, nq, nr = sketches.shape
    assert nr == len(ranks) and sketches.dtype == torch.float32 and bound.dtype == torch.float32
    sketches = sketches.contiguous()
    arr = (C.c_int32 * nr)(*[int(r) for r in ranks])
    with torch.cuda.device(bound.device):
        _lib.check(lib.vdk_topk_bound_from_sketches(sketches.data_ptr(), n_shards, nq, arr, nr, int(k), bound.data_ptr(),
                                                    _lib.stream_ptr()), "vdk_topk_bound_from_sketches")


class _Exchange:
    """What the shards of a sharded search tell each other after every gallery range, and the range schedule they all follow.

    sketch mode (default): every shard publishes lower bounds of its canonical scores at ranks k, k/2, k/4, ... (one all-gather
    of 4 * n_ranks bytes per query) and each shard derives the best provable lower bound of the GLOBAL k-th score
    (bound_from_sketches): ~ the k-th score of the union of all prefixes when a query's neighbours are spread over the shards,
    the best shard's k-th when they sit in one.  VDK_SHARD_SKETCH=0: element-wise max of the shards' k-th bounds only."""

    def __init__(self, schedule, comm, k: int):
        self.schedule, self.comm, self.k = schedule, comm, int(k)
        ranks = [self.k]
        if os.environ.get("VDK_SHARD_SKETCH", "1") != "0":
            r, w = self.k, 1
            while w < comm.world and len(ranks) < 8 and r > 1:
                r, w = -(-r // 2), w * 2
                ranks.append(r)
        self.ranks = ranks

    def __call__(self, bound: torch.Tensor, sketch) -> None:
        """bound [n_query] fp32, in place.  sketch(ranks) -> this shard's [n_query, len(ranks)] rank sketch."""
        if len(self.ranks) == 1:
            self.comm.all_reduce_max_(bound)
            return
        bound_from_sketches(self.comm.all_gather(sketch(self.ranks)), self.ranks, self.k, bound)


def shard_schedule(ng_max: int, world: int, k: int):
    """Gallery range ends every shard of a `world`-way search follows (computed from the LARGEST shard).  After a range every
    shard knows (from the rank sketches) about the k-th score of the union of `world` prefixes, so the next range may grow `world`
    times faster at the same expected admissions per query: 2 ranges per shard on 8 GPUs instead of 3.
    The first range is the single-GPU one and the growth 1 + 7 * world.  VDK_SHARD_FIRST / VDK_SHARD_GROWTH override (tuning)."""
    first = int(os.environ.get("VDK_SHARD_FIRST", min(max(4096, (4 * k + 255) // 256 * 256), 16384)))
    first = min(first, (max(ng_max, 1) + 255) // 256 * 256)
    growth = int(os.environ.get("VDK_SHARD_GROWTH", 1 + 7 * world))
    schedule, e = [], first
    while e < ng_max and len(schedule) < 7:
        schedule.append(e)
        e = (e * growth + 255) // 256 * 256
        if e >= 0.75 * ng_max:  # no sliver of a last range
            break
    return schedule


def sharded_flat_search(index: "FlatIPIndex", q_local: torch.Tensor, q_sizes, k: int, defer_check: bool = False, comm=None):
    """The multi-GPU search call (BASELINE config 4): every rank holds one row shard of the gallery in `index` (built with its
    `id_offset`) and `q_sizes[rank]` query embeddings; returns the GLOBAL top-k of ALL queries on every rank, bit-identical
    to the unsharded search (scores are canonical, the merge uses the same (score desc, id asc) rule).

    Exchanges: all-gather of the query embeddings; after EVERY gallery range an all-gather of the shards' rank sketches (a few
    floats per query, see _Exchange) from which each shard derives a lower bound of the global k-th score — it filters the next
    range, and finally re-ranks, only what can still reach the global top-k; ONE all-gather of the packed per-shard lists.
    Overflowed queries are resolved locally before the last exchange, so the merge never sees an incomplete list (one host
    synchronisation per search); defer_check=True skips that synchronisation — the caller then MUST call
    `index.check_status(all_ranks=True)` before trusting the result (it raises if any shard overflowed).

    comm: the shards' collectives (default sharding.DistComm = torch.distributed / NCCL).  With a sharding.LocalShardGroup comm
    (W shards on one device, one thread each: the test / measurement harness) q_local must already hold ALL queries."""
    from . import sharding

    dist_comm = comm is None or isinstance(comm, sharding.DistComm)
    comm = comm or sharding.DistComm()
    world = comm.world
    schedule = None
    if world > 1:
        # one schedule for all shards, from the LARGEST shard (cached on the index: one tiny all-reduce per index build)
        index._finalize()
        if getattr(index, "_shard_rows_max", None) is None or index._shard_rows_max[0] != index.ntotal:
            t = torch.tensor([float(index.ntotal)], device=index.device)
            comm.all_reduce_max_(t)
            index._shard_rows_max = (index.ntotal, int(t.item()))
        schedule = shard_schedule(index._shard_rows_max[1], world, k)
    ex = _Exchange(schedule, comm, k) if world > 1 else None  # one shard: the plain vdk_ip_topk call, nothing to exchange
    q_all = sharding.all_gather_rows(q_local, list(q_sizes)) if dist_comm else q_local
    s, i = index.search_device(q_all, k, resolve_overflow=not defer_check, exchange=ex)
    if world == 1:
        return s, i
    return merge_topk_packed(comm.all_gather(pack_topk(s, i)), k)


def exact_pair_scores(q32: torch.Tensor, g32: torch.Tensor, qi: torch.Tensor, gi: torch.Tensor) -> torch.Tensor:
    """Canonical scores of explicit (query, gallery) pairs — the verification kernel used by tests/bench."""
    lib = _lib.load()
    out = torch.empty((qi.numel(),), dtype=torch.float32, device=q32.device)
    with torch.cuda.device(q32.device):
        _lib.check(lib.vdk_ip_exact_pairs(q32.data_ptr(), g32.data_ptr(), q32.shape[1], qi.contiguous().data_ptr(),
                                          gi.contiguous().data_ptr(), qi.numel(), out.data_ptr(), _lib.stream_ptr()),
                   "vdk_ip_exact_pairs")
    return out
