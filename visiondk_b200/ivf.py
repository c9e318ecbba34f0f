"""Inverted-file indexes on H100: the approximate faiss index_factory strings of the reference's CBIR path.

engine/cbir/evaluation.py:110,155 and cbir_eval.py:40,82 pass `index_factory` to
`faiss.index_factory(dim, index_factory, METRIC_INNER_PRODUCT)`.  `index_factory()` here accepts exactly "Flat" (FlatIPIndex),
"IVF<nlist>,Flat" and "IVF<nlist>,PQ<M>[x8]" (IVFIndex) and refuses everything else before any kernel runs.

IVFIndex is faiss-shaped like FlatIPIndex (is_trained / train / add / search / search_device / nprobe / ntotal / reset).  Its
arithmetic is deterministic and restated bit for bit in oracle/ivf.py: k-means with the fixed-order update of
vdk_kmeans_update, coarse assignment and probing by a FlatIPIndex over the centroids (canonical scores, ties to the lowest
list), PQ encoding / lookup tables / list scans in csrc/ivf.cu, and the exact key selection of the exhaustive flat path.
"""
from __future__ import annotations

import re
from typing import Optional

import numpy as np
import torch

from . import _lib
from .retrieval import FlatIPIndex, PreparedRows, _dev

NITER = 25
SEED = 1234
MAX_ROWS_PER_CENTROID = 256
PQ_K = 256
MAX_PQ_M = 128  # one query's lookup table, M * 256 fp32, must fit in shared memory

_FACTORY = re.compile(r"IVF([1-9][0-9]*),(?:(Flat)|PQ([1-9][0-9]*)(?:x8)?)")
_ACCEPTED = "'Flat', 'IVF<nlist>,Flat', 'IVF<nlist>,PQ<M>' and 'IVF<nlist>,PQ<M>x8' (inner product)"


def parse_index_factory(spec, d: Optional[int] = None):
    """-> None for "Flat", (nlist, None) for IVF-Flat, (nlist, M) for IVF-PQ.  Raises ValueError for any other string, and for
    M that does not divide d (when d is given) or exceeds 128."""
    if spec == "Flat":
        return None
    m = _FACTORY.fullmatch(spec) if isinstance(spec, str) else None
    if m is None:
        raise ValueError(f"index_factory {spec!r} is not built: the indexes built are {_ACCEPTED}")
    nlist = int(m.group(1))
    if m.group(2):
        return nlist, None
    M = int(m.group(3))
    if M > MAX_PQ_M:
        raise ValueError(f"index_factory {spec!r}: PQ{M} has more than {MAX_PQ_M} sub-quantizers (one query's lookup table, "
                         f"M x 256 floats, must fit in shared memory); the indexes built are {_ACCEPTED}")
    if d is not None and d % M != 0:
        raise ValueError(f"index_factory {spec!r}: PQ{M} does not divide the dimension {d}; the indexes built are {_ACCEPTED}")
    return nlist, M


def index_factory(d: int, spec: str, device=None, id_offset: int = 0):
    """faiss.index_factory(d, spec, METRIC_INNER_PRODUCT) for the strings parse_index_factory accepts."""
    p = parse_index_factory(spec, d)
    if p is None:
        return FlatIPIndex(d, device, id_offset=id_offset)
    if id_offset:
        raise ValueError(f"index_factory {spec!r}: IVF indexes are not sharded (id_offset must be 0)")
    return IVFIndex(d, p[0], p[1], device)


def _rows_of(x, ids: torch.Tensor, device) -> torch.Tensor:
    """Rows `ids` (ascending, CPU int64) of a numpy array / memmap or tensor -> device fp32."""
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x[ids.numpy()], dtype=np.float32)).to(device)
    return x[ids.to(x.device)].to(device, torch.float32).contiguous()


def _slice_of(x, a: int, b: int, device) -> torch.Tensor:
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x[a:b], dtype=np.float32)).to(device)
    return x[a:b].to(device, torch.float32).contiguous()


def _as_rows(x, d: int):
    if isinstance(x, np.ndarray) or isinstance(x, torch.Tensor):
        if x.ndim != 2 or x.shape[1] != d:
            raise ValueError(f"index dimension is {d}, got rows of shape {tuple(x.shape)}")
        return x
    raise TypeError("expected a numpy array (a memmap is read chunk by chunk) or a torch tensor")


class IVFIndex:
    """faiss IndexIVFFlat (pq_m=None) or IndexIVFPQ (pq_m=M, 8-bit codes by residual), METRIC_INNER_PRODUCT, on one GPU.

    Trained state, readable: `centroids` fp32 [nlist, d]; `codebooks` fp32 [M, 256, d/M] (IVF-PQ).  Stored rows, list-major
    with ascending ids inside a list: `list_offsets` int64 [nlist + 1], `list_ids` int64 [ntotal], and `list_rows` fp32
    [ntotal, d] (IVF-Flat) or `codes` uint8 [ntotal, M] (IVF-PQ)."""

    assign_chunk_rows = 1 << 15  # queries per coarse-quantizer call (its workspace is ~160 KB per query)
    add_chunk_rows = 1 << 16     # fp32 rows resident at once while adding
    search_chunk_keys = 1 << 25  # candidate keys resident at once while searching (256 MB)

    def __init__(self, d: int, nlist: int, pq_m: Optional[int] = None, device=None):
        _lib.load()
        self.d, self.nlist = int(d), int(nlist)
        if self.d % 64 != 0 or not 64 <= self.d <= 512:
            raise ValueError(f"IVF indexes take a dimension that is a multiple of 64, at most 512 (got {d}): the coarse quantizer "
                             "is a FlatIPIndex")
        if not 1 <= self.nlist < (1 << 31):
            raise ValueError(f"nlist must be positive (got {nlist})")
        self.pq_m = None if pq_m is None else int(pq_m)
        if self.pq_m is not None and (not 1 <= self.pq_m <= MAX_PQ_M or self.d % self.pq_m != 0):
            raise ValueError(f"PQ{pq_m}: M must divide the dimension {d} and be at most {MAX_PQ_M}")
        self.device = _dev(device)
        self._nprobe = 1
        self.centroids: Optional[torch.Tensor] = None
        self.codebooks: Optional[torch.Tensor] = None
        self._quantizer: Optional[FlatIPIndex] = None
        self.reset()

    # ---- faiss-shaped surface -------------------------------------------------------------------
    @property
    def is_trained(self) -> bool:
        return self.centroids is not None

    @property
    def nprobe(self) -> int:
        return self._nprobe

    @nprobe.setter
    def nprobe(self, v: int) -> None:
        v = int(v)
        if v < 1:
            raise ValueError(f"nprobe must be >= 1 (got {v})")
        self._nprobe = v

    @property
    def ntotal(self) -> int:
        return int(self.list_ids.numel())

    @property
    def nbytes(self) -> int:
        """Bytes resident on the device: centroids and the quantizer's prepared copy, codebooks, lists and their payload."""
        ts = [self.centroids, self.codebooks, self.list_offsets, self.list_ids, self.list_rows, self.codes]
        if self._quantizer is not None and self._quantizer._rows is not None:
            r = self._quantizer._rows
            ts += [r.xh, r.norm, r.err]
        return sum(t.numel() * t.element_size() for t in ts if t is not None)

    def reset(self) -> None:
        """Removes the stored rows; the trained state stays (faiss' reset)."""
        dev = self.device
        self.list_offsets = torch.zeros((self.nlist + 1,), dtype=torch.int64, device=dev)
        self.list_ids = torch.empty((0,), dtype=torch.int64, device=dev)
        self.list_rows = None if self.pq_m else torch.empty((0, self.d), dtype=torch.float32, device=dev)
        self.codes = torch.empty((0, self.pq_m), dtype=torch.uint8, device=dev) if self.pq_m else None

    def train(self, x) -> None:
        """k-means of the coarse quantizer (and the PQ codebooks) on a seeded sample of x: numpy / memmap (only the sampled rows
        are read) or a tensor."""
        _lib.require_device()
        x = _as_rows(x, self.d)
        n = int(x.shape[0])
        if n < self.nlist:
            raise ValueError(f"training IVF{self.nlist} needs at least {self.nlist} rows (got {n})")
        if self.pq_m and n < PQ_K:
            raise ValueError(f"training PQ codebooks needs at least {PQ_K} rows (got {n})")
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(SEED))
        ids = perm[:min(n, MAX_ROWS_PER_CENTROID * self.nlist)].sort().values
        xs = _rows_of(x, ids, self.device)
        c = xs[torch.searchsorted(ids, perm[:self.nlist]).to(self.device)].clone()
        for _ in range(NITER):
            a = self._assign(xs, c)
            c = PreparedRows(self._kmeans_step(xs, self.d, 1, self.nlist, a[None], c), True).x32
        self._set_centroids(c)
        del xs
        if self.pq_m:
            M, dsub = self.pq_m, self.d // self.pq_m
            ids = perm[:min(n, MAX_ROWS_PER_CENTROID * PQ_K)].sort().values
            xp = _rows_of(x, ids, self.device)
            lists = self._assign(xp, self.centroids)
            r = torch.empty_like(xp)
            codes = torch.empty((xp.shape[0], M), dtype=torch.uint8, device=self.device)
            cb = torch.zeros((M, PQ_K, dsub), dtype=torch.float32, device=self.device)
            self._encode(xp, lists, cb, r, codes)  # fills the residuals
            init = torch.searchsorted(ids, perm[:PQ_K]).to(self.device)
            cb = r[init].reshape(PQ_K, M, dsub).transpose(0, 1).contiguous()
            for _ in range(NITER):
                self._encode(xp, lists, cb, r, codes)
                cb = self._kmeans_step(r, dsub, M, PQ_K, codes.t().long(), cb)
            self.codebooks = cb

    def add(self, x) -> None:
        """Appends rows with ids ntotal, ntotal + 1, ...  Rows are uploaded, assigned and encoded add_chunk_rows at a time,
        so an IVF-PQ add never holds more than one chunk of fp32 rows on the device."""
        if not self.is_trained:
            raise RuntimeError("IVFIndex.add: the index is not trained")
        _lib.require_device()
        x = _as_rows(x, self.d)
        n, base = int(x.shape[0]), self.ntotal
        if base + n >= (1 << 31):
            raise ValueError("IVF indexes hold fewer than 2^31 rows")
        lists, payload = [], []
        for a in range(0, n, self.add_chunk_rows):
            t = _slice_of(x, a, min(n, a + self.add_chunk_rows), self.device)
            lt = self._assign(t, self.centroids)
            if self.pq_m:
                codes = torch.empty((t.shape[0], self.pq_m), dtype=torch.uint8, device=self.device)
                self._encode(t, lt, self.codebooks, torch.empty_like(t), codes)
                payload.append(codes)
            else:
                payload.append(t)
            lists.append(lt)
        if n == 0:
            return
        sizes = self.list_offsets[1:] - self.list_offsets[:-1]
        old = torch.repeat_interleave(torch.arange(self.nlist, device=self.device), sizes)
        all_lists = torch.cat([old] + lists)
        order = torch.argsort(all_lists, stable=True)  # existing rows of a list stay ahead of (smaller ids than) new ones
        stored = self.codes if self.pq_m else self.list_rows
        new_payload = torch.cat([stored] + payload)[order]
        new_ids = torch.cat([self.list_ids, torch.arange(base, base + n, device=self.device)])[order]
        counts = torch.bincount(all_lists, minlength=self.nlist)
        self.list_offsets = torch.cat([torch.zeros((1,), dtype=torch.int64, device=self.device), torch.cumsum(counts, 0)])
        self.list_ids = new_ids
        if self.pq_m:
            self.codes = new_payload
        else:
            self.list_rows = new_payload

    def search(self, x, k: int):
        """numpy float32 [n, d] -> (scores float32 [n, k], ids int64 [n, k]); the faiss call of evaluation.py:193."""
        s, i = self.search_device(x, k)
        return s.cpu().numpy(), i.cpu().numpy()

    def search_device(self, q, k: int, resolve_overflow: bool = True):
        """Device tensors in/out: the exact (score desc, id asc) top-k over the rows of the min(nprobe, nlist) best lists,
        padded with (-FLT_MAX, -1).  IVF scans keep every candidate, so nothing overflows (resolve_overflow is accepted for
        FlatIPIndex compatibility)."""
        if not self.is_trained:
            raise RuntimeError("IVFIndex.search: the index is not trained")
        _lib.require_device()
        k = int(k)
        if not 1 <= k <= 1024:
            raise ValueError("k must be in [1, 1024]")
        nprobe = min(self._nprobe, self.nlist)
        if nprobe > 1024:
            raise ValueError(f"nprobe must be at most 1024 (got {nprobe})")
        if isinstance(q, np.ndarray):
            q = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32))
        q = _as_rows(q, self.d).to(self.device, torch.float32).contiguous()
        nq = q.shape[0]
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        if nq == 0:
            return out_s, out_i
        ps, pl = self._quantizer.search_device(q, nprobe, resolve_overflow=True)
        sizes = self.list_offsets[1:] - self.list_offsets[:-1]
        psz = sizes[pl]
        within = torch.cumsum(psz, 1) - psz  # offset of each probed list inside its query's candidates
        cnt = psz.sum(1)
        cum = torch.cumsum(cnt, 0).cpu()
        a = 0
        while a < nq:  # query chunks of at most search_chunk_keys candidates (at least one query)
            base = int(cum[a - 1]) if a else 0
            b = int(torch.searchsorted(cum, base + self.search_chunk_keys, right=True))
            b = min(nq, max(b, a + 1))
            self._search_chunk(q[a:b], ps[a:b], pl[a:b], within[a:b], cnt[a:b], int(cum[b - 1]) - base, k, out_s[a:b], out_i[a:b])
            a = b
        return out_s, out_i

    # ---- internals -----------------------------------------------------------------------------
    def _set_centroids(self, c: torch.Tensor) -> None:
        self.centroids = c.contiguous()
        self._quantizer = FlatIPIndex(self.d, self.device)
        self._quantizer.add(self.centroids)
        self._quantizer._finalize()  # prepared now, so nbytes does not depend on whether a search ran

    def _assign(self, x: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
        """Canonical argmax over the centroids c (ties -> lowest), by a FlatIPIndex search with k = 1."""
        quant = FlatIPIndex(self.d, self.device)
        quant.add(c)
        out = torch.empty((x.shape[0],), dtype=torch.int64, device=self.device)
        for a in range(0, x.shape[0], self.assign_chunk_rows):
            _, i = quant.search_device(x[a:a + self.assign_chunk_rows], 1, resolve_overflow=True)
            out[a:a + self.assign_chunk_rows] = i[:, 0]
        return out

    def _kmeans_step(self, x: torch.Tensor, dim: int, n_sub: int, k: int, assign: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
        """assign [n_sub, n] -> the centroids [n_sub * k, dim] (shape of c) after one vdk_kmeans_update."""
        n = assign.shape[1]
        keys = (assign + torch.arange(n_sub, device=self.device)[:, None] * k).flatten()
        order = torch.argsort(keys, stable=True) % n  # grouped by centroid, ascending rows inside a group
        counts = torch.bincount(keys, minlength=n_sub * k)
        offsets = torch.cat([torch.zeros((1,), dtype=torch.int64, device=self.device), torch.cumsum(counts, 0)])
        c = c.contiguous().clone()
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.vdk_kmeans_update(x.data_ptr(), x.shape[1], dim, n_sub, k, order.data_ptr(), offsets.data_ptr(),
                                             counts.data_ptr(), c.data_ptr(), _lib.stream_ptr()), "vdk_kmeans_update")
        return c

    def _encode(self, x: torch.Tensor, lists: torch.Tensor, cb: torch.Tensor, residual: torch.Tensor, codes: torch.Tensor) -> None:
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.vdk_pq_encode(x.data_ptr(), x.shape[0], self.d, self.centroids.data_ptr(), lists.data_ptr(), self.pq_m,
                                         cb.data_ptr(), residual.data_ptr(), codes.data_ptr(), _lib.stream_ptr()), "vdk_pq_encode")

    def _search_chunk(self, q, ps, pl, within, cnt, total: int, k: int, out_s, out_i) -> None:
        lib = _lib.load()
        nc, nprobe = pl.shape
        coff = torch.cumsum(cnt, 0) - cnt
        pair_out = (coff[:, None] + within).contiguous()
        keys = torch.empty((max(total, 1),), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            if self.pq_m:
                lut = torch.empty((nc, self.pq_m, PQ_K), dtype=torch.float32, device=self.device)
                _lib.check(lib.vdk_pq_lut(q.data_ptr(), nc, self.d, self.pq_m, self.codebooks.data_ptr(), lut.data_ptr(),
                                          _lib.stream_ptr()), "vdk_pq_lut")
                _lib.check(lib.vdk_ivf_pq_scan(nc, nprobe, pl.contiguous().data_ptr(), ps.contiguous().data_ptr(), pair_out.data_ptr(),
                                               self.list_offsets.data_ptr(), self.codes.data_ptr(), self.pq_m, self.list_ids.data_ptr(),
                                               lut.data_ptr(), keys.data_ptr(), _lib.stream_ptr()), "vdk_ivf_pq_scan")
            elif total > 0:
                # invert the (query, list) pairs: each list's queries are scored as groups of <= 8 per CTA
                flat = pl.flatten()
                order = torch.argsort(flat, stable=True)
                per = torch.bincount(flat, minlength=self.nlist)
                start = torch.cumsum(per, 0) - per
                n_items_per = (per + 7) // 8
                item_list = torch.repeat_interleave(torch.arange(self.nlist, device=self.device), n_items_per)
                item_base = torch.cumsum(n_items_per, 0) - n_items_per
                rank = torch.arange(item_list.numel(), device=self.device) - torch.repeat_interleave(item_base, n_items_per)
                first = start[item_list] + 8 * rank
                count = torch.clamp(per[item_list] - 8 * rank, max=8)
                items = torch.stack([item_list, first, count], 1).to(torch.int32).contiguous()
                pair_query = (order // nprobe).to(torch.int32)
                pair_out_sorted = pair_out.flatten()[order].contiguous()
                _lib.check(lib.vdk_ivf_flat_scan(q.data_ptr(), self.d, items.data_ptr(), items.shape[0], pair_query.data_ptr(),
                                                 pair_out_sorted.data_ptr(), self.list_offsets.data_ptr(), self.list_rows.data_ptr(),
                                                 self.list_ids.data_ptr(), keys.data_ptr(), _lib.stream_ptr()), "vdk_ivf_flat_scan")
            _lib.check(lib.vdk_topk_select_keys(keys.data_ptr(), coff.data_ptr(), cnt.contiguous().data_ptr(), nc, k, out_s.data_ptr(),
                                                out_i.data_ptr(), _lib.stream_ptr()), "vdk_topk_select_keys")
