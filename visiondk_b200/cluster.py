"""DBSCAN over embeddings on H100: the drop-in for scikit-learn's cosine DBSCAN in the reference's tools/clustering.py.

    from visiondk_b200.cluster import DBSCAN
    db = DBSCAN(eps=0.4, min_samples=5, metric="cosine", n_jobs=16).fit(X)   # the reference's call, import changed
    db.labels_, db.core_sample_indices_

Labels and core indices equal those of `sklearn.cluster.DBSCAN(eps, min_samples, metric="cosine").fit(X)` under the canonical
score of oracle/retrieval.py (oracle/cluster.py restates the rules; DESIGN §3c):
  * rows are L2-normalised by `vdk_rows_prepare` (F.normalize);
  * j is a neighbour of i iff i == j or clip(fl32(1 - s_ij), 0, 2) <= fl32(eps): scikit-learn computes float32 cosine
    distances for float32 input, and NumPy compares them with the Python float eps in float32;
  * core rows have >= min_samples neighbours (self included); clusters are the connected components of the core-core
    neighbour graph, numbered by their smallest core row; a border row takes the smallest label among its core neighbours;
    every other row is noise (-1).
The Gram matrix is never written: three fp16 tensor-core passes decide every pair, and pairs within the tensor-core error bound
of the threshold are decided by the canonical fp64 score (`vdk_dbscan`).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .retrieval import PreparedRows

MIN_DIM, MAX_DIM = 64, 512
MAX_ROWS = 2**25 - 4096  # vdk_dbscan's limit: the count pass's grid of 128 x 4096 units stays below 2^31 CTAs
F_NORMALIZE_EPS = 1e-12


def _f32(v) -> np.float32:
    return np.float32(v)


def neighbour_rule(s, eps: float) -> np.ndarray:
    """The float32 distance test scikit-learn applies to a float32 score s (array): clip(fl32(1 - s), 0, 2) <= fl32(eps)."""
    s = np.asarray(s, np.float32)
    d = np.clip(np.float32(1.0) - s, np.float32(0.0), np.float32(2.0))
    return d <= _f32(eps)


def _ord(bits: np.ndarray) -> np.ndarray:
    """float32 bit patterns (uint32) -> order-preserving int64 keys."""
    b = bits.astype(np.int64)
    return np.where(b & 0x80000000, 0x7FFFFFFF - (b & 0x7FFFFFFF), b | 0x80000000) - 0x80000000


def _unord(key: int) -> np.float32:
    k = int(key) + 0x80000000
    bits = (0x7FFFFFFF - (k & 0x7FFFFFFF)) | 0x80000000 if k < 0x80000000 else k & 0x7FFFFFFF
    return np.array([bits], np.uint32).view(np.float32)[0]


def neighbour_threshold(eps: float) -> np.float32:
    """The least float32 score s (over -inf .. +inf) that `neighbour_rule` accepts.  The rule is monotone in s, so the device
    tests s >= T.  Bisection over the ordered float32 values."""
    lo = int(_ord(np.array([0xFF800000], np.uint32))[0])  # -inf
    hi = int(_ord(np.array([0x7F800000], np.uint32))[0])  # +inf, always accepted for eps > 0
    if neighbour_rule(_unord(lo), eps):
        return _unord(lo)
    while hi - lo > 1:  # invariant: rule(lo) false, rule(hi) true
        mid = (lo + hi) // 2
        if neighbour_rule(_unord(mid), eps):
            hi = mid
        else:
            lo = mid
    return _unord(hi)


def _check_params(eps, min_samples, metric):
    if metric != "cosine":
        raise ValueError(f"DBSCAN: only metric='cosine' is supported (got {metric!r})")
    if isinstance(eps, bool) or not isinstance(eps, (int, float, np.floating, np.integer)):
        raise ValueError(f"DBSCAN: eps must be a real number (got {eps!r})")
    if not math.isfinite(float(eps)) or float(eps) <= 0.0:
        raise ValueError(f"DBSCAN: eps must be finite and > 0 (got {eps!r})")
    if isinstance(min_samples, bool) or not isinstance(min_samples, (int, np.integer)) or int(min_samples) < 1:
        raise ValueError(f"DBSCAN: min_samples must be an integer >= 1 (got {min_samples!r})")


def _check_shape(shape):
    if len(shape) != 2:
        raise ValueError(f"DBSCAN: expected rows [n, dim], got shape {tuple(shape)}")
    n, d = shape
    if n < 1:
        raise ValueError("DBSCAN: found an array with 0 rows")
    if n > MAX_ROWS:
        raise ValueError(f"DBSCAN: at most {MAX_ROWS} rows (got {n})")
    if d < MIN_DIM or d > MAX_DIM or d % 64 != 0:
        raise ValueError(f"DBSCAN: dim must be a multiple of 64 in [{MIN_DIM}, {MAX_DIM}] (got {d})")


def _check_rows_host(x: np.ndarray, first: int) -> None:
    """Non-finite rows, and rows F.normalize cannot make unit (norm below its eps 1e-12: zero rows in practice)."""
    if not np.isfinite(x).all():
        bad = first + int(np.nonzero(~np.isfinite(x).all(axis=1))[0][0])
        raise ValueError(f"DBSCAN: row {bad} is not finite")
    nrm = np.sqrt(np.einsum("ij,ij->i", x.astype(np.float64), x.astype(np.float64)))
    if (nrm < F_NORMALIZE_EPS).any():
        bad = first + int(np.nonzero(nrm < F_NORMALIZE_EPS)[0][0])
        raise ValueError(f"DBSCAN: row {bad} has zero norm: cosine distance is undefined for it")


class DBSCAN:
    """scikit-learn-shaped cosine DBSCAN on one GPU.  `n_jobs` is accepted and ignored.  X for `fit`: numpy array, np.memmap
    (read `chunk_rows` rows at a time), or torch tensor; `fit_device` takes a CUDA tensor and leaves `labels_`,
    `core_sample_indices_` and the neighbour counts on the device.  After a fit, `stats_` holds what the device reported:
    core rows, clusters, pairs rechecked by the canonical score, bands redone after a boundary-buffer overflow, and (with
    `timing=True`) per-phase milliseconds."""

    chunk_rows = 1 << 16            # host rows converted and uploaded at once
    boundary_capacity = 1 << 22     # boundary pairs buffered per pass (32 MB)

    def __init__(self, eps: float = 0.5, min_samples: int = 5, metric: str = "cosine", n_jobs=None, device=None,
                 timing: bool = False):
        self.eps = eps
        self.min_samples = min_samples
        self.metric = metric
        self.n_jobs = n_jobs
        self.device = device
        self.timing = timing

    # ---- scikit-learn surface ------------------------------------------------------------------------
    def fit(self, X, y=None, sample_weight=None):
        if sample_weight is not None:
            raise ValueError("DBSCAN: sample_weight is not supported")
        _check_params(self.eps, self.min_samples, self.metric)
        x = self._upload(X)
        labels, core, counts = self._run(x)
        self.labels_ = labels.cpu().numpy().astype(np.int64)
        self.core_sample_indices_ = core.cpu().numpy().astype(np.int64)
        self.neighbour_counts_ = counts.cpu().numpy().astype(np.int64)
        return self

    def fit_predict(self, X, y=None, sample_weight=None):
        return self.fit(X, sample_weight=sample_weight).labels_

    def fit_device(self, x: torch.Tensor):
        """x: CUDA tensor [n, dim].  labels_ (int64), core_sample_indices_ (int64, ascending) and neighbour_counts_ (int32)
        stay on the device."""
        _check_params(self.eps, self.min_samples, self.metric)
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise ValueError("DBSCAN.fit_device: expected a CUDA tensor")
        _check_shape(tuple(x.shape))
        labels, core, counts = self._run(self._device_rows(x))
        self.labels_, self.core_sample_indices_, self.neighbour_counts_ = labels.long(), core, counts
        return self

    # ---- internals ---------------------------------------------------------------------------------------
    def _dev(self) -> torch.device:
        d = torch.device(self.device if self.device is not None else "cuda")
        if d.type != "cuda":
            raise RuntimeError("visiondk_b200 runs on CUDA (sm_90a) devices only; there is no CPU path")
        return d

    def _upload(self, X) -> torch.Tensor:
        """Every check runs on the host before anything reaches the device: numpy / memmap chunks are converted to float32
        and checked, then copied into one device buffer."""
        if isinstance(X, torch.Tensor):
            _check_shape(tuple(X.shape))
            if X.is_cuda:
                return self._device_rows(X)
            X = X.detach().float().numpy()
        if not isinstance(X, np.ndarray):
            X = np.asarray(X)
        _check_shape(X.shape)
        n, d = X.shape
        for a in range(0, n, self.chunk_rows):
            _check_rows_host(np.asarray(X[a:a + self.chunk_rows], np.float32), a)
        _lib.load()
        _lib.require_device()
        out = torch.empty((n, d), dtype=torch.float32, device=self._dev())
        for a in range(0, n, self.chunk_rows):
            out[a:a + self.chunk_rows].copy_(torch.from_numpy(np.ascontiguousarray(X[a:a + self.chunk_rows], np.float32)))
        return out

    @staticmethod
    def _device_rows(x: torch.Tensor) -> torch.Tensor:
        """The host checks of _upload for rows already on the device (torch reductions, before any vdk kernel)."""
        x = x.detach().to(torch.float32).contiguous()
        if not bool(torch.isfinite(x).all()):
            raise ValueError("DBSCAN: rows must be finite")
        if bool((x.double().norm(dim=1) < F_NORMALIZE_EPS).any()):
            raise ValueError("DBSCAN: a row has zero norm: cosine distance is undefined for it")
        return x

    def _run(self, x: torch.Tensor):
        lib = _lib.load()
        _lib.require_device()
        dev = x.device
        n, d = x.shape
        threshold = float(neighbour_threshold(float(self.eps)))
        with torch.cuda.device(dev):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)] if self.timing else None
            if ev:
                ev[0].record()
            rows = PreparedRows(x, normalize=True)
            norm_max, err_max = rows.maxima()
            if ev:
                ev[1].record()
            labels = torch.empty((n,), dtype=torch.int32, device=dev)
            counts = torch.empty((n,), dtype=torch.int32, device=dev)
            need = lib.vdk_dbscan_workspace_bytes(n, d, self.boundary_capacity)
            ws = torch.empty((need,), dtype=torch.uint8, device=dev)
            st = _lib.DbscanStats()
            _lib.check(lib.vdk_dbscan(_lib.ptr(rows.x32), _lib.ptr(rows.xh), _lib.ptr(rows.norm), _lib.ptr(rows.err),
                                      _lib.ptr(norm_max), _lib.ptr(err_max), n, d, threshold, int(self.min_samples),
                                      self.boundary_capacity, _lib.ptr(labels), _lib.ptr(counts), C.byref(st), int(self.timing),
                                      ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_dbscan")
        self.threshold_ = threshold
        self.stats_ = {"n_core": st.n_core, "n_clusters": st.n_clusters, "rechecked_pairs": st.rechecked_pairs,
                       "redone_bands": st.redone_bands}
        if self.timing:
            self.stats_["ms"] = {"prepare": ev[0].elapsed_time(ev[1]), "count": st.phase_ms[0], "union": st.phase_ms[1],
                                 "border": st.phase_ms[2], "finalise": st.phase_ms[3]}
            self.stats_["gram_ms"] = {"count": st.gram_ms[0], "union": st.gram_ms[1], "border": st.gram_ms[2]}
        core = torch.nonzero(counts >= int(self.min_samples)).flatten()
        return labels, core, counts
