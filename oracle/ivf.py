"""Oracle for the IVF-Flat and IVF-PQ indexes (TEST INFRASTRUCTURE — see oracle/__init__.py).

Reference behaviour: engine/cbir/evaluation.py:110,155 and cbir_eval.py:40,82 pass `index_factory` straight to
`faiss.index_factory(dim, index_factory, METRIC_INNER_PRODUCT)`.  faiss is not vendored (see oracle/retrieval.py), and its
RNG and float order cannot be reproduced, so these definitions are ours; defaults follow faiss' documented ones
(25 Lloyd iterations, at most 256 training rows per centroid, nprobe 1, 8-bit PQ codes by residual, the empty-cluster split).

  training sample   the first min(n, 256 * k) rows of torch.randperm(n, Generator().manual_seed(1234)), taken in ascending
                    row order; the first k rows of the permutation are the initial centroids
  assignment        coarse: the canonical argmax (oracle/retrieval.py canonical score, ties -> lowest centroid);
                    PQ: argmin_j of the sequential fp64 sum over t of (r_t - cw_jt)^2 (no fused multiply-add), ties -> lowest j
  update            per centroid the fp64 sum of its members in ascending row order, then fp32(sum / count); each empty
                    centroid (ascending) copies the then-largest one (lowest index on ties), the copies are scaled by 1 + 1/1024
                    and 1 - 1/1024 on even dimensions and the other way on odd ones, and the count is halved between them;
                    coarse centroids are then L2-normalised (l2_normalize = the rows_prepare normalisation)
  PQ                residual r = fl32(x - c); codebooks [M][256][d/M] trained by L2 k-means on residual sub-vectors
  LUT               lut[m][j] = fp32(sequential fp64 sum over t of q[m*dsub + t] * cw[m][j][t])
  scores            IVF-Flat: canonical score of the row; IVF-PQ: s = coarse score; s = fl32(s + lut[m][code_m]), m = 0..M-1
  search            the nprobe best lists (canonical coarse scores, score desc, id asc); the exact (score desc, id asc) top-k
                    of the rows of those lists, padded with (-FLT_MAX, -1)
"""
from __future__ import annotations

import numpy as np
import torch

from .retrieval import FLT_LOWEST, canonical_scores, l2_normalize, topk_from_scores

NITER = 25
SEED = 1234
MAX_ROWS_PER_CENTROID = 256
PQ_K = 256
SPLIT_EPS = np.float32(1.0 / 1024.0)


def permutation(n: int) -> np.ndarray:
    return torch.randperm(n, generator=torch.Generator().manual_seed(SEED)).numpy()


def training_sample(n: int, k: int):
    """(ascending row ids of the training sample, row ids of the k initial centroids)."""
    perm = permutation(n)
    return np.sort(perm[:min(n, MAX_ROWS_PER_CENTROID * k)]), perm[:k]


def split_empty(c: np.ndarray, cnt: np.ndarray) -> None:
    """The empty-cluster split, in place on centroids c [k, dim] and counts cnt [k]."""
    even = (np.arange(c.shape[1]) % 2) == 0
    up, down = np.float32(1) + SPLIT_EPS, np.float32(1) - SPLIT_EPS
    for ci in range(c.shape[0]):
        if cnt[ci] == 0:
            cj = int(np.argmax(cnt))
            v = c[cj].copy()
            c[ci] = np.where(even, v * up, v * down)
            c[cj] = np.where(even, v * down, v * up)
            cnt[ci] = cnt[cj] // 2
            cnt[cj] -= cnt[ci]


def kmeans_update(x: np.ndarray, assign: np.ndarray, c: np.ndarray):
    """One Lloyd update (vdk_kmeans_update): -> (new centroids, counts after the split)."""
    k = c.shape[0]
    c = c.copy()
    cnt = np.bincount(assign, minlength=k).astype(np.int64)
    order = np.argsort(assign, kind="stable")
    offs = np.concatenate([[0], np.cumsum(cnt)])
    x64 = x.astype(np.float64)
    for g in range(k):
        lo, hi = offs[g], offs[g + 1]
        if hi > lo:
            s = np.add.accumulate(x64[order[lo:hi]], axis=0)[-1]  # sequential, ascending row order
            c[g] = (s / np.float64(hi - lo)).astype(np.float32)
    split_empty(c, cnt)
    return c, cnt


def coarse_assign(x: np.ndarray, c: np.ndarray) -> np.ndarray:
    return np.argmax(canonical_scores(x, c), axis=1)


def pq_assign(r: np.ndarray, cb: np.ndarray) -> np.ndarray:
    """Residuals r [n, d], codebooks [M, 256, dsub] -> codes uint8 [n, M]."""
    n = r.shape[0]
    M, kc, dsub = cb.shape
    codes = np.empty((n, M), np.uint8)
    cb64 = cb.astype(np.float64)
    for m in range(M):
        rs = r[:, m * dsub:(m + 1) * dsub].astype(np.float64)
        acc = np.zeros((n, kc), np.float64)
        for t in range(dsub):
            df = rs[:, None, t] - cb64[m][None, :, t]
            acc = acc + df * df
        codes[:, m] = np.argmin(acc, axis=1)
    return codes


def residuals(x: np.ndarray, c: np.ndarray, lists: np.ndarray) -> np.ndarray:
    return (np.asarray(x, np.float32) - c[lists]).astype(np.float32)


def train_coarse(x: np.ndarray, nlist: int, niter: int = NITER) -> np.ndarray:
    x = np.asarray(x, np.float32)
    ids, init = training_sample(x.shape[0], nlist)
    xs = x[ids]
    c = x[init].copy()
    for _ in range(niter):
        c, _ = kmeans_update(xs, coarse_assign(xs, c), c)
        c = l2_normalize(c)
    return c


def train_pq(x: np.ndarray, centroids: np.ndarray, M: int, niter: int = NITER) -> np.ndarray:
    x = np.asarray(x, np.float32)
    d = x.shape[1]
    dsub = d // M
    ids, init = training_sample(x.shape[0], PQ_K)
    r = residuals(x[ids], centroids, coarse_assign(x[ids], centroids))
    r0 = r[np.searchsorted(ids, init)]
    cb = np.ascontiguousarray(r0.reshape(PQ_K, M, dsub).transpose(1, 0, 2))
    for _ in range(niter):
        codes = pq_assign(r, cb)
        for m in range(M):
            cb[m], _ = kmeans_update(r[:, m * dsub:(m + 1) * dsub], codes[:, m], cb[m])
    return cb


def pq_lut(q: np.ndarray, cb: np.ndarray) -> np.ndarray:
    """-> lut float32 [nq, M, 256]."""
    q = np.asarray(q, np.float32)
    M, _, dsub = cb.shape
    out = np.empty((q.shape[0], M, PQ_K), np.float32)
    cb64 = cb.astype(np.float64)
    for m in range(M):
        acc = np.zeros((q.shape[0], PQ_K), np.float64)
        for t in range(dsub):
            acc = acc + q[:, m * dsub + t, None].astype(np.float64) * cb64[m][None, :, t]
        out[:, m] = acc.astype(np.float32)
    return out


def adc_scores(coarse: np.float32, lut_q: np.ndarray, codes: np.ndarray) -> np.ndarray:
    """lut_q [M, 256], codes [n, M] -> float32 [n]: s = coarse; s = fl32(s + lut[m][code_m])."""
    s = np.full(codes.shape[0], coarse, np.float32)
    for m in range(codes.shape[1]):
        s = (s + lut_q[m][codes[:, m]]).astype(np.float32)
    return s


def search(q: np.ndarray, centroids: np.ndarray, lists: np.ndarray, k: int, nprobe: int, rows: np.ndarray = None,
           codes: np.ndarray = None, codebooks: np.ndarray = None, ids: np.ndarray = None):
    """IVF search.  lists [n]: the list of every stored row; rows [n, d] (IVF-Flat) or codes [n, M] + codebooks (IVF-PQ);
    ids [n]: the stored rows' ids (default 0..n-1).  -> (scores float32 [nq, k], ids int64 [nq, k])."""
    q = np.asarray(q, np.float32)
    nq = q.shape[0]
    ids = np.arange(lists.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    nprobe = min(nprobe, centroids.shape[0])
    ps, pl = topk_from_scores(canonical_scores(q, centroids), nprobe)
    lut = pq_lut(q, codebooks) if codes is not None else None
    out_s = np.full((nq, k), FLT_LOWEST, np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    for r in range(nq):
        cs, ci = [], []
        for p in range(nprobe):
            sel = np.nonzero(lists == pl[r, p])[0]
            if sel.size == 0:
                continue
            if codes is None:
                cs.append(canonical_scores(q[r:r + 1], rows[sel])[0])
            else:
                cs.append(adc_scores(ps[r, p], lut[r], codes[sel]))
            ci.append(ids[sel])
        if not cs:
            continue
        s, i = np.concatenate(cs), np.concatenate(ci)
        order = np.lexsort((i, -s.astype(np.float64)))[:k]
        out_s[r, :order.size] = s[order]
        out_i[r, :order.size] = i[order]
    return out_s, out_i


def build(x: np.ndarray, nlist: int, M: int = None):
    """Train on x and add x: -> dict(centroids, lists, codebooks, codes) of the oracle index."""
    x = np.asarray(x, np.float32)
    c = train_coarse(x, nlist)
    lists = coarse_assign(x, c)
    out = {"centroids": c, "lists": lists, "codebooks": None, "codes": None}
    if M is not None:
        cb = train_pq(x, c, M)
        out["codebooks"], out["codes"] = cb, pq_assign(residuals(x, c, lists), cb)
    return out
