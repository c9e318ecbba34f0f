"""Oracle for DBSCAN with metric="cosine" (TEST INFRASTRUCTURE — see oracle/__init__.py).

Reference behaviour restated here: tools/clustering.py runs
    DBSCAN(eps=0.4, min_samples=5, metric="cosine", n_jobs=16).fit(X)
with scikit-learn (1.9.0 installed; its cosine neighbours are brute force).  scikit-learn computes float32 cosine distances
d = 1 - s (clipped to [0, 2]) for float32 input and keeps j in i's neighbourhood iff d <= eps, a comparison NumPy 2 runs in
float32 (the Python float eps becomes fl32(eps); tests/test_oracle_cluster_cpu.py pins this with a crafted pair).  Its score
s is a float32 BLAS dot, whose summation order is unspecified, so parity needs a canonical score; ours is the one of
oracle/retrieval.py on rows normalised by l2_normalize (F.normalize):

  neighbour(i, j)  iff  i == j  or  clip(fl32(1 - s_ij), 0, 2) <= fl32(eps)
  core(i)          iff  #neighbours(i) (self included) >= min_samples
  labels           clusters = connected components of the core-core neighbour graph, numbered 0, 1, ... by ascending
                   smallest core row; a non-core row with a core neighbour takes the smallest label among them (the
                   order in which dbscan_inner's depth-first search reaches it); every other row is -1.

`dbscan_inner_literal` transcribes sklearn/cluster/_dbscan_inner.pyx so that the component formulation can be checked
against the DFS.
"""
from __future__ import annotations

import numpy as np

from .retrieval import canonical_dot, canonical_scores, l2_normalize

# |float64 BLAS dot - exact dot| for unit rows of <= 512 dims is below 1e-13; pairs whose BLAS score is farther than this from
# the threshold are decided by it, the others by the canonical score
_PREFILTER_MARGIN = 1e-6


def neighbour_rule(s, eps: float) -> np.ndarray:
    s = np.asarray(s, np.float32)
    d = np.clip(np.float32(1.0) - s, np.float32(0.0), np.float32(2.0))
    return d <= np.float32(eps)


def threshold_of(eps: float) -> np.float32:
    """Least float32 s accepted by neighbour_rule (the rule is monotone in s): bisection over float64 x of the rule at fl32(x),
    until the two ends round to adjacent float32 values."""
    inf = np.float32(np.inf)
    if neighbour_rule(-inf, eps):  # fl32(eps) >= 2: the clipped distance always passes
        return -inf
    lo, hi = -2.0, 1.0  # rule(fl32(-2)) fails when fl32(eps) < 2; rule(1) passes for eps > 0
    while np.nextafter(np.float32(lo), inf) != np.float32(hi):
        mid = 0.5 * (lo + hi)
        if neighbour_rule(np.float32(mid), eps):
            hi = mid
        else:
            lo = mid
    return np.float32(hi)


def neighbourhoods(X: np.ndarray, eps: float, block: int = 256, exact_all: bool = False):
    """Neighbour lists (ascending int64 arrays, self included) of every row under the canonical rule.  exact_all computes
    every canonical score with canonical_scores; otherwise a float64 BLAS score decides the pairs far from the threshold
    and canonical_dot the rest (identical result, see _PREFILTER_MARGIN)."""
    xn = l2_normalize(np.asarray(X, np.float32))
    n = xn.shape[0]
    t = threshold_of(eps)
    x64 = xn.astype(np.float64)
    out = []
    for a in range(0, n, block):
        b = min(n, a + block)
        if exact_all:
            nb = neighbour_rule(canonical_scores(xn[a:b], xn), eps)
        else:
            g = x64[a:b] @ x64.T
            nb = g >= float(t) + _PREFILTER_MARGIN
            near = np.nonzero(np.abs(g - float(t)) < _PREFILTER_MARGIN)
            if near[0].size:
                s = canonical_dot(xn[a + near[0]], xn[near[1]])
                nb[near] = neighbour_rule(s, eps)
        nb[np.arange(b - a), np.arange(a, b)] = True
        out.extend(np.nonzero(r)[0].astype(np.int64) for r in nb)
    return out


def labels_from_components(is_core: np.ndarray, neigh) -> np.ndarray:
    """The component formulation: union-find over core-core edges (larger root under the smaller, so a root is its
    component's smallest core row), roots ranked in ascending order, border rows take their smallest core neighbour label."""
    n = is_core.shape[0]
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for i in np.nonzero(is_core)[0]:
        for j in neigh[i]:
            if j > i and is_core[j]:
                a, b = find(i), find(j)
                if a != b:
                    parent[max(a, b)] = min(a, b)
    labels = np.full(n, -1, np.int64)
    roots = {}
    for i in np.nonzero(is_core)[0]:
        r = find(i)
        if r not in roots:
            roots[r] = len(roots)  # core rows ascend, so roots are met in ascending order
        labels[i] = roots[r]
    for i in np.nonzero(~is_core)[0]:
        c = [labels[j] for j in neigh[i] if is_core[j]]
        if c:
            labels[i] = min(c)
    return labels


def dbscan_inner_literal(is_core: np.ndarray, neigh) -> np.ndarray:
    """sklearn/cluster/_dbscan_inner.pyx, line for line."""
    labels = np.full(is_core.shape[0], -1, np.int64)
    label_num = 0
    stack = []
    for i in range(labels.shape[0]):
        if labels[i] != -1 or not is_core[i]:
            continue
        while True:
            if labels[i] == -1:
                labels[i] = label_num
                if is_core[i]:
                    neighb = neigh[i]
                    for i in range(neighb.shape[0]):
                        v = neighb[i]
                        if labels[v] == -1:
                            stack.append(v)
            if len(stack) == 0:
                break
            i = stack.pop()
        label_num += 1
    return labels


def dbscan(X: np.ndarray, eps: float, min_samples: int, exact_all: bool = False):
    """-> (labels int64 [n], core_sample_indices int64 ascending, neighbour counts int64 [n])."""
    neigh = neighbourhoods(X, eps, exact_all=exact_all)
    counts = np.array([len(v) for v in neigh], np.int64)
    is_core = counts >= min_samples
    return labels_from_components(is_core, neigh), np.nonzero(is_core)[0].astype(np.int64), counts


def identity_rows(n_ids: int, per_id: int, n_noise: int, dim: int, noise: float, seed: int) -> np.ndarray:
    """Seeded identity clusters (centre + noise * N(0, I), not normalised) followed by uniform-direction noise rows."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_ids, dim)).astype(np.float32)
    x = np.repeat(centres, per_id, axis=0) + noise * rng.standard_normal((n_ids * per_id, dim)).astype(np.float32)
    x = np.concatenate([x, rng.standard_normal((n_noise, dim)).astype(np.float32)])
    return x[rng.permutation(x.shape[0])]
