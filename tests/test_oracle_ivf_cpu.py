"""CPU checks of the IVF indexes: the index_factory grammar and its refusals (raised before any kernel), and the numpy oracle
(oracle/ivf.py) the GPU tests compare against bit for bit: k-means descent, the empty-cluster split, and the recall of both
index types on a seeded identity-structured gallery."""
import numpy as np
import pytest

from oracle import ivf as O
from oracle import retrieval as R
from visiondk_b200.ivf import parse_index_factory


@pytest.mark.parametrize("spec,d,expect", [
    ("Flat", 512, None), ("IVF4096,Flat", 512, (4096, None)), ("IVF4096,PQ64", 512, (4096, 64)),
    ("IVF1024,PQ64x8", 512, (1024, 64)), ("IVF1,PQ128", 128, (1, 128)),
])
def test_factory_accepts(spec, d, expect):
    assert parse_index_factory(spec, d) == expect


@pytest.mark.parametrize("spec,d", [
    ("HNSW32", 512), ("IVF64,SQ8", 512), ("OPQ16,IVF64,PQ16", 512), ("PQ64", 512), ("IVF64,PQ16x4", 512), ("IVF64,PQ48", 512),
    ("IVF64,PQ256", 512), ("IVF0,Flat", 512), ("flat", 512), ("IVF64,Flat,RFlat", 512), ("IVF64, Flat", 512), (" Flat", 512),
])
def test_factory_refuses(spec, d):
    with pytest.raises(ValueError, match="IVF<nlist>,PQ<M>x8"):
        parse_index_factory(spec, d)


def test_cbir_index_refuses_before_running_anything():
    from visiondk_b200.cbir import index

    class Boom:
        def extract_cbir_device(self, *a, **k):
            raise AssertionError("extraction ran before the factory string was checked")

    with pytest.raises(ValueError, match="HNSW32"):
        index(Boom(), None, "cuda", index_factory="HNSW32")
    with pytest.raises(ValueError, match="not sharded"):
        index(Boom(), None, "cuda", index_factory="IVF64,Flat", memmap_load_embedding=True, shard=(0, 2))


def _objective(x, c, a):
    return float(((x.astype(np.float64) - c[a].astype(np.float64)) ** 2).sum())


def test_kmeans_l2_objective_does_not_increase():
    """Plain (non-spherical) Lloyd with the oracle's update and the PQ assignment rule: the L2 objective never increases."""
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((3000, 8)) + 3 * rng.integers(0, 4, (3000, 1))).astype(np.float32)
    ids, init = O.training_sample(x.shape[0], O.PQ_K)
    xs, c = x[ids], x[init].copy()
    prev = np.inf
    for _ in range(8):
        a = O.pq_assign(xs, c[None])[:, 0].astype(np.int64)
        obj = _objective(xs, c, a)
        assert obj <= prev * (1 + 1e-6), (obj, prev)
        prev = obj
        c, _ = O.kmeans_update(xs, a, c)


def test_empty_cluster_split_with_duplicate_rows():
    """Duplicate rows leave centroids empty: each empty centroid copies the then-largest cluster, the copies move apart by
    1 +- 1/1024 on alternate dimensions, and the count is halved."""
    x = np.repeat(np.array([[1.0, 2.0, 3.0, 4.0], [-1.0, 0.5, 0.25, 8.0]], np.float32), [10, 3], axis=0)
    c0 = np.stack([x[0], x[0], x[10], x[0]])  # centroids 1 and 3 duplicate centroid 0: only the lowest index wins the argmin
    a = O.pq_assign(x, c0[None])[:, 0].astype(np.int64)
    assert list(np.bincount(a, minlength=4)) == [10, 0, 3, 0]
    c, cnt = O.kmeans_update(x, a, c0)
    up, down = np.float32(1) + O.SPLIT_EPS, np.float32(1) - O.SPLIT_EPS
    v = x[0]
    # centroid 1 splits cluster 0 (10 -> 5 + 5); centroid 3 then splits the largest, cluster 0 again (lowest index on ties)
    c0_after_first = np.where(np.arange(4) % 2 == 0, v * down, v * up).astype(np.float32)
    assert np.array_equal(c[1], np.where(np.arange(4) % 2 == 0, v * up, v * down).astype(np.float32))
    assert np.array_equal(c[3], np.where(np.arange(4) % 2 == 0, c0_after_first * up, c0_after_first * down).astype(np.float32))
    assert np.array_equal(c[0], np.where(np.arange(4) % 2 == 0, c0_after_first * down, c0_after_first * up).astype(np.float32))
    assert np.array_equal(c[2], x[10]) and list(cnt) == [3, 5, 3, 2]


@pytest.fixture(scope="module")
def gallery_state():
    g, q, _ = R.synthetic_gallery(400, 20, dim=64, seed=3, noise=1.0)
    q = q[:100]
    return g, q, O.build(g, 32, 8), R.flat_ip_search(q, g, 10)


# recall@10 against the exact Flat search, fixed by this oracle run (8000 x 64-d, nlist 32, PQ8)
RECALL_FLOORS = {("flat", 1): 0.566, ("flat", 8): 0.905, ("flat", 32): 1.0, ("pq", 1): 0.431, ("pq", 8): 0.605, ("pq", 32): 0.621}


@pytest.mark.parametrize("kind,nprobe", sorted(RECALL_FLOORS))
def test_recall_floors(gallery_state, kind, nprobe):
    g, q, st, (fs, fi) = gallery_state
    if kind == "flat":
        s, i = O.search(q, st["centroids"], st["lists"], 10, nprobe, rows=g)
    else:
        s, i = O.search(q, st["centroids"], st["lists"], 10, nprobe, codes=st["codes"], codebooks=st["codebooks"])
    recall = np.mean([len(set(i[r]) & set(fi[r])) / 10 for r in range(q.shape[0])])
    assert recall >= RECALL_FLOORS[(kind, nprobe)] - 1e-9, recall
    if kind == "flat" and nprobe == 32:  # every list probed: the exact Flat result, bit for bit
        assert np.array_equal(i, fi) and np.array_equal(s.view(np.uint32), fs.view(np.uint32))
