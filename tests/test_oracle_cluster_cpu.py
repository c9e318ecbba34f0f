"""The DBSCAN oracle against scikit-learn's cosine DBSCAN, its rules on crafted inputs, the host threshold of
visiondk_b200.cluster and the refusals of its DBSCAN class: everything here runs without a GPU."""
import ctypes as C

import numpy as np
import pytest
from sklearn.cluster import DBSCAN as SkDBSCAN
from sklearn.metrics.pairwise import cosine_distances

from oracle import cluster as OC
from oracle.retrieval import l2_normalize
from visiondk_b200 import cluster as VC


def assert_no_pair_near_eps(x, eps, tol=1e-5):
    xn = l2_normalize(x).astype(np.float64)
    d = 1.0 - xn @ xn.T
    np.fill_diagonal(d, 10.0)
    gap = np.abs(d - eps).min()
    assert gap > tol, f"a pair's distance lies {gap:.2e} from eps: library rounding would decide it"


def sk(x, eps, min_samples):
    db = SkDBSCAN(eps=eps, min_samples=min_samples, metric="cosine").fit(x)
    return db.labels_.astype(np.int64), db.core_sample_indices_.astype(np.int64)


def families():
    """(name, rows, eps, min_samples): identity clusters of several spreads plus uniform noise, duplicates, the extremes of
    min_samples and eps, at d = 128 and 512."""
    ident = lambda seed, d, noise=0.5, ids=12, per=20, extra=60: OC.identity_rows(ids, per, extra, d, noise, seed)
    rng = np.random.default_rng(5)
    base = ident(3, 128, 0.5, 8, 6, 30)
    dups = np.concatenate([base, base[rng.choice(base.shape[0], 60)]])[rng.permutation(base.shape[0] + 60)]
    return [
        ("identity_noise_d128", ident(10, 128), 0.4, 5),
        ("identity_noise_d512", ident(11, 512), 0.4, 5),
        ("identity_border_rows", ident(1, 128, 0.8, 10, 12, 30), 0.4, 5),
        ("exact_duplicates", dups, 0.4, 5),
        ("min_samples_1_all_core", ident(12, 128), 0.4, 1),
        ("min_samples_large_all_noise", ident(13, 128), 0.4, 400),
        ("eps_small", ident(14, 128, 0.3), 0.05, 3),
        ("eps_large", ident(15, 128), 1.5, 5),
    ]


@pytest.mark.parametrize("name,x,eps,ms", families(), ids=[f[0] for f in families()])
def test_oracle_equals_sklearn(name, x, eps, ms):
    assert_no_pair_near_eps(x, eps)
    labels, core, _ = OC.dbscan(x, eps, ms)
    ref_labels, ref_core = sk(x, eps, ms)
    np.testing.assert_array_equal(core, ref_core)
    np.testing.assert_array_equal(labels, ref_labels)


def test_families_are_not_degenerate():
    """The sets exercise what they are named for: several clusters, border rows, noise, all-core and all-noise."""
    f = {name: (x, eps, ms) for name, x, eps, ms in families()}
    lab, core, _ = OC.dbscan(*f["identity_noise_d128"])
    assert lab.max() >= 5 and (lab == -1).sum() > 0
    lab, core, _ = OC.dbscan(*f["identity_border_rows"])
    border = np.setdiff1d(np.nonzero(lab >= 0)[0], core)
    assert border.size > 0
    x, eps, ms = f["min_samples_1_all_core"]
    assert OC.dbscan(x, eps, ms)[1].size == x.shape[0]
    x, eps, ms = f["min_samples_large_all_noise"]
    assert (OC.dbscan(x, eps, ms)[0] == -1).all()


def test_prefilter_equals_all_canonical_scores():
    x = OC.identity_rows(10, 12, 40, 128, 0.45, 21)
    for eps in (0.2, 0.4, 0.9):
        a = OC.neighbourhoods(x, eps)
        b = OC.neighbourhoods(x, eps, exact_all=True)
        assert all(np.array_equal(u, v) for u, v in zip(a, b))


def test_distance_comparison_runs_in_float32():
    """A crafted pair whose float32 distance d equals fl32(eps) while eps < d in float64: scikit-learn (NumPy 2 comparing a
    float32 array with a Python float) keeps the pair, so the comparison runs in float32."""
    x = np.array([[1.0, 0.0], [0.6, 0.8]], np.float32)
    d = cosine_distances(x)[0, 1]
    eps = float(d) - 1e-12
    assert np.float32(eps) == d and eps < float(d)
    labels, core = sk(x, eps, 2)
    np.testing.assert_array_equal(core, [0, 1])
    np.testing.assert_array_equal(labels, [0, 0])
    s = np.float32(1.0) - d  # the score whose float32 distance is d
    assert np.float32(1.0) - s == d
    assert OC.neighbour_rule(s, eps) and VC.neighbour_rule(s, eps)
    # the float64 reading would drop it
    assert not float(d) <= eps


def _graph(n, edges):
    neigh = [{i} for i in range(n)]
    for a, b in edges:
        neigh[a].add(b)
        neigh[b].add(a)
    return [np.array(sorted(s), np.int64) for s in neigh]


def test_border_row_takes_the_lowest_numbered_cluster():
    """Row 6 (not core) touches core 5 of cluster 1 and core 2 of cluster 0; its nearest / first-listed core neighbour is in
    cluster 1, yet the DFS reaches it from cluster 0 first."""
    neigh = _graph(8, [(0, 1), (1, 2), (3, 4), (4, 5), (6, 5), (6, 2), (7, 3)])
    is_core = np.array([1, 1, 1, 1, 1, 1, 0, 0], bool)
    ref = OC.dbscan_inner_literal(is_core, neigh)
    np.testing.assert_array_equal(OC.labels_from_components(is_core, neigh), ref)
    assert ref[6] == 0 and ref[5] == 1


def test_two_chains_joined_by_a_high_index_bridge_core():
    """Two chains 0-2-4 and 1-3-5 are one component only through core 9: numbered by the smallest core row, both get 0."""
    neigh = _graph(11, [(0, 2), (2, 4), (1, 3), (3, 5), (4, 9), (5, 9), (10, 5), (10, 7), (7, 8), (6, 8)])
    is_core = np.array([1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 0], bool)
    ref = OC.dbscan_inner_literal(is_core, neigh)
    np.testing.assert_array_equal(OC.labels_from_components(is_core, neigh), ref)
    assert ref[1] == ref[0] == 0 and ref[7] == 1 and ref[10] == 0


def test_component_rule_on_random_graphs():
    rng = np.random.default_rng(0)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        m = int(rng.integers(0, 3 * n))
        edges = [tuple(rng.integers(0, n, 2)) for _ in range(m)]
        neigh = _graph(n, edges)
        is_core = np.array([len(v) >= int(rng.integers(1, 5)) for v in neigh])
        np.testing.assert_array_equal(OC.labels_from_components(is_core, neigh), OC.dbscan_inner_literal(is_core, neigh))


@pytest.mark.parametrize("eps", [0.4, 0.5, 1e-7, 0.3, 1.0, 1.9999999, 2.0, 3.0, 0.123456789])
def test_host_threshold_is_the_least_accepted_float32(eps):
    t = VC.neighbour_threshold(eps)
    assert t.dtype == np.float32 and t == OC.threshold_of(eps)
    around = [t]
    lo = hi = t
    for _ in range(64):
        lo = np.nextafter(lo, np.float32(-np.inf))
        hi = np.nextafter(hi, np.float32(np.inf))
        around += [lo, hi]
    s = np.array(around, np.float32)
    np.testing.assert_array_equal(VC.neighbour_rule(s, eps), s >= t)
    np.testing.assert_array_equal(OC.neighbour_rule(s, eps), s >= t)


def test_threshold_of_eps_two_accepts_everything():
    assert VC.neighbour_threshold(2.0) == -np.inf
    assert VC.neighbour_threshold(1.5) > -1.0


def _x(n=20, d=64, seed=0):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


@pytest.mark.parametrize("kwargs,fit_kwargs,x,match", [
    ({"metric": "euclidean"}, {}, _x(), "metric"),
    ({"metric": "precomputed"}, {}, _x(), "metric"),
    ({}, {"sample_weight": np.ones(20)}, _x(), "sample_weight"),
    ({"eps": 0.0}, {}, _x(), "eps"),
    ({"eps": -0.1}, {}, _x(), "eps"),
    ({"eps": float("nan")}, {}, _x(), "eps"),
    ({"eps": float("inf")}, {}, _x(), "eps"),
    ({"min_samples": 0}, {}, _x(), "min_samples"),
    ({"min_samples": 2.5}, {}, _x(), "min_samples"),
    ({}, {}, _x()[0], "shape"),
    ({}, {}, _x()[None], "shape"),
    ({}, {}, _x(d=100), "dim"),
    ({}, {}, _x(d=32), "dim"),
    ({}, {}, _x(d=576), "dim"),
    ({}, {}, _x(n=0), "0 rows"),
    ({}, {}, np.concatenate([_x(), np.zeros((1, 64), np.float32)]), "zero norm"),
    ({}, {}, np.where(np.arange(64) == 3, np.nan, _x()).astype(np.float32), "not finite"),
], ids=["metric", "precomputed", "sample_weight", "eps0", "eps_neg", "eps_nan", "eps_inf", "min_samples0", "min_samples_float",
        "1d", "3d", "dim100", "dim32", "dim576", "empty", "zero_row", "nan_row"])
def test_every_refusal_is_a_value_error_before_the_device(kwargs, fit_kwargs, x, match):
    with pytest.raises(ValueError, match=match):
        VC.DBSCAN(**kwargs).fit(x, **fit_kwargs)


def test_memmap_rows_are_checked_chunk_by_chunk(tmp_path):
    x = _x(n=300, d=64)
    x[250] = 0
    mm = np.memmap(tmp_path / "store.f16", dtype=np.float16, mode="w+", shape=x.shape)
    mm[:] = x
    mm.flush()
    view = np.memmap(tmp_path / "store.f16", dtype=np.float16, mode="r").reshape(-1, 64)
    db = VC.DBSCAN()
    db.chunk_rows = 64
    with pytest.raises(ValueError, match="row 250 has zero norm"):
        db.fit(view)


def test_dbscan_symbols_exported_and_validated(lib):
    from visiondk_b200 import _lib
    assert hasattr(lib, "vdk_dbscan") and hasattr(lib, "vdk_dbscan_workspace_bytes")
    assert C.sizeof(_lib.DbscanStats) == 64
    assert lib.vdk_dbscan_workspace_bytes(1000, 512, 1 << 20) >= 1000 * 512 * 2 + (1 << 20) * 8
    assert lib.vdk_dbscan_workspace_bytes(1000, 100, 1 << 20) == 0
    assert lib.vdk_dbscan_workspace_bytes(1000, 512, 100) == 0
    st = _lib.DbscanStats()
    args = [1, 1, 1, 1, 1, 1, 1000, 512, 0.6, 5, 1 << 20, 1, 1, C.byref(st), 0, 0, 0, 0]
    for i, v, msg in [(0, 0, "null row"), (11, 0, "null output"), (7, 100, "multiple of 64"), (9, 0, "min_samples"),
                      (6, 0, "n must be"), (10, 10, "boundary_capacity"), (8, float("nan"), "NaN"), (15, 0, "workspace")]:
        a = list(args)
        a[i] = v
        assert lib.vdk_dbscan(*a) == _lib.VDK_ERR_INVALID
        assert msg in _lib.last_error(), (msg, _lib.last_error())
