"""DBSCAN on the device (vdk_dbscan through visiondk_b200.cluster.DBSCAN) against the oracle, label for label: the CPU-test
families at a few thousand rows, scikit-learn itself on one seeded set, boundary floods that overflow the boundary buffer,
degenerate sets, determinism, property checks at 262 144 rows, the tensor-core error bound, and the clustering tool."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cluster as OC
from oracle import retrieval as R
from visiondk_b200 import _lib
from visiondk_b200.cluster import DBSCAN, neighbour_threshold
from visiondk_b200.retrieval import PreparedRows, exact_pair_scores

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ident(seed, d, noise, ids, per, extra):
    return OC.identity_rows(ids, per, extra, d, noise, seed)


def gpu_families():
    rng = np.random.default_rng(5)
    base = ident(3, 128, 0.5, 150, 12, 600)
    dups = np.concatenate([base, base[rng.choice(base.shape[0], 800)]])[rng.permutation(base.shape[0] + 800)]
    return [
        ("identity_noise_d128", ident(20, 128, 0.5, 200, 16, 896), 0.4, 5),
        ("identity_noise_d512", ident(21, 512, 0.5, 200, 16, 896), 0.4, 5),
        ("identity_border_rows", ident(22, 128, 0.8, 250, 12, 600), 0.4, 5),
        ("identity_d256_min_samples_3", ident(23, 256, 0.7, 300, 8, 500), 0.35, 3),
        ("exact_duplicates", dups, 0.4, 5),
        ("min_samples_1_all_core", ident(24, 128, 0.5, 200, 16, 896), 0.4, 1),
        ("min_samples_large_all_noise", ident(25, 128, 0.5, 200, 16, 896), 0.4, 5000),
        ("eps_small", ident(26, 128, 0.3, 200, 16, 896), 0.05, 3),
        ("eps_large", ident(27, 64, 0.5, 50, 20, 300), 1.5, 5),
    ]


def check_equal(db, x, eps, ms):
    labels, core, counts = OC.dbscan(x, eps, ms)
    np.testing.assert_array_equal(db.neighbour_counts_, counts)
    np.testing.assert_array_equal(db.core_sample_indices_, core)
    np.testing.assert_array_equal(db.labels_, labels)
    assert db.labels_.dtype == np.int64 and db.core_sample_indices_.dtype == np.int64
    return labels


@pytest.mark.parametrize("name,x,eps,ms", gpu_families(), ids=[f[0] for f in gpu_families()])
def test_labels_equal_the_oracle(lib, name, x, eps, ms):
    db = DBSCAN(eps=eps, min_samples=ms, metric="cosine", n_jobs=16).fit(x)
    check_equal(db, x, eps, ms)
    assert db.stats_["n_core"] == db.core_sample_indices_.size
    assert db.stats_["n_clusters"] == int(db.labels_.max()) + 1


def test_fit_predict_and_memmap_store_equal_the_oracle(lib, tmp_path):
    x = ident(30, 512, 0.6, 150, 16, 500).astype(np.float16)
    mm = np.memmap(tmp_path / "emb.f16", dtype=np.float16, mode="w+", shape=x.shape)
    mm[:] = x
    mm.flush()
    store = np.memmap(tmp_path / "emb.f16", dtype=np.float16, mode="r").reshape(-1, 512)
    db = DBSCAN(eps=0.4, min_samples=5)
    db.chunk_rows = 1000  # several chunks
    labels = check_equal(db.fit(store), x.astype(np.float32), 0.4, 5)
    np.testing.assert_array_equal(DBSCAN(eps=0.4, min_samples=5).fit_predict(torch.from_numpy(x)), labels)


def test_scikit_learn_parity(lib):
    from sklearn.cluster import DBSCAN as SkDBSCAN
    x = ident(40, 512, 0.55, 180, 14, 500)
    xn = R.l2_normalize(x).astype(np.float64)
    d = 1.0 - xn @ xn.T
    np.fill_diagonal(d, 10.0)
    assert np.abs(d - 0.4).min() > 1e-5, "a pair sits within 1e-5 of eps: library rounding would decide it"
    ref = SkDBSCAN(eps=0.4, min_samples=5, metric="cosine", n_jobs=16).fit(x)
    db = DBSCAN(eps=0.4, min_samples=5, metric="cosine", n_jobs=16).fit(x)
    np.testing.assert_array_equal(db.core_sample_indices_, ref.core_sample_indices_)
    np.testing.assert_array_equal(db.labels_, ref.labels_)
    assert len(set(ref.labels_)) > 100


def flood_rows(m, n_noise, dim, seed):
    """Two groups of m duplicated rows u and v, and eps such that the threshold is exactly the canonical score of (u, v):
    all m^2 cross pairs sit at the threshold, inside the tensor-core error band."""
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(dim).astype(np.float32)
    w = rng.standard_normal(dim).astype(np.float32)
    w -= (w @ u) / (u @ u) * u
    v = (0.6 * u / np.linalg.norm(u) + 0.8 * w / np.linalg.norm(w)).astype(np.float32)
    un, vn = R.l2_normalize(np.stack([u, v]))
    s = R.canonical_dot(un[None], vn[None])[0]
    eps = float(np.float32(1.0) - s)
    x = np.concatenate([np.repeat(u[None], m, 0), np.repeat(v[None], m, 0), rng.standard_normal((n_noise, dim)).astype(np.float32)])
    x = x[rng.permutation(x.shape[0])]
    assert neighbour_threshold(eps) == s
    return x, eps


@pytest.mark.parametrize("dim", [128, 512])
def test_boundary_flood_overflows_and_is_redone(lib, dim):
    x, eps = flood_rows(600, 300, dim, seed=dim)
    db = DBSCAN(eps=eps, min_samples=5)
    db.boundary_capacity = 128 * 256  # one tile: 360 000 cross pairs overflow it, and so does every 128-row band
    labels = check_equal(db.fit(x), x, eps, 5)
    assert db.stats_["redone_bands"] > 0
    assert db.stats_["rechecked_pairs"] >= 600 * 600
    assert np.unique(labels[labels >= 0]).size == 1 and (labels >= 0).sum() >= 1200
    # the default buffer holds the flood: nothing redone, same answer
    db2 = DBSCAN(eps=eps, min_samples=5).fit(x)
    assert db2.stats_["redone_bands"] == 0
    np.testing.assert_array_equal(db2.labels_, labels)


def test_all_rows_identical_form_one_cluster(lib):
    x = np.repeat(np.random.default_rng(1).standard_normal((1, 512)).astype(np.float32), 3000, 0)
    db = DBSCAN(eps=1e-6, min_samples=5).fit(x)
    assert (db.labels_ == 0).all() and db.core_sample_indices_.size == 3000 and (db.neighbour_counts_ == 3000).all()


def test_mutually_orthogonal_rows_are_all_noise(lib):
    x = (np.eye(512, dtype=np.float32) * np.arange(1, 513, dtype=np.float32)[:, None])
    db = DBSCAN(eps=0.5, min_samples=2).fit(x)
    assert (db.labels_ == -1).all() and db.core_sample_indices_.size == 0 and (db.neighbour_counts_ == 1).all()
    db = DBSCAN(eps=0.5, min_samples=1).fit(x)
    np.testing.assert_array_equal(db.labels_, np.arange(512))


def test_two_runs_are_identical(lib):
    x = ident(50, 256, 0.8, 400, 10, 800)
    a = DBSCAN(eps=0.4, min_samples=4).fit(x)
    b = DBSCAN(eps=0.4, min_samples=4).fit(x)
    np.testing.assert_array_equal(a.labels_, b.labels_)
    np.testing.assert_array_equal(a.neighbour_counts_, b.neighbour_counts_)


def chain_rows(n_arcs, per_arc, dim, step):
    """n_arcs arcs of per_arc points, each arc in its own coordinate plane, consecutive points `step` radians apart.  Row
    indices run DOWN each arc and interleave the arcs, so the core-core graph is n_arcs long chains that the union pass
    links end to end (deep trees for the read-only root walk of the finalisation)."""
    x = np.zeros((n_arcs * per_arc, dim), np.float32)
    for a in range(n_arcs):
        k = np.arange(per_arc)
        idx = (per_arc - 1 - k) * n_arcs + a
        x[idx, 2 * a] = np.cos(k * step)
        x[idx, 2 * a + 1] = np.sin(k * step)
    return x


def test_long_chains_of_core_rows(lib):
    step = 0.003
    eps = float(1.0 - np.cos(2.5 * step))  # neighbours: the two points on either side; interior rows have 5, ends 3 and 4
    x = chain_rows(16, 1000, 64, step)
    db = DBSCAN(eps=eps, min_samples=5).fit(x)
    labels = check_equal(db, x, eps, 5)
    assert db.stats_["n_clusters"] == 16 and (labels >= 0).all()
    assert db.stats_["rechecked_pairs"] > 16 * 1000  # the neighbour pairs sit inside the tensor-core error band
    b = DBSCAN(eps=eps, min_samples=5).fit(x)
    np.testing.assert_array_equal(b.labels_, labels)


def device_identity_rows(n, dim, per, seed, noise=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn((n + per - 1) // per, dim, device="cuda", generator=g)
    x = centres.repeat_interleave(per, 0)[:n] + noise * torch.randn(n, dim, device="cuda", generator=g)
    return x[torch.randperm(n, device="cuda", generator=g)]


def test_properties_at_262144_rows(lib):
    n, dim, eps, ms = 262144, 512, 0.4, 5
    # identity groups of 8 with a noise level where groups straddle the threshold: core, border and noise rows all occur
    x = device_identity_rows(n, dim, 8, seed=3, noise=0.8)
    db = DBSCAN(eps=eps, min_samples=ms).fit_device(x)
    labels, counts = db.labels_, db.neighbour_counts_
    core = counts >= ms
    t = float(neighbour_threshold(eps))
    xn = PreparedRows(x, True).x32
    n_core, n_border = int(core.sum()), int(((labels >= 0) & ~core).sum())
    assert n_core > 1000 and n_border > 100 and int((labels == -1).sum()) > 100, (n_core, n_border)
    g = torch.Generator(device="cuda").manual_seed(9)
    sample = torch.cat([torch.nonzero(core).flatten()[torch.randperm(n_core, device="cuda", generator=g)[:24]],
                        torch.nonzero(~core).flatten()[torch.randperm(n - n_core, device="cuda", generator=g)[:40]]])
    cols = torch.arange(n, device="cuda")
    for i in sample.tolist():
        s = exact_pair_scores(xn, xn, torch.full((n,), i, device="cuda", dtype=torch.int64), cols)
        nb = (s >= t) | (cols == i)
        assert int(nb.sum()) == int(counts[i]), f"row {i}: neighbour count"
        cn = nb & core
        if core[i]:
            assert bool((labels[cn] == labels[i]).all()), f"core row {i}: a core neighbour has another label"
        elif bool(cn.any()):
            assert int(labels[i]) == int(labels[cn].min()), f"border row {i}: not the smallest core-neighbour label"
        else:
            assert int(labels[i]) == -1
    # clusters numbered by ascending smallest core row
    nl = int(labels.max()) + 1
    first = torch.full((nl,), n, dtype=torch.int64, device="cuda")
    first.scatter_reduce_(0, labels[core].long(), cols[core], reduce="amin")
    assert bool((first[1:] > first[:-1]).all()) and int(first[-1]) < n
    assert db.stats_["n_clusters"] == nl


def test_tensor_core_error_within_the_bound_used(lib):
    """The epilogue decides a pair from the fp16 tensor-core score a when |a - T| > e_i; measure |a - canonical| on
    identity-structured rows against e_i (the per-row bound bounds_kernel computes).  gram_kernel's scores never leave its
    registers, so vdk_gemm_tn stands in for it here: the same fp16 rows of vdk_rows_prepare, fp16 wgmma with fp32
    accumulation over the same 512-long K.  gram_kernel's own decisions are checked against the canonical scores by every
    oracle comparison in this file, most sharply by the chains below, whose neighbour pairs all fall inside the band."""
    x = device_identity_rows(8192, 512, 16, seed=4)
    rows = PreparedRows(x, True)
    gn, ge = rows.maxima()
    nq = 256
    approx = torch.empty((nq, 8192), dtype=torch.float32, device="cuda")
    _lib.check(lib.vdk_gemm_tn(rows.xh.data_ptr(), rows.xh.data_ptr(), approx.data_ptr(), nq, 8192, 512, 512, 512, 8192,
                               _lib.DTYPE_FP16, _lib.DTYPE_FP32, _lib.EPI_NONE, 0, 0, 0, 0, _lib.stream_ptr()), "vdk_gemm_tn")
    qi = torch.arange(nq, device="cuda").repeat_interleave(8192)
    gi = torch.arange(8192, device="cuda").repeat(nq)
    exact = exact_pair_scores(rows.x32, rows.x32, qi, gi).view(nq, 8192).double()
    err = (approx.double() - exact).abs().max(dim=1).values
    qn = rows.norm[:nq] + rows.err[:nq]
    bound = (rows.err[:nq] * gn + qn * ge + 2.0 ** -13 * qn * (gn + ge)) * 1.0001
    assert bool((err <= bound.double()).all()), (err.max().item(), bound.min().item())
    assert err.max().item() > 0


def test_cluster_tool_copies_the_clusters_scikit_learn_finds(lib, tmp_path):
    from sklearn.cluster import DBSCAN as SkDBSCAN
    x = ident(60, 128, 0.5, 30, 8, 40)
    feats, images, out = tmp_path / "features", tmp_path / "images", tmp_path / "cluster"
    feats.mkdir()
    images.mkdir()
    names = [f"img{i:04d}" for i in range(x.shape[0])]
    for name, row in zip(names, x):
        np.save(feats / f"{name}.npy", row)
        (images / f"{name}.jpg").write_bytes(name.encode())
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "cluster_embeddings.py"), "--features", str(feats), "--images",
                        str(images), "--out", str(out), "--eps", "0.4", "--min_samples", "5"], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    order = sorted(names)  # the tool reads the feature files in sorted order
    xs = np.stack([x[names.index(nm)] for nm in order])
    ref = SkDBSCAN(eps=0.4, min_samples=5, metric="cosine").fit(xs).labels_
    n_clusters = len(set(ref)) - (1 if -1 in ref else 0)
    assert f"Estimated number of clusters: {n_clusters}" in r.stdout
    assert f"Estimated number of noise points: {int((ref == -1).sum())}" in r.stdout
    got = {d.name: sorted(p.name for p in d.iterdir()) for d in out.iterdir()}
    want = {str(c): sorted(f"{order[i]}.jpg" for i in np.nonzero(ref == c)[0]) for c in range(n_clusters)}
    assert got == want and n_clusters > 10
