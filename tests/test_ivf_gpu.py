"""GPU tests of the IVF-Flat and IVF-PQ indexes (visiondk_b200/ivf.py, csrc/ivf.cu) against the numpy oracle (oracle/ivf.py),
bit for bit: trained centroids, codebooks and codes, search scores and ids, and the cbir.index / cbir.search plumbing."""
import numpy as np
import pytest
import torch

from oracle import ivf as O
from oracle import retrieval as R
from visiondk_b200.ivf import IVFIndex, index_factory
from visiondk_b200.retrieval import FlatIPIndex

pytestmark = pytest.mark.gpu


def bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def stored_lists(idx):
    """The GPU index's list of every stored id, in id order."""
    sizes = (idx.list_offsets[1:] - idx.list_offsets[:-1]).cpu()
    lists = np.empty(idx.ntotal, np.int64)
    lists[idx.list_ids.cpu().numpy()] = np.repeat(np.arange(idx.nlist), sizes.numpy())
    return lists


def stored_codes(idx):
    codes = np.empty((idx.ntotal, idx.pq_m), np.uint8)
    codes[idx.list_ids.cpu().numpy()] = idx.codes.cpu().numpy()
    return codes


def duplicate_gallery(n=3000, d=64, n_dup=1200, seed=7):
    """Half random rows, n_dup exact copies of one row (the first nlist rows of the training permutation hold several of
    them, so clusters go empty at the first update and the split runs; scores tie at every top-k boundary)."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((n, d)).astype(np.float32)
    g[rng.choice(n, n_dup, replace=False)] = g[0]
    g = R.l2_normalize(g)
    q = R.l2_normalize(np.concatenate([g[:3] + 0.01 * rng.standard_normal((3, d)).astype(np.float32),
                                       rng.standard_normal((37, d)).astype(np.float32)]))
    return g, q


@pytest.fixture(scope="module")
def small():
    g, q = duplicate_gallery()
    ref = O.build(g, 16, 8)
    pq = IVFIndex(64, 16, 8, "cuda")
    pq.train(g)
    pq.add(g)
    flat = index_factory(64, "IVF16,Flat", "cuda")
    flat.train(g)
    flat.add(g)
    return g, q, ref, pq, flat


def test_training_is_bit_exact(small):
    g, q, ref, pq, flat = small
    ids, init = O.training_sample(g.shape[0], 16)
    assert len(set(map(tuple, g[init]))) < 16  # the initial centroids repeat: the empty-cluster split ran
    assert bits_equal(pq.centroids.cpu().numpy(), ref["centroids"])
    assert bits_equal(flat.centroids.cpu().numpy(), ref["centroids"])
    assert bits_equal(pq.codebooks.cpu().numpy(), ref["codebooks"])
    assert np.array_equal(stored_lists(pq), ref["lists"]) and np.array_equal(stored_lists(flat), ref["lists"])
    assert np.array_equal(stored_codes(pq), ref["codes"])
    for idx in (pq, flat):  # list-major, ascending ids inside a list
        off = idx.list_offsets.cpu().numpy()
        ids_ = idx.list_ids.cpu().numpy()
        assert all(np.all(np.diff(ids_[off[i]:off[i + 1]]) > 0) for i in range(16))
    assert bits_equal(flat.list_rows.cpu().numpy(), g[flat.list_ids.cpu().numpy()])


@pytest.mark.parametrize("nprobe", [1, 3, 40])
@pytest.mark.parametrize("k", [10, 1024])
def test_search_is_bit_exact(small, nprobe, k):
    g, q, ref, pq, flat = small
    for idx, kw in ((pq, {"codes": ref["codes"], "codebooks": ref["codebooks"]}), (flat, {"rows": g})):
        idx.nprobe = nprobe
        s, i = idx.search(q, k)
        rs, ri = O.search(q, ref["centroids"], ref["lists"], k, nprobe, **kw)
        assert np.array_equal(i, ri) and bits_equal(s, rs)
        if k == 1024 and nprobe < 16:
            assert (i == -1).any()  # fewer rows in the probed lists than k: padded


def test_empty_lists_and_chunked_search(small):
    g, q, ref, _, _ = small
    keep = [int(ref["lists"][0]), 5, 11]  # the duplicates' list and two others
    part = g[np.isin(ref["lists"], keep)][:140]
    lists_ref = O.coarse_assign(part, ref["centroids"])
    assert set(np.unique(lists_ref)) <= set(keep)  # the other lists stay empty
    for spec, kw in (("IVF16,PQ8", {"codes": O.pq_assign(O.residuals(part, ref["centroids"], lists_ref), ref["codebooks"]),
                                    "codebooks": ref["codebooks"]}), ("IVF16,Flat", {"rows": part})):
        idx = index_factory(64, spec, "cuda")
        idx.train(g)
        idx.add(part[:50])
        idx.add(part[50:])  # incremental add
        idx.search_chunk_keys = 64  # one query per chunk
        idx.nprobe = 5
        s, i = idx.search(q, 20)
        rs, ri = O.search(q, ref["centroids"], lists_ref, 20, 5, **kw)
        assert np.array_equal(i, ri) and bits_equal(s, rs)


def test_ivf_flat_probing_every_list_is_flat(small):
    g, q, _, _, flat = small
    flat.nprobe = flat.nlist
    exact = FlatIPIndex(64, "cuda")
    exact.add(g)
    for k in (1, 10, 1024):
        s, i = flat.search(q, k)
        fs, fi = exact.search(q, k)
        assert np.array_equal(i, fi) and bits_equal(s, fs)


def test_chunked_memmap_add_equals_in_memory_add(small, tmp_path):
    g, q, _, pq, _ = small
    mm = np.memmap(tmp_path / "g.f16", mode="w+", dtype=np.float16, shape=g.shape)
    mm[:] = g
    mm.flush()
    store = np.memmap(tmp_path / "g.f16", mode="r", dtype=np.float16).reshape(-1, 64)
    a = IVFIndex(64, 16, 8, "cuda")
    a.train(store)
    a.add(torch.from_numpy(np.asarray(store, np.float32)).cuda())
    b = IVFIndex(64, 16, 8, "cuda")
    b.add_chunk_rows = 700
    b.train(store)
    b.add(store)
    assert bits_equal(a.centroids.cpu(), b.centroids.cpu()) and bits_equal(a.codebooks.cpu(), b.codebooks.cpu())
    assert torch.equal(a.list_ids, b.list_ids) and torch.equal(a.codes, b.codes) and torch.equal(a.list_offsets, b.list_offsets)
    a.nprobe = b.nprobe = 4
    sa, ia = a.search(q, 50)
    sb, ib = b.search(q, 50)
    assert np.array_equal(ia, ib) and bits_equal(sa, sb)


@pytest.mark.slow
def test_million_rows_nlist_4096():
    """1 M x 512 identity-structured rows, IVF4096 trained on the GPU: 64 sampled queries equal the oracle recomputed from
    the index's own centroids, codebooks and codes, for IVF-PQ64 and for IVF-Flat on the same centroids."""
    torch.manual_seed(0)
    n, d, per = 1 << 20, 512, 16
    centres = torch.randn(n // per, d, device="cuda")
    g = torch.nn.functional.normalize(centres.repeat_interleave(per, 0) + 0.5 * torch.randn(n, d, device="cuda"))
    q = torch.nn.functional.normalize(centres[torch.randperm(n // per, device="cuda")[:64]] + 0.5 * torch.randn(64, d, device="cuda"))
    pq = IVFIndex(d, 4096, 64, "cuda")
    pq.train(g)
    pq.add(g)
    assert pq.ntotal == n
    # per row: 64 B of codes + an 8 B id; fixed: fp32 centroids, the quantizer's fp16 copy and norm / error scalars,
    # the codebooks and the list offsets (about 12.6 B per row at this nlist)
    fixed = 4096 * d * 4 + 4096 * d * 2 + 2 * 4096 * 4 + 64 * 256 * (d // 64) * 4 + 4097 * 8
    assert pq.nbytes == n * (64 + 8) + fixed, pq.nbytes
    flat = IVFIndex(d, 4096, None, "cuda")
    flat._set_centroids(pq.centroids)
    flat.add(g)
    lists = stored_lists(pq)
    assert np.array_equal(lists, stored_lists(flat))
    gh, qh, c = g.cpu().numpy(), q.cpu().numpy(), pq.centroids.cpu().numpy()
    codes, cb = stored_codes(pq), pq.codebooks.cpu().numpy()
    probe = np.argsort(-R.canonical_scores(qh, c), axis=1, kind="stable")[:, :32]
    sel = np.isin(lists, np.unique(probe))  # only rows of lists some query probes can matter
    sub = np.nonzero(sel)[0]
    for idx, kw in ((pq, {"codes": codes[sub], "codebooks": cb}), (flat, {"rows": gh[sub]})):
        idx.nprobe = 32
        s, i = idx.search(qh, 100)
        rs, ri = O.search(qh, c, lists[sub], 100, 32, ids=sub, **kw)
        assert np.array_equal(i, ri) and bits_equal(s, rs)
    del g


def test_cbir_index_and_search(tmp_path):
    from oracle.convnext import TimmWrapperOracle, randomize_
    from visiondk_b200.backbone import TimmWrapper
    from visiondk_b200.cbir import FeatureExtractor, index, search

    depths, dims = (1, 1, 2, 1), (32, 64, 128, 256)
    oracle = randomize_(TimmWrapperOracle("toy", 64, 64, depths=depths, dims=dims), seed=5).eval()
    model = TimmWrapper("toy", 64, 64, pretrained=False, depths=depths, dims=dims)
    model.load_state_dict(oracle.state_dict(), strict=True)
    torch.manual_seed(0)
    gallery_x, query_x = torch.randn(600, 3, 64, 64), torch.randn(30, 3, 64, 64)
    batches = lambda x: [x[a:a + 64] for a in range(0, x.shape[0], 64)]  # noqa: E731
    ext = FeatureExtractor(model)
    path = str(tmp_path / "gallery.f32")
    q_emb = ext.extract_cbir(batches(query_x), "cuda")
    for spec in ("IVF8,Flat", "IVF8,PQ16x8"):
        idx = index(ext, batches(gallery_x), "cuda", index_factory=spec, memmap_save_path=path)
        assert isinstance(idx, IVFIndex) and idx.ntotal == 600
        idx.nprobe = 3
        scores, ids = search(ext, batches(query_x), idx, "cuda", k=10)
        g_emb = np.asarray(np.memmap(path, mode="r", dtype=np.float32).reshape(-1, 64))
        ref = O.build(g_emb, 8, 16 if "PQ" in spec else None)
        kw = {"codes": ref["codes"], "codebooks": ref["codebooks"]} if "PQ" in spec else {"rows": g_emb}
        rs, ri = O.search(q_emb, ref["centroids"], ref["lists"], 10, 3, **kw)
        assert np.array_equal(ids, ri) and bits_equal(scores, rs)
        idx2 = index(ext, None, "cuda", index_factory=spec, memmap_feat_dim=64, memmap_dtype=np.float32, memmap_save_path=path,
                     memmap_load_embedding=True)
        idx2.nprobe = 3
        s2, i2 = idx2.search(q_emb, 10)
        assert np.array_equal(i2, ri) and bits_equal(s2, rs)
