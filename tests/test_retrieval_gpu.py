"""GPU parity of the retrieval path (rows_prepare -> score_filter -> select/re-rank) against oracle/retrieval.py.

Bar: ids AND scores bit-exact (integer/index work; scores are defined canonically in the oracle).
"""
import numpy as np
import pytest
import torch

from oracle import retrieval as R
from visiondk_b200 import _lib
from visiondk_b200.retrieval import FlatIPIndex, PreparedRows, merge_topk, exact_pair_scores

pytestmark = pytest.mark.gpu


def unit_rows(n, dim, seed):
    rng = np.random.default_rng(seed)
    return R.l2_normalize(rng.standard_normal((n, dim)).astype(np.float32))


def assert_same(got_s, got_i, ref_s, ref_i, what):
    got_s, got_i = np.asarray(got_s), np.asarray(got_i)
    bad_rows = np.nonzero((got_i != ref_i).any(axis=1))[0]
    msg = ""
    if len(bad_rows):
        r = bad_rows[0]
        c = np.nonzero(got_i[r] != ref_i[r])[0][:5]
        msg = (f"{what}: {len(bad_rows)}/{got_i.shape[0]} rows differ; row {r} cols {c.tolist()} got ids "
               f"{got_i[r, c].tolist()} ref ids {ref_i[r, c].tolist()} got s {got_s[r, c].tolist()} ref s {ref_s[r, c].tolist()}")
    assert len(bad_rows) == 0, msg
    assert np.array_equal(got_s.view(np.uint32), ref_s.view(np.uint32)), f"{what}: ids equal but scores differ in bits"


def test_rows_prepare_matches_oracle(lib):
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((777, 512)) * rng.uniform(0.01, 30, (777, 1))).astype(np.float32)
    x[5] = 0.0  # zero row: eps clamp
    p = PreparedRows(torch.from_numpy(x).cuda(), normalize=True)
    ref = R.l2_normalize(x)
    got = p.x32.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    xh = p.xh.cpu().numpy()
    assert np.array_equal(xh.view(np.uint16), ref.astype(np.float16).view(np.uint16))
    err = np.linalg.norm(ref.astype(np.float64) - xh.astype(np.float64), axis=1)
    assert (p.err.cpu().numpy() >= err).all() and (p.err.cpu().numpy() <= err * 1.001 + 1e-20).all()
    nrm = np.linalg.norm(ref.astype(np.float64), axis=1)
    assert (p.norm.cpu().numpy() >= nrm * 0.999999).all()


@pytest.mark.parametrize("nq,ng,dim,k", [(50, 3000, 512, 10), (1, 1, 64, 1), (3, 5, 128, 10), (130, 4096, 256, 100),
                                         (257, 700, 512, 100), (17, 300, 320, 7)])
def test_topk_single_range_bit_exact(lib, nq, ng, dim, k):
    q, g = unit_rows(nq, dim, 10 + nq), unit_rows(ng, dim, 20 + ng)
    idx = FlatIPIndex(dim, "cuda")
    idx.train(g)
    idx.add(g)
    s, i = idx.search(q, k)
    info = idx.check_status()
    ref_s, ref_i = R.flat_ip_search(q, g, k)
    assert_same(s, i, ref_s, ref_i, f"single-range nq={nq} ng={ng} dim={dim} k={k} {info}")


@pytest.mark.parametrize("nq,ng,dim,k", [(300, 40000, 512, 100), (129, 70001, 128, 10), (64, 300000, 64, 1)])
def test_topk_multi_range_bit_exact(lib, nq, ng, dim, k):
    q, g = unit_rows(nq, dim, 1), unit_rows(ng, dim, 2)
    idx = FlatIPIndex(dim, "cuda")
    idx.add(g)
    s, i = idx.search(q, k)
    info = idx.check_status()
    ref_s, ref_i = R.flat_ip_search_candidates(q, g, k)
    assert_same(s, i, ref_s, ref_i, f"multi-range nq={nq} ng={ng} dim={dim} k={k} {info}")


def test_topk_planted_identities_and_normalize(lib):
    g, q, labels = R.synthetic_gallery(n_ids=300, per_id=100, dim=512, seed=2)
    # feed UN-normalised rows and let the index normalise (F.normalize fused in)
    rng = np.random.default_rng(9)
    g_raw = g * rng.uniform(0.5, 4.0, (g.shape[0], 1)).astype(np.float32)
    q_raw = q * rng.uniform(0.5, 4.0, (q.shape[0], 1)).astype(np.float32)
    idx = FlatIPIndex(512, "cuda", normalize=True)
    idx.add(g_raw)
    s, i = idx.search(q_raw, 100)
    idx.check_status()
    ref_s, ref_i = R.flat_ip_search_candidates(R.l2_normalize(q_raw), R.l2_normalize(g_raw), 100)
    assert_same(s, i, ref_s, ref_i, "planted identities")
    recall = np.mean([(labels[i[r]] == r).mean() for r in range(q.shape[0])])
    assert recall > 0.99, f"planted positives not retrieved: recall@100={recall}"


def test_topk_tie_rule_and_padding(lib):
    base = unit_rows(40, 128, 3)
    g = np.concatenate([base, base, base[:7]], axis=0)  # exact duplicates -> exact score ties
    q = unit_rows(9, 128, 4)
    idx = FlatIPIndex(128, "cuda")
    idx.add(g)
    s, i = idx.search(q, 100)  # k > ntotal: padded with (-FLT_MAX, -1)
    idx.check_status()
    ref_s, ref_i = R.flat_ip_search(q, g, 100)
    assert_same(s, i, ref_s, ref_i, "ties + padding")
    assert (i[:, 87:] == -1).all() and (s[:, 87:] == np.float32(-3.4028234663852886e38)).all()


def test_topk_empty_inputs(lib):
    idx = FlatIPIndex(64, "cuda")
    s, i = idx.search(unit_rows(3, 64, 1), 5)  # empty gallery
    assert (i == -1).all() and s.shape == (3, 5)
    idx.add(unit_rows(10, 64, 2))
    s, i = idx.search(np.zeros((0, 64), np.float32), 5)  # empty query block
    assert s.shape == (0, 5) and i.shape == (0, 5)


def test_topk_sharded_merge_equals_unsharded(lib):
    nq, ng, dim, k = 200, 50000, 512, 100
    q, g = unit_rows(nq, dim, 5), unit_rows(ng, dim, 6)
    whole = FlatIPIndex(dim, "cuda")
    whole.add(g)
    ws, wi = whole.search_device(torch.from_numpy(q).cuda(), k)
    whole.check_status()
    bounds = [0, 11000, 11001, 30000, ng]
    ss, ii = [], []
    for a, b in zip(bounds[:-1], bounds[1:]):
        shard = FlatIPIndex(dim, "cuda", id_offset=a)
        shard.add(g[a:b])
        s_, i_ = shard.search_device(torch.from_numpy(q).cuda(), k)
        shard.check_status()
        ss.append(s_)
        ii.append(i_)
    ms, mi = merge_topk(torch.stack(ss), torch.stack(ii), k)
    assert torch.equal(mi, wi) and torch.equal(ms.view(torch.int32), ws.view(torch.int32))
    ref_s, ref_i = R.merge_topk([s_.cpu().numpy() for s_ in ss], [i_.cpu().numpy() for i_ in ii], k)
    assert np.array_equal(mi.cpu().numpy(), ref_i)


def test_tensor_core_error_within_bound(lib):
    """The admission slack 2*eps relies on |fp16 tensor-core score - canonical score| <= eps; measure it."""
    nq, ng, dim = 256, 8192, 512
    q, g = unit_rows(nq, dim, 7), unit_rows(ng, dim, 8)
    qp = PreparedRows(torch.from_numpy(q).cuda(), False)
    gp = PreparedRows(torch.from_numpy(g).cuda(), False)
    approx = torch.empty((nq, ng), dtype=torch.float32, device="cuda")
    rc = lib.vdk_gemm_tn(qp.xh.data_ptr(), gp.xh.data_ptr(), approx.data_ptr(), nq, ng, dim, dim, dim, ng,
                         _lib.DTYPE_FP16, _lib.DTYPE_FP32, _lib.EPI_NONE, 0, 0, 0, 0, _lib.stream_ptr())
    _lib.check(rc, "vdk_gemm_tn")
    exact = (torch.from_numpy(q).cuda().double() @ torch.from_numpy(g).cuda().double().t())
    err = (approx.double() - exact).abs().max().item()
    gn, ge = gp.maxima()
    eps = (qp.err * gn + (qp.norm + qp.err) * ge + 2.0 ** -13 * (qp.norm + qp.err) * (gn + ge)).min().item()
    assert err <= eps, f"measured tensor-core score error {err:.3e} exceeds the bound {eps:.3e}"
    assert err >= 1e-6  # sanity: fp16 rounding really is in play


@pytest.mark.slow
def test_topk_full_size_properties(lib):
    """BASELINE config 4 at full size (10k x 1M x 512, k=100): size-independent properties + sampled brute force."""
    nq, ng, dim, k = 10000, 1000000, 512, 100
    gen = torch.Generator(device="cuda").manual_seed(5)
    g = torch.nn.functional.normalize(torch.randn(ng, dim, device="cuda", generator=gen))
    q = torch.nn.functional.normalize(torch.randn(nq, dim, device="cuda", generator=gen))
    idx = FlatIPIndex(dim, "cuda")
    idx.add(g)
    s, i = idx.search_device(q, k)
    info = idx.check_status()
    # sortedness under (score desc, id asc)
    ds = s[:, 1:] - s[:, :-1]
    assert (ds <= 0).all()
    assert ((ds < 0) | (i[:, 1:] > i[:, :-1])).all()
    assert (i >= 0).all() and (i < ng).all()
    # every returned score is the canonical score of its pair
    qi = torch.arange(nq, device="cuda").repeat_interleave(k)
    assert torch.equal(exact_pair_scores(q, g, qi, i.reshape(-1)).view(torch.int32), s.reshape(-1).view(torch.int32))
    # sampled brute force in fp64
    rows = torch.arange(0, nq, 499, device="cuda")
    full = q[rows].double() @ g.double().t()
    top = full.topk(k, dim=1).indices
    agree = (top == i[rows]).float().mean().item()
    assert agree > 0.999, f"sampled brute-force agreement {agree} ({info})"
    # BIT-EXACT against the oracle on 80 sampled query rows of the same gallery (ids and canonical scores): a dropped
    # true top-k member anywhere in these rows fails the test
    sample = np.arange(0, nq, 125)
    g_host, q_host = g.cpu().numpy(), q[torch.from_numpy(sample).cuda()].cpu().numpy()
    ref_s, ref_i = R.flat_ip_search_candidates(q_host, g_host, k)
    assert_same(s[sample].cpu().numpy(), i[sample].cpu().numpy(), ref_s, ref_i, f"full-size sampled rows ({info})")
    # the sharded path at full size: 8 row shards searched separately and merged (what 8 GPUs do) equals the unsharded
    # result bit for bit on EVERY row, hence the oracle on the sampled ones
    ss, ii = [], []
    for r in range(8):
        lo, hi = ng * r // 8, ng * (r + 1) // 8
        shard = FlatIPIndex(dim, "cuda", id_offset=lo)
        shard.add(g[lo:hi])
        s_, i_ = shard.search_device(q, k)
        shard.check_status()
        ss.append(s_)
        ii.append(i_)
        del shard
    ms, mi = merge_topk(torch.stack(ss), torch.stack(ii), k)
    assert torch.equal(mi, i) and torch.equal(ms.view(torch.int32), s.view(torch.int32))


def test_adversarially_ordered_gallery_takes_the_wide_path(lib):
    """Gallery sorted by increasing similarity to the queries: every later range beats the thresholds learnt on the
    earlier ones, candidate segments overflow, and the flagged queries must be recomputed (all-dense plan) exactly."""
    rng = np.random.default_rng(11)
    dim, ng, nq, k = 128, 60000, 40, 50
    p = rng.standard_normal(dim).astype(np.float32)
    g = R.l2_normalize(rng.standard_normal((ng, dim)).astype(np.float32) + 0.6 * p)
    order = np.argsort(g @ (p / np.linalg.norm(p)), kind="stable")
    g = g[order]
    q = R.l2_normalize(p[None, :] + 0.3 * rng.standard_normal((nq, dim)).astype(np.float32))
    idx = FlatIPIndex(dim, "cuda")
    idx.add(g)
    s, i = idx.search(q, k)  # numpy API resolves overflow
    assert idx.wide_path_rows > 0, "this gallery is built to overflow the admission segments"
    ref_s, ref_i = R.flat_ip_search_candidates(q, g, k)
    assert_same(s, i, ref_s, ref_i, "wide path")
    # the un-resolved device call reports the overflow instead of silently returning incomplete lists
    idx.search_device(torch.from_numpy(q).cuda(), k)
    with pytest.raises(RuntimeError):
        idx.check_status()


def test_massive_duplicates_take_the_exhaustive_path(lib):
    """5000 exact copies of one row: more ties than any carry list holds, on the wide path too.  faiss' flat search
    (engine/cbir/evaluation.py:193) answers such a gallery, so the index must as well: the flagged queries are scored
    against every row canonically and selected exactly (score desc, id asc) — the oracle's answer, bit for bit."""
    rng = np.random.default_rng(5)
    v = unit_rows(1, 64, 1)
    g = np.concatenate([unit_rows(700, 64, 3), np.repeat(v, 5000, axis=0), unit_rows(300, 64, 4)], axis=0)
    g = g[rng.permutation(len(g))]
    q = np.concatenate([unit_rows(2, 64, 2), v, -v], axis=0)  # the duplicated row itself, and its antipode (all ties LAST)
    idx = FlatIPIndex(64, "cuda")
    idx.add(g)
    for k in (10, 100, 1024):
        s, i = idx.search(q, k)
        ref_s, ref_i = R.flat_ip_search(q, g, k)
        assert_same(s, i, ref_s, ref_i, f"massive duplicates k={k}")
    assert idx.exhaustive_rows > 0, "this gallery is built to overflow the carry lists even on the wide path"
    # device call without resolution still reports instead of returning incomplete lists
    idx.search_device(torch.from_numpy(q).cuda(), 10)
    with pytest.raises(RuntimeError):
        idx.check_status()


def test_exhaustive_path_alone_matches_oracle(lib):
    """vdk_ip_topk_exhaustive on its own (every query forced through it), incl. k > ntotal padding and an id offset."""
    q, g = unit_rows(19, 128, 31), unit_rows(3001, 128, 32)
    g[100] = g[7]
    g[2999] = g[7]
    idx = FlatIPIndex(128, "cuda", id_offset=1000)
    idx.add(g)
    idx._finalize()
    for k in (1, 10, 100):
        s, i = idx._exhaustive(torch.from_numpy(q).cuda(), k)
        ref_s, ref_i = R.flat_ip_search(q, g, k, id_offset=1000)
        assert_same(s.cpu().numpy(), i.cpu().numpy(), ref_s, ref_i, f"exhaustive k={k}")
    small = FlatIPIndex(128, "cuda")
    small.add(g[:5])
    small._finalize()
    s, i = small._exhaustive(torch.from_numpy(q).cuda(), 10)
    ref_s, ref_i = R.flat_ip_search(q, g[:5], 10)
    assert_same(s.cpu().numpy(), i.cpu().numpy(), ref_s, ref_i, "exhaustive padded")


def test_l2_variant_of_the_cosine_index(lib):
    """north_star names cosine / L2: for L2-normalised rows the squared distance is 2 - 2 cos, so search_l2 returns the same ids
    as search with ascending distances; checked against a brute-force fp64 L2 ranking of the oracle-normalised rows."""
    from oracle import retrieval as oret
    from visiondk_b200.retrieval import FlatIPIndex
    rng = np.random.default_rng(3)
    g = rng.standard_normal((5000, 128)).astype(np.float32)
    q = rng.standard_normal((37, 128)).astype(np.float32)
    index = FlatIPIndex(128, "cuda", normalize=True)
    index.add(g)
    d, i = index.search_l2(q, 10)
    s, i2 = index.search(q, 10)
    assert np.array_equal(i, i2) and np.all(np.diff(d, axis=1) >= 0)
    np.testing.assert_array_equal(d, (2.0 - 2.0 * s).astype(np.float32))
    qn, gn = oret.l2_normalize(q).astype(np.float64), oret.l2_normalize(g).astype(np.float64)
    d64 = ((qn[:, None, :] - gn[None, :, :]) ** 2).sum(-1)
    ref = np.argsort(d64, axis=1, kind="stable")[:, :10]
    # identical sets per query; order may differ only where fp32 scores tie within rounding
    assert all(set(a) == set(b) for a, b in zip(i.tolist(), ref.tolist()))
    np.testing.assert_allclose(d, np.take_along_axis(d64, i, axis=1), atol=5e-6)
    with pytest.raises(ValueError):
        FlatIPIndex(128, "cuda", normalize=False).search_l2(q, 3)



def test_bound_from_sketches_matches_the_counting_argument(lib):
    from visiondk_b200.retrieval import bound_from_sketches
    rng = np.random.default_rng(3)
    for n_shards, ranks, k in [(8, [100, 50, 25, 13], 100), (2, [10, 5], 10), (5, [7, 4, 2, 1], 7), (3, [1], 1)]:
        nq = 301
        sk = np.sort(rng.standard_normal((n_shards, nq, len(ranks))).astype(np.float32), axis=2)  # smaller rank -> larger score
        sk[rng.random(sk.shape) < 0.2] = -np.inf  # shards with fewer candidates than a rank
        sk[0, :, 0] = np.maximum(sk[0, :, 0], 0.5)  # a rank-k entry that carries an older global bound (not monotone in the rank)
        bound = rng.standard_normal(nq).astype(np.float32)
        bound[::7] = -np.inf
        want = R.bound_from_sketches(sk, ranks, k, bound)
        got = torch.from_numpy(bound).cuda()
        bound_from_sketches(torch.from_numpy(sk).cuda(), ranks, k, got)
        assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32)), (n_shards, ranks, k)


@pytest.mark.parametrize("world,clustered,k", [(8, False, 100), (8, True, 100), (3, False, 100), (8, False, 1)])
def test_sharded_protocol_on_local_shards(lib, world, clustered, k):
    """The W-shard search (range schedule, rank-sketch exchange after every range, bounded re-rank, packed merge) with the
    collectives replaced by barriers between W host threads on one GPU: every shard must return the unsharded answer, bit for
    bit, and every published sketch entry must be a TRUE lower bound (>= r rows of that shard score at least sketch[r]).
    At k = 1 the shards exchange only the element-wise max of their k-th bounds."""
    from visiondk_b200 import sharding
    from visiondk_b200.retrieval import sharded_flat_search, bound_from_sketches, _Exchange
    nq, ng, dim = 256, 120000, 128
    q, g = unit_rows(nq, dim, 41), unit_rows(ng, dim, 42)
    if clustered:  # all near neighbours of query j live in ONE shard (a gallery stored class by class)
        rng = np.random.default_rng(43)
        per = ng // world
        for j in range(nq):
            a = (j % world) * per + 5000 + (j // world) * 160
            g[a:a + 150] = R.l2_normalize(q[j] + 0.05 * rng.standard_normal((150, dim)).astype(np.float32))
    whole = FlatIPIndex(dim, "cuda")
    whole.add(g)
    qd = torch.from_numpy(q).cuda()
    ws, wi = whole.search_device(qd, k, resolve_overflow=True)
    ref_s, ref_i = R.flat_ip_search_candidates(q[:32], g, k)
    assert_same(ws[:32].cpu().numpy(), wi[:32].cpu().numpy(), ref_s, ref_i, "unsharded vs oracle")

    shards = []
    for r in range(world):
        a, b = sharding.shard_bounds(ng, world, r)
        sh = FlatIPIndex(dim, "cuda", id_offset=a)
        sh.add(g[a:b])
        shards.append(sh)
    group = sharding.LocalShardGroup(world)
    gathered = []

    def one(comm):
        class Spy:  # records what the shards publish
            world, rank = comm.world, comm.rank

            def all_gather(self, src):
                out = comm.all_gather(src)
                if comm.rank == 0 and out.dtype == torch.float32 and out.dim() == 3:
                    gathered.append(out.clone())
                return out

            def all_reduce_max_(self, t):
                comm.all_reduce_max_(t)

        return sharded_flat_search(shards[comm.rank], qd, [nq], k, comm=Spy())

    results = group.run(one, device=torch.cuda.current_device())
    for r, (s, i) in enumerate(results):
        assert torch.equal(i, wi) and torch.equal(s.view(torch.int32), ws.view(torch.int32)), f"shard {r} disagrees"
    for sh in shards:
        sh.check_status()
    ranks = _Exchange(None, group.comm(0), k).ranks
    assert ranks == R.sketch_ranks(k, world)
    if k == 1:
        assert ranks == [1] and not gathered  # no sketch is published
    else:
        assert len(ranks) > 1 and len(gathered) >= 2  # one exchange per gallery range
        g_dev = torch.from_numpy(g).cuda()
        kth_true = ws[:, k - 1]  # the global k-th canonical score
        for sk in gathered:
            assert sk.shape == (world, nq, len(ranks))
            for r in range(world):
                a, b = sharding.shard_bounds(ng, world, r)
                scores = qd @ g_dev[a:b].T  # fp32; sketch entries are bounds with >= 1e-4 of slack (eps of the fp16 pass)
                for j, rank in enumerate(ranks):
                    val = sk[r, :, j]
                    cnt = (scores >= (val - 1e-5).unsqueeze(1)).sum(dim=1)
                    ok = (cnt >= rank) | torch.isinf(val)
                    if rank == k:  # a rank-k entry may instead carry the GLOBAL bound the shard already knew: still <= the answer
                        ok |= val <= kth_true + 1e-6
                    assert bool(ok.all()), f"shard {r} rank {rank}: a sketch entry is not a lower bound"
            bound = torch.full((nq,), float("-inf"), device="cuda")
            bound_from_sketches(sk, ranks, k, bound)
            assert bool((bound <= kth_true + 1e-6).all()), "the derived bound exceeds the true global k-th score"
        if not clustered:  # neighbours spread evenly: the sketch bound must beat the best single shard's k-th by a wide margin
            last = gathered[-1]
            kth_best_shard = last[:, :, 0].amax(dim=0)
            share = last[:, :, -1].amin(dim=0)
            assert float((share > kth_best_shard).float().mean()) > 0.9
            final = torch.full((nq,), float("-inf"), device="cuda")
            bound_from_sketches(last, ranks, k, final)
            assert float((kth_true - final).median()) < 0.03  # and it is tight: within 0.03 of the true k-th score (sigma = 0.088)


@pytest.mark.parametrize("n_lists", [1, 2, 3, 5, 8, 17, 32])
def test_packed_merge_matches_the_oracle_rule(lib, n_lists):
    """vdk_topk_merge_packed (grouped-lane kernel) against oracle merge_topk: (score desc, id asc), padding, score ties
    across lists, negative scores, lists that end early, more queries than fit the last warp."""
    from visiondk_b200.retrieval import pack_topk, merge_topk_packed
    rng = np.random.default_rng(100 + n_lists)
    nq, k = 203, 37
    pool = np.round(rng.standard_normal(64).astype(np.float32), 1)  # few distinct scores: ties across and inside lists
    ss, ii = [], []
    for l in range(n_lists):
        ids = np.stack([rng.permutation(1000)[:k] for _ in range(nq)]).astype(np.int64) * n_lists + l  # disjoint between lists
        sc = pool[rng.integers(0, len(pool), size=(nq, k))]
        order = np.lexsort((ids, -sc.astype(np.float64)), axis=1)
        sc, ids = np.take_along_axis(sc, order, 1), np.take_along_axis(ids, order, 1)
        n_valid = rng.integers(0, k + 1, size=nq)  # lists padded with (-FLT_MAX, -1), some empty
        pad = np.arange(k)[None, :] >= n_valid[:, None]
        sc[pad], ids[pad] = R.FLT_LOWEST, -1
        ss.append(sc)
        ii.append(ids)
    ref_s, ref_i = R.merge_topk(ss, ii, k)
    packed = torch.stack([pack_topk(torch.from_numpy(s_).cuda(), torch.from_numpy(i_).cuda()) for s_, i_ in zip(ss, ii)])
    got_s, got_i = merge_topk_packed(packed, k)
    assert_same(got_s.cpu().numpy(), got_i.cpu().numpy(), ref_s, ref_i, f"packed merge of {n_lists} lists")
    gen_s, gen_i = merge_topk(torch.from_numpy(np.stack(ss)).cuda(), torch.from_numpy(np.stack(ii)).cuda(), k)
    assert torch.equal(gen_i, got_i) and torch.equal(gen_s.view(torch.int32), got_s.view(torch.int32))
