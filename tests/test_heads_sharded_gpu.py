"""The class-sharded margin head (heads.ShardedHead, csrc/heads.cu vdk_head_shard_*) on one GPU.

W shards run as sharding.LocalShardGroup threads through the explicit sharded_head_forward / sharded_head_backward (the
autograd node runs collectives inside its backward, which needs one process per rank: tests/test_sharded_head_multi_rank_gpu.py).

- W = 1: the shard calls give vdk_head_forward / vdk_head_backward's outputs bit for bit.
- W in {2, 3, 8}: every output sits in a NaN-guarded buffer (kernel_ref.Guarded).  Cos and logits equal the matching columns
  of an unsharded vdk_head_forward on the gathered batch bit for bit (the per-element contraction and margin are unchanged;
  MV-Softmax's label cosine comes from the same GEMM).  The assembled outputs are checked against fp64 with
  heads_ref.check_head, which uses one grad_out for both gradients: each rank's dfeats is the gradient of its own mean loss,
  W times the gradient of the mean over all W·B rows, so it is compared scaled by 1/W.  Each rank's loss is checked against
  the fp64 mean of its own rows.
- C = 1 000 000, W = 8, B = 128: the eight shards run one after another; cos on sampled rows and columns and row_lse / loss
  on sampled rows against fp64, and the peak memory of one shard against the unsharded head's workspace.
"""
import ctypes as C
import math

import pytest
import torch

import heads_ref as R
from kernel_ref import Guarded
from test_heads_bounds_cpu import KINDS
from test_heads_fp64_gpu import SHAPES, _head, desc_of, run_kernel

pytestmark = pytest.mark.gpu


def run_sharded(k, feats, w, labels, h, world, grad_out=1.0):
    """The sharded step on `world` LocalShardGroup threads; returns the per-rank outputs (guard-checked) in rank order."""
    from visiondk_b200.heads import ShardedHead, sharded_head_backward, sharded_head_forward
    from visiondk_b200.sharding import LocalShardGroup
    N, D = feats.shape
    B = N // world
    full = _head(k, D, w.shape[1], w)
    f_dev, y_dev = feats.cuda(), labels.cuda()
    gout = torch.tensor(grad_out, dtype=torch.float32, device="cuda")

    def shard(comm):
        head = ShardedHead(full, comm)
        cs = head.weight.shape[1]
        g = dict(logits=Guarded(N, cs, cs, torch.float32), cos=Guarded(N, cs, cs, torch.float32),
                 row_lse=Guarded(1, N, N, torch.float32), row_loss=Guarded(1, N, N, torch.float32),
                 loss=Guarded(1, 1, 1, torch.float32), dfeats=Guarded(B, D, D, torch.float32),
                 dweight=Guarded(D, cs, cs, torch.float32))
        rows = slice(comm.rank * B, (comm.rank + 1) * B)
        fwd = dict(logits=g["logits"].view, cos=g["cos"].view, row_lse=g["row_lse"].view[0], row_loss=g["row_loss"].view[0],
                   loss=g["loss"].view[0, 0])
        _, saved = sharded_head_forward(head, f_dev[rows], y_dev[rows], h["label_smooth"], outputs=fwd)
        sharded_head_backward(head, saved, gout, outputs=dict(dfeats=g["dfeats"].view, dweight=g["dweight"].view))
        torch.cuda.synchronize()
        for name, buf in g.items():
            assert not buf.guard_errors(), f"rank {comm.rank} {name}: {buf.guard_errors()}"
        out = {n: g[n].view.clone() for n in ("logits", "cos", "dfeats", "dweight")}
        out.update(row_lse=g["row_lse"].view[0].clone(), row_loss=g["row_loss"].view[0].clone(),
                   loss=g["loss"].view[0, 0].clone(), lo=head.class_offset)
        return out

    return LocalShardGroup(world).run(shard, device=torch.device("cuda", 0))


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{b}-D{d}-C{c}" for b, d, c in SHAPES])
@pytest.mark.parametrize("k", range(len(KINDS)))
def test_one_shard_is_the_unsharded_head_bit_for_bit(lib, k, shape):
    B, D, Cn = shape
    mv_arc = KINDS[k]["kind"] == "mv_softmax" and not KINDS[k]["is_am"]
    for smooth in (0.0, 0.1):
        feats, w, labels = R.make_case(B, D, Cn, seed=7000 + 100 * k + B + Cn, label_cos_max=0.9999 if mv_arc else None)
        h = R.head_consts(**KINDS[k], label_smooth=smooth)
        ref = run_kernel(lib, feats, w, labels, h)
        got = run_sharded(k, feats, w, labels, h, 1)[0]
        for name in ("cos", "logits", "row_lse", "loss", "dfeats", "dweight"):
            assert same_bits(got[name], ref[name]), f"{name} differs from vdk_head_forward/backward ({shape}, eps={smooth})"


CASES = [(2, 9, 8, 64), (2, 58671, 80, 128), (3, 257, 32, 128), (3, 1000, 53, 64), (8, 9, 20, 64), (8, 1000, 20, 128),
         (8, 58671, 20, 512)]  # (W, C, B per rank, D); W·B <= 160


@pytest.mark.parametrize("case", CASES, ids=[f"W{w}-C{c}-B{b}-D{d}" for w, c, b, d in CASES])
@pytest.mark.parametrize("k", range(len(KINDS)))
def test_shards_match_fp64_and_the_unsharded_columns(lib, k, case):
    world, Cn, B, D = case
    N = world * B
    mv_arc = KINDS[k]["kind"] == "mv_softmax" and not KINDS[k]["is_am"]
    stats = {}
    for smooth, same in ((0.0, False), (0.1, False), (0.1, True)):  # same: every label inside one shard
        feats, w, labels = R.make_case(N, D, Cn, seed=9000 + 100 * k + world + Cn, same_label=same,
                                       label_cos_max=0.9999 if mv_arc else None)
        h = R.head_consts(**KINDS[k], label_smooth=smooth)
        tag = f" {h['kind']} W={world} C={Cn} eps={smooth} same={same}"
        shards = run_sharded(k, feats, w, labels, h, world)
        ref = run_kernel(lib, feats, w, labels, h, backward=False)
        for r, s in enumerate(shards):
            lo, cs = s["lo"], s["cos"].shape[1]
            assert same_bits(s["cos"], ref["cos"][:, lo:lo + cs]), f"rank {r}: cos differs from the unsharded columns{tag}"
            assert same_bits(s["logits"], ref["logits"][:, lo:lo + cs]), f"rank {r}: logits differ from the unsharded columns{tag}"
            assert same_bits(s["row_lse"], shards[0]["row_lse"]), f"rank {r}: row_lse differs between the ranks{tag}"
        out = dict(cos=torch.cat([s["cos"] for s in shards], 1), logits=torch.cat([s["logits"] for s in shards], 1),
                   row_lse=shards[0]["row_lse"], dfeats=torch.cat([s["dfeats"] for s in shards], 0) / world,
                   dweight=torch.cat([s["dweight"] for s in shards], 1))
        info = R.check_head(out, feats, w, labels, h, stats=stats, tag=tag)
        assert info["nan_rows"] == 0
        # each rank's loss: the mean CE of its own rows (fixed-order warp mean: ceil(B/32) + 6 roundings)
        s2 = R.stage2_reference(out["cos"].double(), labels.cuda(), h)
        for r, s in enumerate(shards):
            rows = slice(r * B, (r + 1) * B)
            ref_loss = s2["loss_row"][rows].mean()
            bound = s2["e_loss_row"][rows].sum() / B + (math.ceil(B / 32) + 6) * R.A * s2["loss_row"][rows].abs().mean()
            err = abs(float(s["loss"]) - float(ref_loss))
            assert err <= float(bound), f"rank {r} loss {float(s['loss'])} vs fp64 {float(ref_loss)} (bound {float(bound)}){tag}"


@pytest.mark.slow
def test_million_classes_one_shard_of_eight(lib):
    """C = 1 000 000 over W = 8 at B = 128 per rank: each shard holds 1 024 rows x 125 000 classes.  The eight shards run in turn
    on one device and their partials are combined as the exchange would; rank 0 then runs its backward.  Checked against fp64:
    cos on 16 sampled rows x 4 096 sampled columns, row_lse and the row losses on the sampled rows (whose full rows are
    assembled from the shards' cosines), and rank 0's loss as the mean of its row losses; the gradients are checked against
    fp64 at the smaller shapes above and here only for being finite.  Prints the shard's memory next to the unsharded head's."""
    from visiondk_b200 import _lib
    world, Cn, B, D = 8, 1_000_000, 128, 512
    N = world * B
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(N, D, generator=g) * 2.0
    labels = torch.randint(0, Cn, (N,), generator=g)
    h = R.head_consts(**KINDS[0], label_smooth=0.1)
    f, y = feats.cuda(), labels.cuda()
    torch.manual_seed(6)
    w_full = torch.empty(D, Cn, device="cuda").uniform_(-1, 1).renorm_(2, 1, 1e-5).mul_(1e5)
    sample_rows = torch.randperm(B, generator=g)[:16]  # rank 0's rows
    sample_cols = torch.randperm(Cn, generator=g)[:4096].sort().values
    cos_rows = torch.empty(16, Cn, dtype=torch.float32, device="cuda")
    partials = torch.empty(world, N, 4, dtype=torch.float32, device="cuda")
    peak = 0
    from visiondk_b200.sharding import shard_bounds
    for r in range(world):
        lo, hi = shard_bounds(Cn, world, r)
        w = w_full[:, lo:hi].contiguous()
        d = desc_of(h, N, D, hi - lo)
        s = _lib.HeadShard(lo, Cn, world, r)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        ws = torch.empty(lib.vdk_head_workspace_bytes(C.byref(d)), dtype=torch.uint8, device="cuda")
        gt = torch.empty(N, device="cuda")
        cos = torch.empty(N, hi - lo, device="cuda")
        _lib.check(lib.vdk_head_shard_cos(C.byref(d), C.byref(s), f.data_ptr(), w.data_ptr(), y.data_ptr(), gt.data_ptr(),
                                          ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_head_shard_cos")
        _lib.check(lib.vdk_head_shard_forward(C.byref(d), C.byref(s), y.data_ptr(), gt.data_ptr(), 0, cos.data_ptr(),
                                              partials[r].data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()),
                   "vdk_head_shard_forward")
        cos_rows[:, lo:hi] = cos[sample_rows.cuda()]
        del cos
        if r == 0:  # one shard's whole step: forward, combine, backward, finalize
            lse, row_loss, loss = (torch.empty(N, device="cuda"), torch.empty(N, device="cuda"),
                                   torch.empty((), device="cuda"))
            torch.cuda.synchronize()
            keep_ws, keep_gt = ws, gt
        del ws
        torch.cuda.synchronize()
        peak = max(peak, torch.cuda.max_memory_allocated() - base)
    s0 = _lib.HeadShard(0, Cn, world, 0)
    d0 = desc_of(h, N, D, shard_bounds(Cn, world, 0)[1])
    _lib.check(lib.vdk_head_shard_combine(C.byref(d0), C.byref(s0), partials.data_ptr(), lse.data_ptr(), row_loss.data_ptr(),
                                          loss.data_ptr(), _lib.stream_ptr()), "vdk_head_shard_combine")
    w0 = w_full[:, :shard_bounds(Cn, world, 0)[1]].contiguous()
    dfn = torch.empty(N, D, device="cuda")
    dw = torch.empty_like(w0)
    dfe = torch.empty(B, D, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _lib.check(lib.vdk_head_shard_backward(C.byref(d0), C.byref(s0), f.data_ptr(), w0.data_ptr(), y.data_ptr(), keep_gt.data_ptr(),
                                           lse.data_ptr(), 0, dfn.data_ptr(), dw.data_ptr(), keep_ws.data_ptr(), keep_ws.numel(),
                                           _lib.stream_ptr()), "vdk_head_shard_backward")
    _lib.check(lib.vdk_head_shard_finalize(C.byref(d0), C.byref(s0), dfn.data_ptr(), dfe.data_ptr(), keep_ws.data_ptr(),
                                           keep_ws.numel(), _lib.stream_ptr()), "vdk_head_shard_finalize")
    torch.cuda.synchronize()
    assert bool(torch.isfinite(dw).all()) and bool(torch.isfinite(dfe).all())
    shard_ws = keep_ws.numel()
    full_ws = lib.vdk_head_workspace_bytes(C.byref(desc_of(h, B, D, Cn)))
    head_state = 4 * D * Cn * 4  # parameter, gradient, momentum, EMA
    print(f"MEMORY C=1M W=8 B=128: one shard's workspace {shard_ws / 2**30:.2f} GiB (peak forward {peak / 2**30:.2f} GiB, backward "
          f"{(torch.cuda.max_memory_allocated() - base) / 2**30:.2f} GiB over its inputs), head state {head_state / world / 2**30:.2f} "
          f"GiB; unsharded head: workspace {full_ws / 2**30:.2f} GiB, head state {head_state / 2**30:.2f} GiB")
    # fp64 checks on the sampled rows
    fs = feats[sample_rows].cuda()
    cr = R.cos_reference(fs, w_full[:, sample_cols.cuda()])
    from kernel_ref import check_within
    check_within(cos_rows[:, sample_cols.cuda()].double(), cr["cos"], cr["bound"], "cos C=1M", lambda b: f"{int(b.sum())}")
    s2 = R.stage2_reference(cos_rows.double(), y[sample_rows.cuda()], h)
    check_within(lse[sample_rows.cuda()].double(), s2["lse"], s2["e_lse"], "row_lse C=1M", lambda b: f"{int(b.sum())}")
    check_within(row_loss[sample_rows.cuda()].double(), s2["loss_row"], s2["e_loss_row"], "row_loss C=1M",
                 lambda b: f"{int(b.sum())}")
    assert abs(float(loss) - float(row_loss[:B].double().mean())) <= 1e-5 * abs(float(loss)) + 1e-6
