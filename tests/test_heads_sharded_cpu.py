"""CPU checks of the class-sharded head: the shard entry points refuse bad shard descriptors and null operands before any
launch, the ctypes mirror of vdk_head_shard has the C size, the LocalShardGroup sum and barrier timeout behave, and
ShardedHead reads and writes the full [D, C] weight layout."""
import ctypes as C
import threading

import pytest
import torch

from visiondk_b200 import _lib


def _desc(batch=8, feat_dim=16, num_class=3):
    d = _lib.HeadDesc()
    d.kind, d.batch, d.feat_dim, d.num_class, d.scale = 0, batch, feat_dim, num_class, 32.0
    return d


def _calls(lib, d, s):
    """Every shard entry point with non-null dummy operands (never dereferenced: validation comes first)."""
    p = 256
    return {"cos": lambda: lib.vdk_head_shard_cos(C.byref(d), s, p, p, p, p, p, 1 << 30, 0),
            "forward": lambda: lib.vdk_head_shard_forward(C.byref(d), s, p, p, p, p, p, p, 1 << 30, 0),
            "combine": lambda: lib.vdk_head_shard_combine(C.byref(d), s, p, p, p, p, 0),
            "backward": lambda: lib.vdk_head_shard_backward(C.byref(d), s, p, p, p, p, p, p, p, p, p, 1 << 30, 0),
            "finalize": lambda: lib.vdk_head_shard_finalize(C.byref(d), s, p, p, p, 1 << 30, 0)}


@pytest.mark.parametrize("bad", ["null", "total_one", "negative_offset", "past_total", "rank_ge_world", "world_zero",
                                 "batch_not_multiple", "empty_shard"])
def test_shard_entry_points_refuse_bad_shards(lib, bad):
    d = _desc()
    s = _lib.HeadShard(0, 10, 2, 1)
    if bad == "total_one":
        s.num_class_total, d.num_class = 1, 1
    elif bad == "negative_offset":
        s.class_offset = -1
    elif bad == "past_total":
        s.class_offset = 8  # [8, 11) is not inside [0, 10)
    elif bad == "rank_ge_world":
        s.rank = 2
    elif bad == "world_zero":
        s.world, s.rank = 0, 0
    elif bad == "batch_not_multiple":
        s.world, s.rank = 3, 0
    elif bad == "empty_shard":
        d.num_class = 0
    ptr = None if bad == "null" else C.byref(s)
    for name, call in _calls(lib, d, ptr).items():
        assert call() == _lib.VDK_ERR_INVALID, (bad, name)
        assert "shard" in _lib.last_error() or "head shape" in _lib.last_error(), (bad, name, _lib.last_error())


def test_shard_entry_points_refuse_null_operands(lib):
    d = _desc(num_class=1)  # a one-class shard is valid: the refusal below is the operand's
    s = _lib.HeadShard(9, 10, 2, 1)
    assert lib.vdk_head_shard_cos(C.byref(d), C.byref(s), 0, 256, 256, 256, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "null operand" in _lib.last_error()
    assert lib.vdk_head_shard_forward(C.byref(d), C.byref(s), 256, 256, 0, 0, 0, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "null operand" in _lib.last_error()
    d.kind = 2  # MV-Softmax needs the label cosines
    assert lib.vdk_head_shard_forward(C.byref(d), C.byref(s), 256, 0, 0, 0, 256, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert lib.vdk_head_shard_backward(C.byref(d), C.byref(s), 256, 256, 256, 0, 256, 0, 256, 256, 256, 1 << 30, 0) == \
        _lib.VDK_ERR_INVALID
    assert lib.vdk_head_shard_combine(C.byref(d), C.byref(s), 256, 256, 0, 256, 0) == _lib.VDK_ERR_INVALID
    assert lib.vdk_head_shard_finalize(C.byref(d), C.byref(s), 256, 0, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert lib.vdk_head_shard_cos(C.byref(d), C.byref(s), 256, 256, 256, 256, 0, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "workspace" in _lib.last_error()
    d.feat_dim = 12
    assert lib.vdk_head_shard_backward(C.byref(d), C.byref(s), 256, 256, 256, 256, 256, 0, 256, 256, 256, 1 << 30, 0) == \
        _lib.VDK_ERR_INVALID
    assert "multiple of 8" in _lib.last_error()


def test_head_shard_struct_size(lib):
    out = (C.c_size_t * 1)()
    assert lib.vdk_head_shard_struct_sizes(out, 1) == 1
    assert out[0] == C.sizeof(_lib.HeadShard)


def test_local_group_sum_is_rank_ordered_and_identical_everywhere():
    from visiondk_b200.sharding import LocalShardGroup
    vals = [torch.tensor([1e8, 1.0, -1e8], dtype=torch.float32) * (r + 1) for r in range(3)]

    def fn(comm):
        t = vals[comm.rank].clone()
        comm.all_reduce_sum_(t)
        return t

    got = LocalShardGroup(3).run(fn)
    want = vals[0] + vals[1] + vals[2]
    for t in got:
        assert torch.equal(t, want)


def test_local_group_barrier_times_out_on_a_skipped_collective():
    from visiondk_b200.sharding import LocalShardGroup

    def fn(comm):
        if comm.rank == 0:
            return None  # a protocol bug: rank 0 skips the exchange the others wait in
        return comm.all_gather(torch.zeros(1))

    with pytest.raises(threading.BrokenBarrierError):
        LocalShardGroup(2, timeout=0.5).run(fn)


@pytest.mark.parametrize("world,num_class", [(3, 10), (8, 9), (1, 5)])
def test_sharded_head_state_dict_is_the_full_weight(world, num_class):
    from visiondk_b200.heads import ArcFace, ShardedHead
    from visiondk_b200.sharding import LocalShardGroup, shard_bounds
    torch.manual_seed(0)
    full = ArcFace(16, num_class)
    other = torch.randn(16, num_class)

    def fn(comm):
        head = ShardedHead(full, comm)
        lo, hi = shard_bounds(num_class, world, comm.rank)
        assert torch.equal(head.weight.detach(), full.weight.detach()[:, lo:hi])
        sd = head.state_dict()
        head.load_state_dict({"weight": other})
        return sd, head.weight.detach().clone(), head.state_dict()

    for r, (sd, w, sd2) in enumerate(LocalShardGroup(world).run(fn)):
        assert list(sd) == ["weight"] and torch.equal(sd["weight"], full.weight.detach())
        lo, hi = shard_bounds(num_class, world, r)
        assert torch.equal(w, other[:, lo:hi])
        assert torch.equal(sd2["weight"], other)


def test_sharded_head_refuses_a_wrong_full_shape():
    from visiondk_b200.heads import ArcFace, ShardedHead
    from visiondk_b200.sharding import LocalShardGroup
    full = ArcFace(16, 10)

    def fn(comm):
        head = ShardedHead(full, comm)
        with pytest.raises(RuntimeError, match="size mismatch"):
            head.load_state_dict({"weight": torch.zeros(16, 5)})

    LocalShardGroup(2).run(fn)
