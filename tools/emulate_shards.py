#!/usr/bin/env python
"""A W-way sharded search of the bench's gallery emulated on ONE H100 (W shards, one host thread each, the collectives replaced by
barriers — visiondk_b200.sharding.LocalShardGroup): checks the protocol against the unsharded search and prints the device time
of ONE shard's share of the work (total / W) and the range schedule.  What it cannot see: the NCCL
latency of the 2-3 small all-gathers and the 8 MB-per-rank list gather (measured by bench.py --gpus N).

    python tools/emulate_shards.py --world 8 [--nq 10000 --ng 1000000 --k 100]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--ng", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from visiondk_b200 import _lib, sharding
    from visiondk_b200.retrieval import FlatIPIndex, sharded_flat_search, shard_schedule
    _lib.load()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(5)
    whole = FlatIPIndex(a.dim, dev, normalize=True)
    shards = [FlatIPIndex(a.dim, dev, normalize=True, id_offset=sharding.shard_bounds(a.ng, a.world, r)[0]) for r in range(a.world)]
    for lo in range(0, a.ng, 125000):
        hi = min(a.ng, lo + 125000)
        blk = torch.nn.functional.normalize(torch.randn(hi - lo, a.dim, device=dev, generator=gen))
        whole.add(blk)
        for r in range(a.world):
            s0, s1 = sharding.shard_bounds(a.ng, a.world, r)
            s0, s1 = max(s0, lo), min(s1, hi)
            if s1 > s0:
                shards[r].add(blk[s0 - lo:s1 - lo].clone())
    q = torch.nn.functional.normalize(torch.randn(a.nq, a.dim, device=dev, generator=gen))
    ws, wi = whole.search_device(q, a.k, resolve_overflow=True)

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps

    ms1 = timed(lambda: whole.search_device(q, a.k))
    print(json.dumps({"variant": "unsharded", "ms": round(ms1, 3)}), flush=True)
    group = sharding.LocalShardGroup(a.world)

    def search():
        return group.run(lambda comm: sharded_flat_search(shards[comm.rank], q, [a.nq], a.k, defer_check=True, comm=comm), device=dev)

    res = search()
    ok = all(torch.equal(i, wi) and torch.equal(s.view(torch.int32), ws.view(torch.int32)) for s, i in res)
    for sh in shards:
        sh.check_status()
    ms = timed(search)
    with _lib.profile() as prof:
        search()
    torch.cuda.synchronize()
    sf = prof.totals["score_filter"]  # upper bound: another shard's launch can slip between a launch and its closing event
    sf = {"launches": sf["launches"], "ms_per_shard": round(sf["ms"] / a.world, 3)}
    print(json.dumps({"variant": "sharded", "world": a.world, "equals_unsharded": ok,
                      "schedule": shard_schedule(max(sh.ntotal for sh in shards), a.world, a.k),
                      "ms_all_shards": round(ms, 3), "ms_per_shard": round(ms / a.world, 3),
                      "score_filter": sf, "max_candidates": int(max(int(sh.last_status[1]) for sh in shards)),
                      "rerank_rows_max": int(max(int(sh.last_status[2]) for sh in shards))}), flush=True)
    if not ok:
        raise SystemExit("sharded result differs from the unsharded search")


if __name__ == "__main__":
    main()
