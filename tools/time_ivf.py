"""Train, add and search times, resident bytes per row and recall of the IVF indexes against the exact Flat search:

    python tools/time_ivf.py [--rows 1000000] [--queries 10000] [--dim 512] [--nlist 4096] [--nprobe 1 8 32 128]
                             [--factories IVF4096,Flat IVF4096,PQ64] [--repeat 3] [--json out.json]

The gallery is identity-structured (like oracle.retrieval.synthetic_gallery: 16 noisy, L2-normalised members per random
centre, queries drawn the same way), generated on the device from a seed; on random Gaussian rows every list is equally far
from a query and IVF means nothing.  Per factory: train and add wall time (device-synchronised), then per nprobe the median
search time over `--repeat` calls (CUDA events, after a warm-up call), nbytes per row, and recall@1/10/100: the share of the
Flat top-k ids the IVF top-k finds.  The FlatIPIndex search of the same queries is timed in the same run for comparison.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        q = torch.cuda.get_device_name()
    return q


def timed(fn, repeat):
    fn()
    ts = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2], out


def recall(ids, ref, k):
    hit = (ids[:, :k, None] == ref[:, None, :k]).any(2).sum().item()
    return hit / (ref.shape[0] * k)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[1, 8, 32, 128])
    ap.add_argument("--factories", nargs="+", default=["IVF4096,Flat", "IVF4096,PQ64"])
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--json", default=None)
    opt = ap.parse_args(argv)
    from visiondk_b200.ivf import index_factory
    from visiondk_b200.retrieval import FlatIPIndex

    dev = torch.device("cuda", 0)
    g_ = torch.Generator(device=dev).manual_seed(0)
    per = 16
    centres = torch.randn((opt.rows + per - 1) // per, opt.dim, device=dev, generator=g_)
    g = centres.repeat_interleave(per, 0)[:opt.rows]
    g = torch.nn.functional.normalize(g + 0.5 * torch.randn(g.shape, device=dev, generator=g_))
    pick = torch.randint(0, centres.shape[0], (opt.queries,), device=dev, generator=g_)
    q = torch.nn.functional.normalize(centres[pick] + 0.5 * torch.randn(opt.queries, opt.dim, device=dev, generator=g_))
    del centres
    res = {"card": card(), "rows": opt.rows, "queries": opt.queries, "dim": opt.dim, "cases": []}
    print(res["card"], flush=True)

    flat = FlatIPIndex(opt.dim, dev)
    flat.add(g)
    t_flat, (_, ref) = timed(lambda: flat.search_device(q, 100, resolve_overflow=True), opt.repeat)
    res["flat_search_ms"] = t_flat
    res["flat_bytes_per_row"] = sum(t.numel() * t.element_size() for t in (flat._rows.x32, flat._rows.xh, flat._rows.norm,
                                                                           flat._rows.err)) / opt.rows
    print(f"Flat: search {t_flat:.1f} ms, {res['flat_bytes_per_row']:.0f} B/row", flush=True)
    del flat

    for spec in opt.factories:
        idx = index_factory(opt.dim, spec, dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        idx.train(g)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        idx.add(g)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        case = {"factory": spec, "train_s": t1 - t0, "add_s": t2 - t1, "bytes_per_row": idx.nbytes / idx.ntotal, "search": []}
        print(f"{spec}: train {t1 - t0:.1f} s, add {t2 - t1:.1f} s, {case['bytes_per_row']:.1f} B/row", flush=True)
        for nprobe in opt.nprobe:
            idx.nprobe = nprobe
            t, (_, ids) = timed(lambda: idx.search_device(q, 100), opt.repeat)
            row = {"nprobe": nprobe, "search_ms": t, **{f"recall@{k}": recall(ids, ref, k) for k in (1, 10, 100)}}
            case["search"].append(row)
            print(f"  nprobe {nprobe}: search {t:.1f} ms, recall@1/10/100 {row['recall@1']:.4f} {row['recall@10']:.4f} "
                  f"{row['recall@100']:.4f}", flush=True)
        res["cases"].append(case)
        del idx
        torch.cuda.empty_cache()
    if opt.json:
        with open(opt.json, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
