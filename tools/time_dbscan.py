"""Per-phase device times of DBSCAN (cosine) and scikit-learn's time on this host's CPU:

    python tools/time_dbscan.py [--rows 100000 1000000] [--dense_rows 262144] [--dense_group 4096] [--dim 512] [--eps 0.4]
                                [--min_samples 5] [--sklearn_from 10000] [--sklearn_budget 180] [--json out.json]

Rows are identity-structured (groups of 16 noisy members around a random centre, like tools/time_ivf.py), generated on the
device from a seed.  The largest N goes through a raw fp16 memmap store in a temporary directory, as cbir.index writes it,
and is clustered by the reference's call with only the import changed: DBSCAN(eps=0.4, min_samples=5, metric="cosine",
n_jobs=16).fit(X).  Per N: CUDA-event times of prepare, count, union, border and finalise, the Gram kernels alone, pairs
rechecked by the canonical score, bands redone, and the Gram passes' achieved TFLOP/s (2 dim per scored pair over Gram kernel
time) against the H100 SXM's dense fp16 989.  --dense_rows adds one case of near-duplicate groups of --dense_group rows
(noise 0.1): every row is core with thousands of neighbours, the load that stresses the union pass's union-find.
scikit-learn runs at --sklearn_from rows and doubles the size until a run takes longer than --sklearn_budget seconds (or
would pass the largest --rows): the last size is the first it did not finish within the budget.  The card's name and
power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        q = torch.cuda.get_device_name()
    return q


def rows(n, dim, seed=0, per=16, noise=0.5):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    centres = torch.randn((n + per - 1) // per, dim, device=dev, generator=g)
    x = centres.repeat_interleave(per, 0)[:n] + noise * torch.randn(n, dim, device=dev, generator=g)
    return x[torch.randperm(n, device=dev, generator=g)]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--eps", type=float, default=0.4)
    ap.add_argument("--min_samples", type=int, default=5)
    ap.add_argument("--dense_rows", type=int, default=262_144)
    ap.add_argument("--dense_group", type=int, default=4096)
    ap.add_argument("--sklearn_from", type=int, default=10_000)
    ap.add_argument("--sklearn_budget", type=float, default=180.0)
    ap.add_argument("--json", default=None)
    opt = ap.parse_args(argv)
    from visiondk_b200.cluster import DBSCAN

    res = {"card": card(), "dim": opt.dim, "eps": opt.eps, "min_samples": opt.min_samples, "cases": [], "sklearn": []}
    print(res["card"], flush=True)
    DBSCAN(eps=opt.eps, min_samples=opt.min_samples).fit_device(rows(4096, opt.dim, seed=99))  # warm-up: module load
    cases = [(n, 16, 0.5) for n in sorted(opt.rows)]
    if opt.dense_rows:
        cases.insert(0, (opt.dense_rows, opt.dense_group, 0.1))
    for n, per, noise in cases:
        x = rows(n, opt.dim, per=per, noise=noise)
        if n == max(opt.rows):  # the reference's call on a raw fp16 store
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "embeddings.f16")
                mm = np.memmap(path, mode="w+", dtype=np.float16, shape=(n, opt.dim))
                mm[:] = x.half().cpu().numpy()
                mm.flush()
                del mm, x
                X = np.memmap(path, mode="r", dtype=np.float16).reshape(-1, opt.dim)
                db = DBSCAN(eps=opt.eps, min_samples=opt.min_samples, metric="cosine", n_jobs=16)
                db.timing = True
                t0 = time.perf_counter()
                db.fit(X)
                wall = time.perf_counter() - t0
                source = "fp16 memmap, DBSCAN.fit"
                labels = db.labels_
        else:
            db = DBSCAN(eps=opt.eps, min_samples=opt.min_samples, timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            db.fit_device(x)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            source = "device tensor, DBSCAN.fit_device"
            labels = db.labels_.cpu().numpy()
            del x
        st = db.stats_
        nc = st["n_core"]
        pairs = {"count": n * (n - 1) / 2, "union": nc * (nc - 1) / 2, "border": (n - nc) * nc}
        gram_ms = sum(st["gram_ms"].values())
        flop = 2.0 * opt.dim * sum(pairs.values())
        case = {"rows": n, "group": per, "noise": noise, "source": source, "wall_s": wall, "ms": st["ms"], "gram_ms": st["gram_ms"],
                "rechecked_pairs": st["rechecked_pairs"], "redone_bands": st["redone_bands"], "n_core": nc,
                "n_clusters": st["n_clusters"], "n_noise": int((labels == -1).sum()),
                "gram_tflops": flop / (gram_ms * 1e-3) / 1e12 if gram_ms > 0 else None}
        case["share_of_989"] = case["gram_tflops"] / 989.0 if case["gram_tflops"] else None
        res["cases"].append(case)
        print(json.dumps(case), flush=True)
        torch.cuda.empty_cache()

    from sklearn.cluster import DBSCAN as SkDBSCAN
    n = opt.sklearn_from
    while n <= max(opt.rows):
        x = rows(n, opt.dim).cpu().numpy()
        t0 = time.perf_counter()
        ref = SkDBSCAN(eps=opt.eps, min_samples=opt.min_samples, metric="cosine", n_jobs=16).fit(x)
        t = time.perf_counter() - t0
        ours = DBSCAN(eps=opt.eps, min_samples=opt.min_samples, timing=True).fit(x)
        row = {"rows": n, "sklearn_s": t, "cpus": os.cpu_count(), "ours_device_ms": sum(ours.stats_["ms"].values()),
               "labels_equal": bool(np.array_equal(ref.labels_, ours.labels_))}
        res["sklearn"].append(row)
        print(json.dumps(row), flush=True)
        if t > opt.sklearn_budget:
            break
        n *= 2
    if opt.json:
        with open(opt.json, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
