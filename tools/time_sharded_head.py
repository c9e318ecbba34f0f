"""Time and peak memory of the margin head's share of a face train step, unsharded and as one class shard of W ranks:

    python tools/time_sharded_head.py [--classes 58671 1000000 2000000] [--world 8] [--batch 128] [--repeat 10] [--json out.json]

Per case: the fused head forward + backward (ArcFace + CE, label smoothing 0.1, D = 512) and the head's optimizer sweep
(gradient sum of squares + SGD / clip / EMA over the head's parameter, gradient, momentum and EMA), timed with CUDA events
after warm-up, median of `--repeat` runs, and the peak device memory over those calls (head state + workspace + operands).
The unsharded case is one rank at batch B over all C classes; the shard case is one of W ranks: W·B gathered rows against
C/W classes.  The shard runs on one GPU, so the exchanges (all-gathers of features and partials, the sums of label
cosines and feature gradients) are not in its time; their bytes are printed as computed.  The card's name and power limit are
read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        q = torch.cuda.get_device_name()
    return q


def run_case(lib, rows, ncls_shard, ncls_total, world, D, repeat):
    from visiondk_b200 import _lib
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    d = _lib.HeadDesc()
    d.kind, d.batch, d.feat_dim, d.num_class = 0, rows, D, ncls_shard
    d.margin_arc, d.scale, d.label_smooth = 0.35, 32.0, 0.1
    s = _lib.HeadShard(0, ncls_total, world, 0)
    g = torch.Generator(device=dev).manual_seed(0)
    feats = torch.randn(rows, D, device=dev, generator=g)
    labels = torch.randint(0, ncls_shard, (rows,), device=dev, generator=g)
    n = D * ncls_shard
    p = torch.empty(n, device=dev).uniform_(-1, 1, generator=g)
    grad, mom, ema = torch.zeros_like(p), torch.zeros_like(p), p.clone()
    ws = torch.empty(lib.vdk_head_workspace_bytes(C.byref(d)), dtype=torch.uint8, device=dev)
    gt = torch.empty(rows, device=dev)
    partials = torch.empty(world, rows, 4, device=dev)
    lse, row_loss, loss = torch.empty(rows, device=dev), torch.empty(rows, device=dev), torch.empty((), device=dev)
    dfn = torch.empty(rows, D, device=dev)
    dfeats = torch.empty(rows // world, D, device=dev)
    sumsq = torch.zeros((), dtype=torch.float64, device=dev)
    sws = torch.empty(lib.vdk_grad_sumsq_workspace_bytes(), dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr()

    def step():
        if world == 1:  # the unsharded entry points
            _lib.check(lib.vdk_head_forward(C.byref(d), feats.data_ptr(), p.data_ptr(), labels.data_ptr(), 0, loss.data_ptr(),
                                            lse.data_ptr(), 0, ws.data_ptr(), ws.numel(), st), "vdk_head_forward")
            _lib.check(lib.vdk_head_backward(C.byref(d), feats.data_ptr(), p.data_ptr(), labels.data_ptr(), lse.data_ptr(), 0, 0,
                                             dfeats.data_ptr(), grad.data_ptr(), ws.data_ptr(), ws.numel(), st),
                       "vdk_head_backward")
        else:
            _lib.check(lib.vdk_head_shard_cos(C.byref(d), C.byref(s), feats.data_ptr(), p.data_ptr(), labels.data_ptr(),
                                              gt.data_ptr(), ws.data_ptr(), ws.numel(), st), "vdk_head_shard_cos")
            _lib.check(lib.vdk_head_shard_forward(C.byref(d), C.byref(s), labels.data_ptr(), gt.data_ptr(), 0, 0,
                                                  partials[0].data_ptr(), ws.data_ptr(), ws.numel(), st), "vdk_head_shard_forward")
            _lib.check(lib.vdk_head_shard_combine(C.byref(d), C.byref(s), partials.data_ptr(), lse.data_ptr(), row_loss.data_ptr(),
                                                  loss.data_ptr(), st), "vdk_head_shard_combine")
            _lib.check(lib.vdk_head_shard_backward(C.byref(d), C.byref(s), feats.data_ptr(), p.data_ptr(), labels.data_ptr(),
                                                   gt.data_ptr(), lse.data_ptr(), 0, dfn.data_ptr(), grad.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), st), "vdk_head_shard_backward")
            _lib.check(lib.vdk_head_shard_finalize(C.byref(d), C.byref(s), dfn.data_ptr(), dfeats.data_ptr(), ws.data_ptr(),
                                                   ws.numel(), st), "vdk_head_shard_finalize")
        _lib.check(lib.vdk_grad_sumsq(grad.data_ptr(), n, sumsq.data_ptr(), 0, sws.data_ptr(), sws.numel(), st), "vdk_grad_sumsq")
        _lib.check(lib.vdk_sgd_clip_ema_step(p.data_ptr(), grad.data_ptr(), mom.data_ptr(), ema.data_ptr(), n, sumsq.data_ptr(),
                                             10.0, 1e-4, 0.9, 5e-4, 0, 0.999, 0.001, 1, st), "vdk_sgd_clip_ema_step")

    # partials of the other shards: copies of this one's (the combine's work does not depend on their values)
    if world > 1:
        step()
        partials[1:] = partials[0]
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    peak = torch.cuda.max_memory_allocated() - base
    return {"rows": rows, "classes": ncls_shard, "classes_total": ncls_total, "world": world, "ms_median": times[len(times) // 2],
            "ms_min": times[0], "ms_max": times[-1], "peak_gib": peak / 2 ** 30, "workspace_gib": ws.numel() / 2 ** 30,
            "head_state_gib": 4 * n * 4 / 2 ** 30}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", type=int, nargs="+", default=[58671, 1_000_000, 2_000_000])
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--repeat", type=int, default=10)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sharded_head.py needs a CUDA device")
    from visiondk_b200 import _lib
    from visiondk_b200.sharding import shard_bounds
    lib = _lib.load()
    res = {"card": card(), "dim": a.dim, "batch": a.batch, "world": a.world, "cases": []}
    print(f"card: {res['card']}", flush=True)
    for cn in a.classes:
        W, B, D = a.world, a.batch, a.dim
        width = shard_bounds(cn, W, 0)[1]
        for case in (run_case(lib, B, cn, cn, 1, D, a.repeat), run_case(lib, W * B, width, cn, W, D, a.repeat)):
            # bytes on the wire per rank and step (ring collectives: (W-1)/W of the buffer each way)
            if case["world"] == 1:
                case["ddp_head_allreduce_bytes"] = 2 * (W - 1) / W * D * cn * 4
            else:
                gathered = W * B * D * 4 + W * B * 8 + W * W * B * 16  # features, labels, softmax partials
                summed = W * B * D * 4 + W * B * 4                     # feature-gradient partials, label cosines (MV)
                case["exchange_bytes"] = (W - 1) / W * gathered + 2 * (W - 1) / W * summed
            res["cases"].append(case)
            print(json.dumps(case), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
