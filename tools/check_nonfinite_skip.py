"""Two-rank check that a non-finite gradient on ONE rank makes EVERY rank skip the optimizer step, under torchrun on one node:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29535 tools/check_nonfinite_skip.py

Backend: NCCL with one GPU per rank when the box has >= WORLD_SIZE GPUs; otherwise every rank uses cuda:0 and the collectives
run over gloo (tests/test_nonfinite_skip_multi_rank_gpu.py launches this script in whichever mode the box allows).

The clip norm is global, so its non-finite test is too: the DDP mean spreads a NaN in one rank's backbone gradient to every
rank, and the sharded head's sum of squares is summed over the ranks before any rank reads it.  On the toy ConvNeXt of
tools/check_multi_gpu.py with an ArcFace head, after one finite FaceTrainer step:
1. shard_head=True, a NaN in rank 1's head-shard gradient only;
2. shard_head=False (plain DDP mean), a NaN in rank 1's backbone gradient only, injected into the first gradient section
   before its all-reduce.
In each case every rank must leave its parameters and momentum unchanged bit for bit, zero its gradients and report a
non-finite grad_norm(); the replicated buffers (parameters and momentum of the DDP groups, and their EMA with the sharded head,
where every rank starts it from rank 0's) must stay equal across the ranks bit for bit; and the following finite step must apply on every rank and keep them equal.
Prints one JSON line on rank 0; exit code != 0 on any failed check.
"""
import hashlib
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist


def digest(ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def same_on_every_rank(value, world):
    everyone = [None] * world
    dist.all_gather_object(everyone, value)
    return all(v == everyone[0] for v in everyone)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    nccl = torch.cuda.device_count() >= world
    dev = torch.device("cuda", local if nccl else 0)
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    from visiondk_b200.train import FaceTrainer, FaceTrainingModel
    out = {"world": world, "backend": dist.get_backend()}
    ncls, B = 51, 8
    cfg = {"backbone": {"timm-toy": {"pretrained": False, "image_size": 64, "feat_dim": 64, "depths": (1, 1, 2, 1),
                                     "dims": (64, 128, 128, 256)}},
           "head": {"arcface": {"feat_dim": 64, "num_class": ncls, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32}}}
    gen = torch.Generator(device="cpu").manual_seed(23)
    xs = torch.randn(3, world * B, 3, 64, 64, generator=gen)
    ys = torch.randint(0, ncls, (3, world * B), generator=gen)
    for tag, shard in (("head_shard_nan", True), ("backbone_nan", False)):
        torch.manual_seed(13 + 1000 * rank)
        tr = FaceTrainer(FaceTrainingModel(cfg).to(dev), lr0=0.01, momentum=0.9, weight_decay=5e-4, label_smooth=0.1,
                         layer_wise=True, warm_steps=0, total_steps=100, use_ema=True, shard_head=shard)
        batch = lambda s: (xs[s, rank * B:(rank + 1) * B].to(dev), ys[s, rank * B:(rank + 1) * B].to(dev))
        tr.step(*batch(0))
        groups = tr.opt.groups
        replicated = tr._ddp_groups
        p0 = [g.p.clone() for g in groups]
        m0 = [g.mom.clone() for g in groups]
        u0 = tr.opt.updates
        poisoned = {"done": rank != 1}
        if shard:
            orig_step = tr.opt.step

            def step_with_nan():
                if rank == 1:
                    groups[-1].g[groups[-1].n // 2] = float("nan")
                    poisoned["done"] = True
                orig_step()
            tr.opt.step = step_with_nan
        else:
            orig_section = tr._on_section

            def section_with_nan(names):
                if rank == 1 and not poisoned["done"]:
                    sl = tr._flat_slice(names)
                    if sl is not None:
                        g, lo, _ = sl
                        g.g[lo] = float("nan")
                        poisoned["done"] = True
                orig_section(names)
            tr._on_section = section_with_nan
        tr.step(*batch(1))
        torch.cuda.synchronize()
        out[f"{tag}_injected"] = poisoned["done"]
        out[f"{tag}_params_kept"] = all(torch.equal(g.p.view(torch.int32), a.view(torch.int32)) for g, a in zip(groups, p0))
        out[f"{tag}_momentum_kept"] = all(torch.equal(g.mom.view(torch.int32), a.view(torch.int32)) for g, a in zip(groups, m0))
        out[f"{tag}_grads_zeroed"] = all(not bool(g.g.any()) for g in groups)
        out[f"{tag}_grad_norm_not_finite"] = not math.isfinite(tr.opt.grad_norm())
        out[f"{tag}_updates_counted"] = tr.opt.updates == u0 + 1
        # every rank's EMA starts from its own initialisation without shard_head (the reference keeps it on rank 0 only)
        rep = lambda: [g.p for g in replicated] + [g.mom for g in replicated] + ([g.ema for g in replicated] if shard else [])
        out[f"{tag}_ranks_equal_after_skip"] = same_on_every_rank(digest(rep()), world)
        if shard:
            tr.opt.step = orig_step
        else:
            tr._on_section = orig_section
        tr.step(*batch(2))
        torch.cuda.synchronize()
        out[f"{tag}_next_step_applies"] = (all(not torch.equal(g.p, a) for g, a in zip(groups, p0)) and
                                           math.isfinite(tr.opt.grad_norm()))
        out[f"{tag}_ranks_equal_after_next_step"] = same_on_every_rank(digest(rep()), world)
    everyone = [None] * world
    dist.all_gather_object(everyone, {k: v for k, v in out.items() if not isinstance(v, bool) or not v})
    out["by_rank"] = everyone  # each rank's failed checks
    flags = torch.tensor([1.0 if all(v for v in out.values() if isinstance(v, bool)) else 0.0], device=dev)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    ok = bool(flags.item() == 1.0)
    if rank == 0:
        out["ok"] = ok
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
