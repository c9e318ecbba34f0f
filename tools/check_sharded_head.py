"""Class-sharded head parity under torchrun on one node:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29534 tools/check_sharded_head.py

Backend: NCCL with one GPU per rank when the box has >= WORLD_SIZE GPUs; otherwise every rank uses cuda:0 and the collectives
run over gloo (tests/test_sharded_head_multi_rank_gpu.py launches this script in whichever mode the box allows).

For ArcFace and MV-Softmax on the toy ConvNeXt of tools/check_multi_gpu.py, with C = 51 classes (not divisible by the world
size) and both layer_wise settings (one or two parameter groups):
1. FaceTrainer steps with the head sharded and unsharded, from the same initial state and batches: each rank's losses, the
   backbone parameters, and the gathered head weight, momentum and head EMA agree within fp32-rounding tolerances (below: the
   two modes differ only in the order of the softmax combine and of the feature-gradient sum, a few ulps per step, which the
   SGD steps carry into the weights).  ArcFace runs three steps.  MV-Softmax runs one: its logit is discontinuous in cos (the
   hard-negative threshold, the label's gt > 0 branch), so once the two trajectories differ in the last bits an element can
   land on the other side of a branch and change its gradient by a finite amount (seen in the second and third steps here:
   up to 7e-3 of the largest momentum).  The per-element arithmetic of the branches is held bit for bit to the unsharded
   logits by tests/test_heads_sharded_gpu.py;
2. the Epoch_N.pt dicts of both modes have the same keys and tensor shapes;
3. each mode restores the other's checkpoint with the head, EMA head and head momentum bit for bit.
Prints one JSON line on rank 0; exit code != 0 on any mismatch.
"""
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

LOSS_RTOL = 2e-5    # a loss: a few fp32 roundings of the combined log-sum-exp apart
PARAM_RTOL = 2e-5   # parameters, momentum and EMA after three steps, relative to the tensor's largest magnitude


def rel_err(a, b):
    """max |a - b| over the tensor's largest magnitude"""
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def shapes(tree):
    if isinstance(tree, dict):
        return {k: shapes(v) for k, v in tree.items()}
    if isinstance(tree, (list, tuple)):
        return [shapes(v) for v in tree]
    if torch.is_tensor(tree):
        return ["tensor", list(tree.shape), str(tree.dtype)]
    return type(tree).__name__


def head_states(trainer):
    from engine.vision_engine import CenterProcessor
    if trainer.shard_head:
        return CenterProcessor.gathered_head_state(trainer)
    host = lambda sd: {k: v.detach().cpu().clone() for k, v in sd.items()}
    return {"head": host(trainer.model.trainingwrapper["head"].state_dict()),
            "ema_head": host(trainer.ema.trainingwrapper["head"].state_dict()), "trainer": trainer.state_dict()}


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    nccl = torch.cuda.device_count() >= world
    dev = torch.device("cuda", local if nccl else 0)
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    from engine.vision_engine import CenterProcessor
    from visiondk_b200.train import FaceTrainer, FaceTrainingModel
    out = {"world": world, "backend": dist.get_backend()}
    ncls, B = 51, 8
    heads = {"arcface": {"feat_dim": 64, "num_class": ncls, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32},
             "mv-softmax": {"feat_dim": 64, "num_class": ncls, "is_am": False, "margin": 0.35, "mv_weight": 1.12, "scale": 32}}
    gen = torch.Generator(device="cpu").manual_seed(21)
    xs = torch.randn(3, world * B, 3, 64, 64, generator=gen)
    ys = torch.randint(0, ncls, (3, world * B), generator=gen)
    ok = True
    for name, hcfg in heads.items():
        for layer_wise in (True, False):
            tag = f"{name}_{'layerwise' if layer_wise else 'onegroup'}"
            cfg = {"backbone": {"timm-toy": {"pretrained": False, "image_size": 64, "feat_dim": 64, "depths": (1, 1, 2, 1),
                                             "dims": (64, 128, 128, 256)}}, "head": {name: hcfg}}
            torch.manual_seed(11 + 1000 * rank)  # different per rank: only rank 0's broadcast state may survive
            base = FaceTrainingModel(cfg).to(dev)
            kw = dict(lr0=0.01, momentum=0.9, weight_decay=5e-4, label_smooth=0.1, layer_wise=layer_wise, warm_steps=0,
                      total_steps=100, use_ema=True)
            tu = FaceTrainer(copy.deepcopy(base), **kw)
            ts = FaceTrainer(copy.deepcopy(base), shard_head=True, **kw)
            losses = {"u": [], "s": []}
            for step in range(3 if name == "arcface" else 1):
                x = xs[step, rank * B:(rank + 1) * B].to(dev)
                y = ys[step, rank * B:(rank + 1) * B].to(dev)
                losses["u"].append(float(tu.step(x, y)))
                losses["s"].append(float(ts.step(x, y)))
            out[f"{tag}_losses"] = losses
            out[f"{tag}_losses_close"] = all(abs(a - b) <= LOSS_RTOL * abs(b) for a, b in zip(losses["s"], losses["u"]))
            bu = torch.cat([p.detach().reshape(-1) for p in tu.model.trainingwrapper["backbone"].parameters()])
            bs = torch.cat([p.detach().reshape(-1) for p in ts.model.trainingwrapper["backbone"].parameters()])
            su, ss = head_states(tu), head_states(ts)
            mu, ms = su["trainer"]["optimizer"]["momentum_buffers"], ss["trainer"]["optimizer"]["momentum_buffers"]
            errs = {"backbone": rel_err(bs, bu), "head": rel_err(ss["head"]["weight"], su["head"]["weight"]),
                    "momentum": max(rel_err(a, b) for a, b in zip(ms, mu)) if len(mu) == len(ms) else float("inf")}
            # the unsharded trainer's EMA is rank 0's (the other ranks' copies start from their own initialisation)
            if rank == 0:
                errs["ema_head"] = rel_err(ss["ema_head"]["weight"], su["ema_head"]["weight"])
            out[f"{tag}_rank{rank}_errors"] = errs
            for k, e in errs.items():
                out[f"{tag}_{k}_close"] = e <= PARAM_RTOL
            # 2. checkpoints of both modes have the same layout (rank 0 writes the file every rank reads)
            cu = CenterProcessor.checkpoint(tu, 0, 3, {"fitness": {}}, None)
            cs = CenterProcessor.checkpoint(ts, 0, 3, {"fitness": {}}, ss)
            box = [cu, cs]
            dist.broadcast_object_list(box, src=0)
            cu, cs = box
            out[f"{tag}_checkpoint_layout_equal"] = shapes(cu) == shapes(cs)
            if rank != 0:
                out[f"{tag}_ema_head_close"] = True  # keeps the key set equal on every rank
            # 3. cross-mode resume restores the head bit for bit
            fresh_s = FaceTrainer(FaceTrainingModel(cfg).to(dev), shard_head=True, **kw)
            CenterProcessor.restore_checkpoint(fresh_s, cu)
            rs = head_states(fresh_s)
            fresh_u = FaceTrainer(FaceTrainingModel(cfg).to(dev), **kw)
            CenterProcessor.restore_checkpoint(fresh_u, cs)
            ru = head_states(fresh_u)
            out[f"{tag}_resume_sharded_from_unsharded_exact"] = (
                torch.equal(rs["head"]["weight"], cu["head"]["weight"]) and
                torch.equal(rs["ema_head"]["weight"], cu["ema_head"]["weight"]) and
                torch.equal(rs["trainer"]["optimizer"]["momentum_buffers"][-1], cu["optimizer"]["momentum_buffers"][-1]))
            out[f"{tag}_resume_unsharded_from_sharded_exact"] = (
                torch.equal(ru["head"]["weight"], cs["head"]["weight"]) and
                torch.equal(ru["ema_head"]["weight"], cs["ema_head"]["weight"]) and
                torch.equal(ru["trainer"]["optimizer"]["momentum_buffers"][-1], cs["optimizer"]["momentum_buffers"][-1]))
    everyone = [None] * world
    dist.all_gather_object(everyone, {k: v for k, v in out.items() if not isinstance(v, bool) or not v})
    out["by_rank"] = everyone  # each rank's errors and failed checks
    flags = torch.tensor([1.0 if all(v for v in out.values() if isinstance(v, bool)) else 0.0], device=dev)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)  # every rank's own comparisons must hold
    ok = bool(flags.item() == 1.0)
    if rank == 0:
        out["ok"] = ok
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
