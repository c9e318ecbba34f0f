#!/usr/bin/env python
"""main.py — train entry point (reference flags: --cfgs --resume --sync_bn --project --name --local_rank --print_freq
--save_freq; env LOCAL_RANK / WORLD_SIZE from torchrun).  New code: dispatches the faceX / cbir embedding task to
engine.vision_engine.CenterProcessor.run_embedding on the H100 kernels.

    python main.py --cfgs configs/faceX/cbir_convnext_b200.yaml
    torchrun --nproc_per_node 8 --master-addr 127.0.0.1 main.py --cfgs configs/faceX/cbir_convnext_b200.yaml
"""
import argparse
import os
import shutil
from pathlib import Path

import torch
import torch.distributed as dist

from engine.vision_engine import CenterProcessor, check, increment_path, yaml_load

LOCAL_RANK = int(os.getenv("LOCAL_RANK", -1))
WORLD_SIZE = int(os.getenv("WORLD_SIZE", 1))


def parse_opt():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfgs", default="configs/faceX/cbir_convnext_b200.yaml")
    ap.add_argument("--resume", default="")
    ap.add_argument("--sync_bn", action="store_true", help="SyncBatchNorm for the neck (vision_engine.py:224-225); a no-op on one rank, refused on several")
    ap.add_argument("--project", default="run")
    ap.add_argument("--name", default="exp")
    ap.add_argument("--local_rank", type=int, default=-1)
    ap.add_argument("--print_freq", type=int, default=50)
    ap.add_argument("--save_freq", type=int, default=1)
    ap.add_argument("--shard_head", action="store_true",
                    help="split the margin head's classes over the ranks (each holds and updates C/W columns; checkpoints keep "
                         "the full head)")
    return ap.parse_args()


def main(opt):
    save_dir = increment_path(Path(opt.project) / opt.name)
    if LOCAL_RANK != -1:
        assert torch.cuda.device_count() > LOCAL_RANK, "not enough CUDA devices for this rank"
        dist.init_process_group(backend="nccl", world_size=WORLD_SIZE, rank=LOCAL_RANK)
    cfgs = yaml_load(opt.cfgs)
    check(cfgs["model"]["task"], cfgs)  # utils/checks.py:225-229
    if LOCAL_RANK in (-1, 0):
        save_dir.mkdir(parents=True, exist_ok=True)
        shutil.copy(opt.cfgs, save_dir)
    cpu = CenterProcessor(cfgs, LOCAL_RANK, project=str(save_dir), opt=opt)
    cpu.run_embedding(opt.resume or None)
    if LOCAL_RANK != -1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main(parse_opt())
