"""faceX train step on H100 (SURVEY.md §8a rows a1-a3, a9-a12): the reference's model container and step, same names.

  FaceTrainingModel      models/faceX/face_model.py:28-54   (trainingwrapper = ModuleDict{'backbone','head'})
  cosine_with_warm       engine/scheduler.py:47-57          (LinearLR 0.1->1 then CosineAnnealingLR, stepped per batch)
  SeperateLayerParams    built/layer_optimizer.py:9-29      (backbone lr, head lr x10)
  FaceTrainer.step       engine/procedure/train.py:196-215,230  (criterion∘model, backward, clip, SGD, zero_grad, EMA, LR)
  DDP                    engine/vision_engine.py:509-510    -> one NCCL all-reduce(mean) of the flat gradient buffers

All arithmetic is the sm_90a kernels: backbone forward/backward (csrc/convnext_train.cu), fused margin head + CE
(csrc/heads.cu), fused clip + SGD + EMA (csrc/optim.cu).
"""
from __future__ import annotations

import copy
import math
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .backbone import BackboneFactory
from .heads import HeadFactory, ShardedHead, margin_ce_loss, sharded_margin_ce_loss
from .optim import FusedSGDClipEMA


class FaceTrainingModel(nn.Module):
    """models/faceX/face_model.py:28-54."""

    def __init__(self, model_cfg: dict):
        super().__init__()
        backbone = BackboneFactory(model_cfg["backbone"]).get_backbone()
        head = HeadFactory(model_cfg["head"]).get_head()
        self.trainingwrapper = nn.ModuleDict({"backbone": backbone, "head": head})

    def forward(self, data, label):
        feat = self.trainingwrapper["backbone"](data)
        return self.trainingwrapper["head"](feat, label)

    def loss(self, data, label, label_smooth: float = 0.0):
        """criterion(self(data, label), label) with criterion = CrossEntropyLoss(label_smoothing), fused
        (train.py:196: the two are only ever called together)."""
        feat = self.trainingwrapper["backbone"](data)
        head = self.trainingwrapper["head"]
        if isinstance(head, ShardedHead):
            return sharded_margin_ce_loss(head, feat, label, label_smooth)
        return margin_ce_loss(head, feat, label, label_smooth)

    def shard_head_(self, comm=None) -> None:
        """Replaces the head by this rank's class shard (heads.ShardedHead) of rank 0's full weight: the columns the unsharded
        trainer would hold after broadcasting rank 0's initial state."""
        head = self.trainingwrapper["head"]
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(head.weight.data, src=0)
        self.trainingwrapper["head"] = ShardedHead(head, comm)


def cosine_with_warm_lr(step: int, base_lr: float, lr0: float, warm: int, total: int, lrf_ratio: Optional[float]) -> float:
    """Learning rate of a param group with base lr `base_lr` after `step` scheduler steps under engine/scheduler.py:47-57:
    SequentialLR([LinearLR(0.1 -> 1, warm), CosineAnnealingLR(total - warm, eta_min = lrf * lr0)], milestones=[warm]).
    Note eta_min is lrf * the GLOBAL lr0 for every group (the head group's base lr is 10 * lr0)."""
    lrf = 0.1 if lrf_ratio is None else lrf_ratio
    if warm > 0 and step < warm:
        return base_lr * (0.1 + 0.9 * step / warm)
    eta_min = lrf * lr0
    t, T = step - warm, max(1, total - warm)
    return eta_min + (base_lr - eta_min) * 0.5 * (1 + math.cos(math.pi * t / T))


def layer_wise_groups(model: FaceTrainingModel, layer_wise: bool, lr: float):
    """built/layer_optimizer.py:9-29."""
    if not layer_wise:
        return [{"params": list(model.parameters()), "lr": lr}]
    return [{"params": list(model.trainingwrapper["backbone"].parameters()), "lr": lr},
            {"params": list(model.trainingwrapper["head"].parameters()), "lr": lr * 10}]


class FaceTrainer:
    """The per-batch body of Trainer.train_one_epoch_face (engine/procedure/train.py:217-233) on H100.

    shard_head: split the head's classes over the ranks (heads.ShardedHead).  The head then is its own flat parameter group
    (also with layer_wise=False), which the DDP all-reduce and the initial broadcast leave out; clipping uses the global
    gradient norm.  Every rank must pass the same use_ema: each keeps the EMA of its own head columns.  `state_dict` and
    `load_state_dict` read and write the unsharded layout, so checkpoints move between the two modes; `state_dict` is then
    a collective."""

    def __init__(self, model: FaceTrainingModel, lr0: float, momentum: float, weight_decay: float, label_smooth: float = 0.0,
                 layer_wise: bool = True, warm_steps: int = 0, total_steps: int = 1, lrf_ratio: Optional[float] = None,
                 use_ema: bool = True, max_norm: float = 10.0, shard_head: bool = False):
        self.model = model
        self.label_smooth = label_smooth
        self.shard_head, self.layer_wise = shard_head, layer_wise
        if shard_head:
            model.shard_head_()
        self.ema = copy.deepcopy(model).eval() if use_ema else None  # models/ema.py:20-26
        if self.ema is not None:
            for p in self.ema.parameters():
                p.requires_grad_(False)
        groups = layer_wise_groups(model, layer_wise, lr0)
        if shard_head and not layer_wise:
            groups = [{"params": list(model.trainingwrapper["backbone"].parameters()), "lr": lr0},
                      {"params": list(model.trainingwrapper["head"].parameters()), "lr": lr0}]
        self.base_lrs = [g["lr"] for g in groups]
        self.opt = FusedSGDClipEMA(groups, lr=lr0, momentum=momentum, weight_decay=weight_decay, max_norm=max_norm, model=model,
                                   ema_model=self.ema, sharded_groups=(len(groups) - 1,) if shard_head else ())
        # the groups DDP averages and the initial broadcast covers: every group but the head's shard
        self._ddp_groups = self.opt.groups[:-1] if shard_head else self.opt.groups
        self.lr0, self.warm, self.total, self.lrf = lr0, warm_steps, total_steps, lrf_ratio
        self.sched_step = 0
        self._apply_lr()
        self._broadcast_initial_state()

    def _broadcast_initial_state(self):
        """DistributedDataParallel broadcasts rank 0's parameters and buffers when it wraps the model
        (engine/vision_engine.py:509-510); without it every rank would keep its own random initialisation and only the
        gradients would be shared.  Same here, on the flat parameter buffers (+ momentum) and every module buffer."""
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        for g in self._ddp_groups:
            dist.broadcast(g.p, src=0)
            dist.broadcast(g.mom, src=0)
            if self.shard_head and g.ema is not None:  # every rank keeps an EMA: start it from rank 0's
                dist.broadcast(g.ema, src=0)
        for b in self.model.buffers():
            dist.broadcast(b, src=0)
        if self.shard_head and self.ema is not None:
            for b in self.ema.buffers():
                dist.broadcast(b, src=0)
        self.opt._invalidate_packed()

    def state_dict(self) -> dict:
        """The trainer-side entries of the reference's checkpoint (engine/procedure/train.py:266-276): 'optimizer',
        'scheduler' (position in cosine_with_warm) and the EMA's 'updates'."""
        opt = self.opt.state_dict()
        if self.shard_head:
            opt = self._unsharded_optimizer_state(opt)
        return {"optimizer": opt, "scheduler": {"step": self.sched_step}, "updates": self.opt.updates}

    def load_state_dict(self, state: dict) -> None:
        opt = state["optimizer"]
        if self.shard_head:
            opt = self._sharded_optimizer_state(opt)
        self.opt.load_state_dict(opt)
        self.opt.updates = int(state.get("updates", self.opt.updates))
        self.sched_step = int(state["scheduler"]["step"])
        self._apply_lr()  # param_groups' lr follow the restored schedule position, not the saved (pre-step) value

    def _head_dims(self):
        head = self.model.trainingwrapper["head"]
        return head, head.weight.shape[0], head.num_class_total

    def _unsharded_optimizer_state(self, opt: dict) -> dict:
        """The sharded optimizer state in the unsharded trainer's layout: the head's momentum gathered to [D, C] (a collective)
        and, with layer_wise=False, the backbone and head groups joined into the single group the unsharded trainer has."""
        from .heads import gather_columns
        head, D, Cn = self._head_dims()
        mom = self.opt.groups[-1].mom.view(D, -1)
        bufs = opt["momentum_buffers"][:-1] + [gather_columns(head.comm, mom, Cn).reshape(-1).cpu()]
        pgs = opt["param_groups"]
        if not self.layer_wise:
            bufs, pgs = [torch.cat(bufs)], pgs[:1]
        return dict(opt, momentum_buffers=bufs, param_groups=pgs)

    def _sharded_optimizer_state(self, opt: dict) -> dict:
        """The inverse of _unsharded_optimizer_state: this rank's columns of the head's momentum."""
        from .heads import shard_columns
        head, D, Cn = self._head_dims()
        bufs, pgs = list(opt["momentum_buffers"]), [dict(pg) for pg in opt["param_groups"]]
        if not self.layer_wise:
            if len(bufs) != 1:
                raise ValueError("optimizer state has a different number of parameter groups")
            nb = self.opt.groups[0].n
            bufs, pgs = [bufs[0][:nb], bufs[0][nb:]], pgs * 2
        if bufs[-1].numel() != D * Cn:
            raise ValueError("optimizer state does not match the full head (different model?)")
        bufs[-1] = shard_columns(bufs[-1].reshape(D, Cn), head.comm.world, head.comm.rank).reshape(-1)
        return dict(opt, momentum_buffers=bufs, param_groups=pgs)

    def _apply_lr(self):
        for pg, base in zip(self.opt.param_groups, self.base_lrs):
            pg["lr"] = cosine_with_warm_lr(self.sched_step, base, self.lr0, self.warm, self.total, self.lrf)

    def set_momentum(self, momentum: float):  # vision_engine.py:545-546 switches warm-up momentum -> momentum
        for pg in self.opt.param_groups:
            pg["momentum"] = momentum

    # ---- DDP: gradient mean on the flat buffers, overlapped with the backward (what DistributedDataParallel's buckets do
    # in the reference, engine/vision_engine.py:509-510) ----
    def _flat_slice(self, names):
        """The slice of a flat gradient buffer that holds exactly the gradients of `names` (None if they do not form one
        contiguous run inside a single group: the caller then reduces whole buffers after the backward)."""
        params = dict(self.model.trainingwrapper["backbone"].named_parameters())
        ps = [params[n] for n in names if n in params]
        if not ps or any(p.grad is None for p in ps):
            return None
        for g in self.opt.groups:
            base, n_el = g.g.data_ptr(), g.g.numel()
            offs = [(p.grad.data_ptr() - base) // 4 for p in ps]
            if all(0 <= o < n_el for o in offs):
                lo = min(offs)
                hi = max(o + p.numel() for o, p in zip(offs, ps))
                if hi - lo <= sum(p.numel() for p in ps) + 64 * len(ps):  # contiguous up to alignment padding
                    return g, lo, hi
        return None

    @staticmethod
    def _all_reduce_mean(t: torch.Tensor, async_op: bool = False):
        """Gradient mean over the ranks: ReduceOp.AVG on NCCL (the product path); gloo (the test harness: two ranks sharing
        one GPU, or CPU tensors) has no AVG, so it sums synchronously and divides."""
        if dist.get_backend() == "nccl":
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, async_op=async_op)
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        t.div_(dist.get_world_size())
        return None

    def _on_section(self, names):
        sl = self._flat_slice(names)
        if sl is None:
            self._overlap_failed = True
            return
        g, lo, hi = sl
        work = self._all_reduce_mean(g.g[lo:hi], async_op=True)
        if work is not None:
            self._pending.append(work)
        self._reduced.append((id(g), lo, hi))

    def step(self, images: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """One batch: returns the (device) loss; does not synchronise (the reference's loss.item() every step,
        train.py:233, is a forced sync the hot path does not need)."""
        self.model.train()
        ddp = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        backbone = self.model.trainingwrapper["backbone"]
        self._pending, self._reduced, self._overlap_failed = [], [], False
        if ddp and hasattr(backbone, "backward_sections"):
            backbone.grad_section_hook = self._on_section
        loss = self.model.loss(images, labels, self.label_smooth)
        loss.backward()
        if ddp:
            backbone.grad_section_hook = None
            for w in self._pending:
                w.wait()  # the compute stream waits for the collectives (no host block)
            for g in self._ddp_groups:  # whatever the sections did not cover (the head group; gaps; a failed overlap)
                done = sorted((lo, hi) for gid, lo, hi in self._reduced if gid == id(g)) if not self._overlap_failed else []
                if self._overlap_failed and self._reduced:
                    raise RuntimeError("DDP overlap: gradient sections were not contiguous after some were already reduced")
                pos = 0
                for lo, hi in done + [(g.g.numel(), g.g.numel())]:
                    if lo > pos:
                        self._all_reduce_mean(g.g[pos:lo])
                    pos = max(pos, hi)
        self.opt.step()
        self.sched_step += 1  # scheduler.step() per batch (train.py:230)
        self._apply_lr()
        return loss.detach()


class DevicePrefetcher:
    """Host -> device staging for the loop `for images, labels in loader:` (engine/procedure/train.py:221-226, where the
    reference calls `.to(device, non_blocking=True)` on the compute stream, i.e. the copy and the step serialise).
    Batch i+1 is copied from pinned host memory on a side stream while batch i trains; the consumer stream waits on the
    copy's event, and a batch's device buffers are only reused once the step that read them has been enqueued."""

    def __init__(self, loader, device):
        self.loader = iter(loader)
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.next = None
        self._preload()

    def _preload(self):
        try:
            images, labels = next(self.loader)
        except StopIteration:
            self.next = None
            return
        with torch.cuda.stream(self.stream):
            x = images.to(self.device, non_blocking=True)
            y = labels.to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(self.stream)
        self.next = (x, y, ev)

    def __iter__(self):
        return self

    def __next__(self):
        if self.next is None:
            raise StopIteration
        x, y, ev = self.next
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        x.record_stream(cur)  # the caching allocator must not hand these buffers back to the copy stream early
        y.record_stream(cur)
        self._preload()
        return x, y

