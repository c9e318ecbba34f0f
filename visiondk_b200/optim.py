"""Optimizer half of the faceX train step on H100 (SURVEY.md §8b, Seam 4).

Reference: `Trainer.update(model, loss, scaler, optimizer, ema)` (engine/procedure/train.py:203-215) =
backward -> clip_grad_norm_(10) -> SGD step -> zero_grad -> ModelEMA.update, with param groups from
built/layer_optimizer.py:26-29 (backbone lr, head lr x10), SGD from engine/optimizer.py:119-133 and the EMA decay
ramp of models/ema.py:24.  FusedSGDClipEMA does everything after backward in two kernel sweeps per param group
(csrc/optim.cu) over flat fp32 buffers that the parameters and their .grad are re-pointed into.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib
from .wrapper import BackboneWrapper


class _FlatGroup:
    def __init__(self, params: List[nn.Parameter], lr: float):
        self.params, self.lr = params, lr
        dev = params[0].device
        n = sum(p.numel() for p in params)
        self.n = n
        self.p = torch.empty(n, dtype=torch.float32, device=dev)
        self.g = torch.zeros(n, dtype=torch.float32, device=dev)
        self.mom = torch.zeros(n, dtype=torch.float32, device=dev)
        self.ema: Optional[torch.Tensor] = None
        off = 0
        for q in params:  # re-point parameter storage and gradients into the flat buffers
            k = q.numel()
            self.p[off:off + k].copy_(q.data.reshape(-1))
            q.data = self.p[off:off + k].view_as(q)
            q.grad = self.g[off:off + k].view_as(q)
            off += k


class FusedSGDClipEMA:
    """SGD(momentum, weight_decay) + clip_grad_norm_ + zero_grad + EMA in one fused pass per param group.

    param_groups: list of {'params': iterable, 'lr': float} like SeperateLayerParams.create_ParamSequence.
    ema_model: a deepcopy of the model (ModelEMA.ema) whose floating state is updated in place; its parameters
    are re-pointed into flat buffers parallel to the model's.
    sharded_groups: indices of groups that hold a different shard of one tensor on every rank (the class-sharded head).
    clip_grad_norm_ then uses the global norm: their sum of squares is summed over the ranks (one fp64 scalar) before the
    replicated groups' is added.
    """

    def __init__(self, param_groups, lr: float, momentum: float, weight_decay: float, max_norm: float = 10.0,
                 model: Optional[nn.Module] = None, ema_model: Optional[nn.Module] = None, ema_decay: float = 0.9999,
                 ema_tau: float = 2000.0, sharded_groups: Sequence[int] = ()):
        lib = _lib.load()
        if isinstance(param_groups, (list, tuple)) and param_groups and isinstance(param_groups[0], dict):
            groups = [(list(g["params"]), float(g.get("lr", lr))) for g in param_groups]
        else:
            groups = [(list(param_groups), float(lr))]
        for ps, _ in groups:
            if any(p.device.type != "cuda" for p in ps):
                raise RuntimeError("FusedSGDClipEMA runs on CUDA (sm_90a) parameters only; there is no CPU fallback")
        self.groups = [_FlatGroup([p for p in ps if p.requires_grad], g_lr) for ps, g_lr in groups]
        self.param_groups = [{"lr": g.lr, "initial_lr": g.lr, "momentum": momentum, "weight_decay": weight_decay}
                             for g in self.groups]  # scheduler-facing view (torch LR schedulers mutate 'lr')
        self.max_norm = float(max_norm)
        self.sharded_groups = tuple(sharded_groups)
        self.steps = 0
        dev = self.groups[0].p.device
        self._sumsq = torch.zeros((), dtype=torch.float64, device=dev)
        self._ws = torch.empty((lib.vdk_grad_sumsq_workspace_bytes(),), dtype=torch.uint8, device=dev)
        self.ema_model, self.ema_decay, self.ema_tau, self.updates = ema_model, ema_decay, ema_tau, 0
        self.model = model
        self._buffers = []
        if ema_model is not None:
            assert model is not None, "pass the live model so EMA buffers can be paired by name"
            name_of = {id(p): n for n, p in model.named_parameters()}
            ema_params = dict(ema_model.named_parameters())
            for g in self.groups:
                g.ema = torch.empty_like(g.p)
                off = 0
                for q in g.params:
                    e = ema_params[name_of[id(q)]]
                    k = q.numel()
                    g.ema[off:off + k].copy_(e.data.reshape(-1))
                    e.data = g.ema[off:off + k].view_as(e)
                    off += k
            ema_bufs = dict(ema_model.named_buffers())
            for n, b in model.named_buffers():
                if b.dtype.is_floating_point:
                    self._buffers.append((ema_bufs[n], b))

    def decay(self, updates: int) -> float:
        return self.ema_decay * (1 - math.exp(-updates / self.ema_tau))  # models/ema.py:24

    @torch.no_grad()
    def step(self) -> None:
        """Everything Trainer.update does after backward (train.py:206-215)."""
        lib = _lib.load()
        s = _lib.stream_ptr()
        if self.sharded_groups:
            self._global_sumsq(lib, s)
        else:
            for i, g in enumerate(self.groups):
                _lib.check(lib.vdk_grad_sumsq(g.g.data_ptr(), g.n, self._sumsq.data_ptr(), int(i > 0), self._ws.data_ptr(),
                                              self._ws.numel(), s), "vdk_grad_sumsq")
        d, omd = -1.0, 0.0
        if self.ema_model is not None:
            self.updates += 1
            d = self.decay(self.updates)
            omd = 1 - d
        for g, pg in zip(self.groups, self.param_groups):
            _lib.check(lib.vdk_sgd_clip_ema_step(g.p.data_ptr(), g.g.data_ptr(), g.mom.data_ptr(),
                                                 g.ema.data_ptr() if g.ema is not None else 0, g.n,
                                                 self._sumsq.data_ptr(), self.max_norm, float(pg["lr"]),
                                                 float(pg["momentum"]), float(pg["weight_decay"]),
                                                 int(self.steps == 0), d, omd, 1, s), "vdk_sgd_clip_ema_step")
        for e, b in self._buffers:
            _lib.check(lib.vdk_ema_update(e.data_ptr(), b.data_ptr(), b.numel(), d, omd, s), "vdk_ema_update")
        self.steps += 1
        self._invalidate_packed()

    def _global_sumsq(self, lib, s) -> None:
        """Sum of squares of the whole model's gradient when some groups are sharded over the ranks: the shards' sums first,
        summed over the ranks, then the replicated groups' added on every rank."""
        from .sharding import all_reduce_sum_
        order = list(self.sharded_groups) + [i for i in range(len(self.groups)) if i not in self.sharded_groups]
        for j, i in enumerate(order):
            g = self.groups[i]
            _lib.check(lib.vdk_grad_sumsq(g.g.data_ptr(), g.n, self._sumsq.data_ptr(), int(j > 0), self._ws.data_ptr(),
                                          self._ws.numel(), s), "vdk_grad_sumsq")
            if j == len(self.sharded_groups) - 1:
                all_reduce_sum_(self._sumsq)

    def _invalidate_packed(self) -> None:
        """The kernels above write parameters, EMA parameters and EMA buffers through raw pointers, which does not bump
        torch's `_version` counters — the key every backbone wrapper's packed inference weights (`BackboneWrapper._pack`)
        are cached under.  Drop those caches explicitly so that the next `embed()` of the live model or of the EMA copy
        (the in-training eval, engine/procedure/train.py:244-262) re-packs the CURRENT weights."""
        for root in (self.model, self.ema_model):
            if root is None:
                continue
            for m in root.modules():
                if isinstance(m, BackboneWrapper):
                    m.invalidate_pack()

    def state_dict(self) -> dict:
        """What torch.optim.SGD.state_dict() carries for the reference's checkpoint (engine/procedure/train.py:273): the
        per-group hyper-parameters and the momentum buffers (one flat tensor per group), plus the step / EMA counters."""
        return {"steps": self.steps, "updates": self.updates, "param_groups": [dict(pg) for pg in self.param_groups],
                "momentum_buffers": [g.mom.detach().cpu().clone() for g in self.groups]}

    def load_state_dict(self, state: dict) -> None:
        if len(state["momentum_buffers"]) != len(self.groups):
            raise ValueError("optimizer state has a different number of parameter groups")
        for g, m in zip(self.groups, state["momentum_buffers"]):
            if m.numel() != g.n:
                raise ValueError("optimizer state does not match the parameter groups (different model?)")
            g.mom.copy_(m.to(g.mom.device))
        for pg, saved in zip(self.param_groups, state["param_groups"]):
            pg.update(saved)
        self.steps, self.updates = int(state["steps"]), int(state["updates"])
        self._invalidate_packed()

    def grad_norm(self) -> float:
        return float(self._sumsq.sqrt().item())

    def zero_grad(self) -> None:  # gradients are zeroed inside step(); kept for surface compatibility
        return None
