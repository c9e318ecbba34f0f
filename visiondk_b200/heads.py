"""Head seam of the faceX train step on H100 (SURVEY.md §8b, Seam 2 and Seam 4).

`HeadFactory(model_cfg['head']).get_head()` (models/faceX/head/head_def.py:14-56) returns an nn.Module with
`.weight: Parameter[feat_dim, num_class]` and `forward(feats[B,D], labels[B]) -> logits[B,C]`.  ArcFace and
CircleLoss here keep that surface and parameter initialisation (arcface.py:11-12) while the arithmetic — both
normalisations, the cos(theta) contraction on wgmma, the margin, and (in the fused form the trainer uses) the
cross-entropy with label smoothing and the whole backward — is csrc/heads.cu.

`margin_ce_loss(head, feats, labels, label_smooth)` is criterion∘head fused: the two are only ever called
together (engine/procedure/train.py:196), so the caller never holds a [B,C] logits tensor or its autograd graph.  Inside the
kernels the cosines and the two gradient factors still live in a caller-owned fp32 workspace of 3 x B x C floats (113 MB at the
reference's face config, B = 160, C = 58 671, configs/faceX/face.yaml:34,42 — tested at that size in tests/test_heads_gpu.py).

`ShardedHead` splits the classes over the ranks for million-class problems: rank r holds the columns
`sharding.shard_bounds(C, W, r)` of `weight [D, C]` and never exchanges them.  Per step the ranks exchange the features
and labels (all-gather, W·B rows), the label cosines (MV-Softmax), four floats per row to combine the softmax, and the
partial feature gradients (sum); the loss, both gradients and the trained weights equal the unsharded DDP step's.
`sharded_head_forward` / `sharded_head_backward` are the step as explicit calls; `sharded_margin_ce_loss` wraps them in
an autograd node.  The workspace is still [W·B, C/W]: a streaming softmax that avoids it is not built.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from .sharding import DistComm, shard_bounds

HEAD_ARCFACE, HEAD_CIRCLELOSS, HEAD_MV_SOFTMAX = 0, 1, 2


def _desc(head, batch: int, label_smooth: float) -> _lib.HeadDesc:
    d = _lib.HeadDesc()
    d.kind = head.kind
    d.batch, d.feat_dim, d.num_class = batch, head.weight.shape[0], head.weight.shape[1]
    d.margin_arc = float(getattr(head, "margin_arc", 0.0))
    d.margin_am = float(getattr(head, "margin_am", 0.0))
    d.scale = float(getattr(head, "scale", 1.0))
    d.margin = float(getattr(head, "margin", 0.0))
    d.gamma = float(getattr(head, "gamma", 1.0))
    d.label_smooth = float(label_smooth)
    d.mv_weight = float(getattr(head, "mv_weight", 1.0))
    d.is_am = int(bool(getattr(head, "is_am", False)))
    return d


def _workspace(desc, device):
    lib = _lib.load()
    n = lib.vdk_head_workspace_bytes(C.byref(desc))
    return torch.empty((n,), dtype=torch.uint8, device=device)


def _check_inputs(feats, weight, labels):
    if feats.device.type != "cuda":
        raise RuntimeError("visiondk_b200 heads run on CUDA (sm_90a) only; there is no CPU fallback")
    if feats.dim() != 2 or feats.shape[1] != weight.shape[0]:
        raise ValueError(f"feats must be [B, {weight.shape[0]}], got {tuple(feats.shape)}")
    if labels.shape != (feats.shape[0],):
        raise ValueError("labels must be [B]")


def _check_backward(feats):
    if feats.shape[1] % 8:
        raise ValueError(f"the head backward needs feat_dim to be a multiple of 8, got {feats.shape[1]} (the forward has no such "
                         f"restriction)")


class _HeadLogits(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, weight, labels, head):
        lib = _lib.load()
        _check_inputs(feats, weight, labels)
        feats, weight, labels = feats.contiguous().float(), weight.contiguous().float(), labels.contiguous().long()
        B = feats.shape[0]
        desc = _desc(head, B, 0.0)
        ws = _workspace(desc, feats.device)
        logits = torch.empty((B, weight.shape[1]), dtype=torch.float32, device=feats.device)
        loss = torch.empty((), dtype=torch.float32, device=feats.device)
        lse = torch.empty((B,), dtype=torch.float32, device=feats.device)
        with torch.cuda.device(feats.device):
            _lib.check(lib.vdk_head_forward(C.byref(desc), feats.data_ptr(), weight.data_ptr(), labels.data_ptr(),
                                            logits.data_ptr(), loss.data_ptr(), lse.data_ptr(), 0, ws.data_ptr(), ws.numel(),
                                            _lib.stream_ptr()), "vdk_head_forward")
        ctx.save_for_backward(feats, weight, labels)
        ctx.head, ctx.ws = head, ws
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        lib = _lib.load()
        feats, weight, labels = ctx.saved_tensors
        _check_backward(feats)
        desc = _desc(ctx.head, feats.shape[0], 0.0)
        dlogits = dlogits.contiguous().float()
        df, dw = torch.empty_like(feats), torch.empty_like(weight)
        with torch.cuda.device(feats.device):
            _lib.check(lib.vdk_head_backward(C.byref(desc), feats.data_ptr(), weight.data_ptr(), labels.data_ptr(), 0, 0,
                                             dlogits.data_ptr(), df.data_ptr(), dw.data_ptr(), ctx.ws.data_ptr(),
                                             ctx.ws.numel(), _lib.stream_ptr()), "vdk_head_backward")
        return df, dw, None, None


class _HeadCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, weight, labels, head, label_smooth):
        lib = _lib.load()
        _check_inputs(feats, weight, labels)
        feats, weight, labels = feats.contiguous().float(), weight.contiguous().float(), labels.contiguous().long()
        B = feats.shape[0]
        desc = _desc(head, B, label_smooth)
        ws = _workspace(desc, feats.device)
        loss = torch.empty((), dtype=torch.float32, device=feats.device)
        lse = torch.empty((B,), dtype=torch.float32, device=feats.device)
        with torch.cuda.device(feats.device):
            _lib.check(lib.vdk_head_forward(C.byref(desc), feats.data_ptr(), weight.data_ptr(), labels.data_ptr(), 0,
                                            loss.data_ptr(), lse.data_ptr(), 0, ws.data_ptr(), ws.numel(),
                                            _lib.stream_ptr()), "vdk_head_forward")
        ctx.save_for_backward(feats, weight, labels, lse)
        ctx.head, ctx.ws, ctx.label_smooth = head, ws, label_smooth
        return loss

    @staticmethod
    def backward(ctx, gout):
        lib = _lib.load()
        feats, weight, labels, lse = ctx.saved_tensors
        _check_backward(feats)
        desc = _desc(ctx.head, feats.shape[0], ctx.label_smooth)
        gout = gout.contiguous().float()
        df, dw = torch.empty_like(feats), torch.empty_like(weight)
        with torch.cuda.device(feats.device):
            _lib.check(lib.vdk_head_backward(C.byref(desc), feats.data_ptr(), weight.data_ptr(), labels.data_ptr(),
                                             lse.data_ptr(), gout.data_ptr(), 0, df.data_ptr(), dw.data_ptr(),
                                             ctx.ws.data_ptr(), ctx.ws.numel(), _lib.stream_ptr()), "vdk_head_backward")
        return df, dw, None, None, None


class _MarginHead(nn.Module):
    kind = -1

    def __init__(self, feat_dim: int, num_class: int):
        super().__init__()
        # arcface.py:11-12 / circleloss.py:11-12: uniform(-1,1) renormed to unit columns
        self.weight = nn.Parameter(torch.empty(feat_dim, num_class))
        self.weight.data.uniform_(-1, 1).renorm_(2, 1, 1e-5).mul_(1e5)

    def forward(self, feats: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        return _HeadLogits.apply(feats, self.weight, labels, self)


class ArcFace(_MarginHead):
    """models/faceX/head/arcface.py:6-36."""
    kind = HEAD_ARCFACE

    def __init__(self, feat_dim, num_class, margin_arc=0.35, margin_am=0.0, scale=32):
        super().__init__(feat_dim, num_class)
        self.margin_arc, self.margin_am, self.scale = margin_arc, margin_am, scale


class CircleLoss(_MarginHead):
    """models/faceX/head/circleloss.py:5-43."""
    kind = HEAD_CIRCLELOSS

    def __init__(self, feat_dim, num_class, margin=0.25, gamma=256):
        super().__init__(feat_dim, num_class)
        self.margin, self.gamma = margin, gamma


class MV_Softmax(_MarginHead):
    """models/faceX/head/mv_softmax.py:9-44 (same constructor; hard negatives re-weighted by mv_weight)."""
    kind = HEAD_MV_SOFTMAX

    def __init__(self, feat_dim, num_class, is_am, margin=0.35, mv_weight=1.12, scale=32):
        super().__init__(feat_dim, num_class)
        self.is_am, self.margin, self.mv_weight, self.scale = bool(is_am), margin, mv_weight, scale


def margin_ce_loss(head: _MarginHead, feats: torch.Tensor, labels: torch.Tensor, label_smooth: float = 0.0) -> torch.Tensor:
    """Fused criterion(head(feats, labels), labels) with criterion = CrossEntropyLoss(label_smoothing)."""
    return _HeadCE.apply(feats, head.weight, labels, head, float(label_smooth))


class HeadFactory:
    """models/faceX/head/head_def.py:7-56 (arcface, circleloss and mv-softmax are built)."""

    def __init__(self, head_config: dict):
        for k, v in head_config.items():
            self.head_type, self.head_param = k, v

    def get_head(self) -> nn.Module:
        p = self.head_param
        if self.head_type == "arcface":
            return ArcFace(p["feat_dim"], p["num_class"], p["margin_arc"], p["margin_am"], p["scale"])
        if self.head_type == "circleloss":
            return CircleLoss(p["feat_dim"], p["num_class"], p["margin"], p["gamma"])
        if self.head_type == "mv-softmax":
            return MV_Softmax(p["feat_dim"], p["num_class"], p["is_am"], p["margin"], p["mv_weight"], p["scale"])
        raise NotImplementedError(f"head '{self.head_type}': arcface, circleloss and mv-softmax are built for H100; magface returns "
                                  f"a (logits, loss) tuple the reference's own train loop cannot consume (magface.py:47 vs train.py:196)")


# ---- class-sharded head ------------------------------------------------------------------------------------------------------

_HYPER = ("margin_arc", "margin_am", "scale", "margin", "gamma", "mv_weight", "is_am")


def shard_columns(full: torch.Tensor, world: int, rank: int) -> torch.Tensor:
    """Rank `rank`'s columns of a full [D, C] head tensor."""
    lo, hi = shard_bounds(full.shape[1], world, rank)
    return full[:, lo:hi]


def gather_columns(comm, local: torch.Tensor, num_class: int) -> torch.Tensor:
    """Every rank's column shard [D, C_r] -> the full [D, C] on every rank (a collective: every rank must call it)."""
    world = comm.world
    widest = max(shard_bounds(num_class, world, r)[1] - shard_bounds(num_class, world, r)[0] for r in range(world))
    padded = local.new_zeros((local.shape[0], widest))
    padded[:, :local.shape[1]] = local
    parts = comm.all_gather(padded)
    return torch.cat([parts[r, :, :hi - lo] for r, (lo, hi) in
                      enumerate(shard_bounds(num_class, world, r) for r in range(world))], dim=1)


class ShardedHead(nn.Module):
    """The columns [class_offset, class_offset + C/W) of a margin head, on one of W ranks (`comm`: sharding.DistComm, or
    a sharding.LocalShardGroup shard in tests).  `weight [D, C_hi - C_lo]` is the trained Parameter.  `state_dict()` gathers
    the full `weight [D, C]` of the unsharded head (a collective: every rank must call it) and `load_state_dict` takes a full
    weight and keeps this rank's columns, so checkpoints are interchangeable with the unsharded head's."""

    def __init__(self, head: _MarginHead, comm=None):
        super().__init__()
        self.comm = comm if comm is not None else DistComm()
        self.kind = head.kind
        for a in _HYPER:
            if hasattr(head, a):
                setattr(self, a, getattr(head, a))
        self.num_class_total = head.weight.shape[1]
        self.class_offset, hi = shard_bounds(self.num_class_total, self.comm.world, self.comm.rank)
        self.weight = nn.Parameter(head.weight.detach()[:, self.class_offset:hi].clone())

    def forward(self, feats, labels):
        raise NotImplementedError("the class-sharded head computes the fused loss only (sharded_margin_ce_loss): logits "
                                  "[B, C] would need every rank's columns")

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        destination[prefix + "weight"] = gather_columns(self.comm, self.weight.detach(), self.num_class_total)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        key = prefix + "weight"
        if key not in state_dict:
            missing_keys.append(key)
            return
        full = state_dict[key]
        want = (self.weight.shape[0], self.num_class_total)
        if tuple(full.shape) != want:
            error_msgs.append(f"size mismatch for {key}: the checkpoint holds {tuple(full.shape)}, the full head is {want}")
            return
        with torch.no_grad():  # in place: the parameter may live in the optimizer's flat buffer
            self.weight.copy_(shard_columns(full, self.comm.world, self.comm.rank))


def _shard_desc(head: ShardedHead) -> _lib.HeadShard:
    s = _lib.HeadShard()
    s.class_offset, s.num_class_total = head.class_offset, head.num_class_total
    s.world, s.rank = head.comm.world, head.comm.rank
    return s


def sharded_head_forward(head: ShardedHead, feats: torch.Tensor, labels: torch.Tensor, label_smooth: float = 0.0,
                         outputs: Optional[dict] = None):
    """This rank's mean CE over its own B rows, computed with every rank (a collective).  Returns (loss, saved) where `saved`
    feeds sharded_head_backward.  `outputs` may hold preallocated tensors to write into: 'logits' and 'cos' ([W·B, C_r]
    of this shard), 'row_lse', 'row_loss' ([W·B]) and 'loss' (scalar)."""
    lib, comm = _lib.load(), head.comm
    _check_inputs(feats, head.weight, labels)
    feats, labels = feats.contiguous().float(), labels.contiguous().long()
    dev, B = feats.device, feats.shape[0]
    out = dict(outputs or {})
    sizes = comm.all_gather(torch.tensor([B], dtype=torch.int64, device=dev))
    if not bool((sizes == B).all()):
        raise ValueError(f"the class-sharded head needs the same batch on every rank, got {sizes.flatten().tolist()}")
    f_all = comm.all_gather(feats).reshape(comm.world * B, feats.shape[1])
    y_all = comm.all_gather(labels).reshape(comm.world * B)
    n = f_all.shape[0]
    desc, shard = _desc(head, n, label_smooth), _shard_desc(head)
    ws = _workspace(desc, dev)
    gt = torch.empty((n,), dtype=torch.float32, device=dev)
    partials = torch.empty((n, 4), dtype=torch.float32, device=dev)
    for k, shape in (("row_lse", (n,)), ("row_loss", (n,)), ("loss", ())):
        if out.get(k) is None:
            out[k] = torch.empty(shape, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.vdk_head_shard_cos(C.byref(desc), C.byref(shard), f_all.data_ptr(), head.weight.data_ptr(),
                                          y_all.data_ptr(), gt.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()),
                   "vdk_head_shard_cos")
        if head.kind == HEAD_MV_SOFTMAX:  # every element needs its row's label cosine, held by one rank
            comm.all_reduce_sum_(gt)
        _lib.check(lib.vdk_head_shard_forward(C.byref(desc), C.byref(shard), y_all.data_ptr(), gt.data_ptr(),
                                              _lib.ptr(out.get("logits")), _lib.ptr(out.get("cos")), partials.data_ptr(),
                                              ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_head_shard_forward")
        parts = comm.all_gather(partials)
        _lib.check(lib.vdk_head_shard_combine(C.byref(desc), C.byref(shard), parts.data_ptr(), out["row_lse"].data_ptr(),
                                              out["row_loss"].data_ptr(), out["loss"].data_ptr(), _lib.stream_ptr()),
                   "vdk_head_shard_combine")
    saved = dict(feats=f_all, labels=y_all, label_cos=gt, row_lse=out["row_lse"], ws=ws, label_smooth=float(label_smooth),
                 batch=B)
    return out["loss"], saved


def sharded_head_backward(head: ShardedHead, saved: dict, grad_loss: Optional[torch.Tensor] = None,
                          outputs: Optional[dict] = None):
    """(dfeats [B, D] of this rank's rows, dweight [D, C_r]) for `saved` of sharded_head_forward (a collective).  dfeats is
    the gradient of this rank's loss; dweight the gradient of the mean of the W ranks' losses (what the DDP average of the
    unsharded head's gradient holds in these columns).  `outputs` may hold preallocated 'dfeats' and 'dweight'."""
    lib, comm = _lib.load(), head.comm
    f_all = saved["feats"]
    _check_backward(f_all)
    dev, n, D = f_all.device, f_all.shape[0], f_all.shape[1]
    out = dict(outputs or {})
    if out.get("dweight") is None:
        out["dweight"] = torch.empty_like(head.weight)
    if out.get("dfeats") is None:
        out["dfeats"] = torch.empty((saved["batch"], D), dtype=torch.float32, device=dev)
    desc, shard = _desc(head, n, saved["label_smooth"]), _shard_desc(head)
    ws = saved["ws"]
    dfn = torch.empty((n, D), dtype=torch.float32, device=dev)
    gout = grad_loss.contiguous().float() if grad_loss is not None else None
    with torch.cuda.device(dev):
        _lib.check(lib.vdk_head_shard_backward(C.byref(desc), C.byref(shard), f_all.data_ptr(), head.weight.data_ptr(),
                                               saved["labels"].data_ptr(), saved["label_cos"].data_ptr(),
                                               saved["row_lse"].data_ptr(), _lib.ptr(gout), dfn.data_ptr(),
                                               out["dweight"].data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()),
                   "vdk_head_shard_backward")
        comm.all_reduce_sum_(dfn)
        _lib.check(lib.vdk_head_shard_finalize(C.byref(desc), C.byref(shard), dfn.data_ptr(), out["dfeats"].data_ptr(),
                                               ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_head_shard_finalize")
    return out["dfeats"], out["dweight"]


class _ShardedHeadCE(torch.autograd.Function):
    """Autograd node of the sharded step.  Its backward runs collectives, so every rank must be its own process: the autograd
    engine runs CUDA backward nodes on one worker thread per device, which would serialise LocalShardGroup's threads."""

    @staticmethod
    def forward(ctx, feats, weight, labels, head, label_smooth):
        loss, ctx.saved = sharded_head_forward(head, feats, labels, label_smooth)
        ctx.head = head
        return loss

    @staticmethod
    def backward(ctx, gout):
        df, dw = sharded_head_backward(ctx.head, ctx.saved, gout)
        ctx.saved = None
        return df, dw, None, None, None


def sharded_margin_ce_loss(head: ShardedHead, feats: torch.Tensor, labels: torch.Tensor,
                           label_smooth: float = 0.0) -> torch.Tensor:
    """margin_ce_loss for a ShardedHead: this rank's mean CE over its own rows (a collective in forward and backward)."""
    return _ShardedHeadCE.apply(feats, head.weight, labels, head, float(label_smooth))
