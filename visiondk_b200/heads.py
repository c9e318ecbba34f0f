"""Head seam of the faceX train step on H100 (SURVEY.md §8b, Seam 2 and Seam 4).

`HeadFactory(model_cfg['head']).get_head()` (models/faceX/head/head_def.py:14-56) returns an nn.Module with
`.weight: Parameter[feat_dim, num_class]` and `forward(feats[B,D], labels[B]) -> logits[B,C]`.  ArcFace and
CircleLoss here keep that surface and parameter initialisation (arcface.py:11-12) while the arithmetic — both
normalisations, the cos(theta) contraction on wgmma, the margin, and (in the fused form the trainer uses) the
cross-entropy with label smoothing and the whole backward — is csrc/heads.cu.

`margin_ce_loss(head, feats, labels, label_smooth)` is criterion∘head fused: the two are only ever called
together (engine/procedure/train.py:196), so the caller never holds a [B,C] logits tensor or its autograd graph.  Inside the
kernels the cosines and the two gradient factors still live in a caller-owned fp32 workspace of 3 x B x C floats (113 MB at the
reference's face config, B = 160, C = 58 671, configs/faceX/face.yaml:34,42 — tested at that size in tests/test_heads_gpu.py);
a class-sharded / streaming-softmax head for million-class problems is not built.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib

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
