"""Swin Transformer V2 backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 SwinTransformerV2).

`SwinV2Wrapper` is the reference's TimmWrapper for a `timm-swinv2_*` backbone (models/faceX/backbone/timm_wrapper.py:16-54):
the timm SwinTransformerV2 built with num_classes=0, global_pool='' under `model.`, and the neck the wrapper's rank rule
builds for it.  timm 0.9's Swin returns an NHWC [B, 8, 8, C] map, a 4-D tensor, so the wrapper takes its CNN branch with
channels = shape[1] = 8: `output_layer.{0: BatchNorm2d(8) over the h axis, 1: Flatten in (h, w, c) order, 2: Linear(64 C),
3: BatchNorm1d}`.  Parameter names and shapes are timm's, so timm checkpoints load with strict=True.  The arithmetic is
csrc/swin.cu (vdk_swinv2_forward): the Linears on the wgmma GEMM, the shifted-window attention in one fused kernel.
Extraction only: a train-mode forward raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from .wrapper import BackboneWrapper, cnn_neck, fold_neck

IMAGE_SIZE = 256  # both towers' default img_size; timm_wrapper.py passes none to create_model
HEAD_DIM = 32
# timm 0.9.16 swin_transformer_v2.py model_args
SWINV2_ARCHS = {
    "swinv2_base_window8_256": dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=8,
                                    pretrained_window_sizes=(0, 0, 0, 0)),
    "swinv2_large_window12to16_192to256": dict(embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window_size=16,
                                               pretrained_window_sizes=(12, 12, 12, 6)),
}


def stage_windows(window_size: int, image_size: int = IMAGE_SIZE):
    """timm's SwinTransformerV2Block._calc_window_shift per stage: [(w, shift of the odd blocks)] with w = min(window, map) and
    shift w / 2, or 0 when the map is one window."""
    out = []
    for i in range(4):
        r = (image_size // 4) >> i
        w = min(r, window_size)
        out.append((w, 0 if r <= w else w // 2))
    return out


def relative_coords_table(w: int, pretrained_w: int) -> torch.Tensor:
    """timm WindowAttention's log-spaced relative_coords_table, [(2w-1)^2, 2] fp32, rows in (dy, dx) order."""
    c = torch.arange(-(w - 1), w, dtype=torch.float32)
    t = torch.stack(torch.meshgrid(c, c, indexing="ij"), dim=-1)
    t = t / (pretrained_w - 1 if pretrained_w > 0 else w - 1) * 8
    return (torch.sign(t) * torch.log2(t.abs() + 1.0) / math.log2(8)).reshape(-1, 2)


class _WindowAttention(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.logit_scale = nn.Parameter(torch.log(10 * torch.ones(heads, 1, 1)))
        self.cpb_mlp = nn.Sequential(nn.Linear(2, 512), nn.ReLU(inplace=True), nn.Linear(512, heads, bias=False))
        self.qkv = nn.Linear(dim, 3 * dim, bias=False)
        self.q_bias = nn.Parameter(torch.zeros(dim))
        self.v_bias = nn.Parameter(torch.zeros(dim))
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(dim, 4 * dim), nn.Linear(4 * dim, dim)


class _Block(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.attn = _WindowAttention(dim, heads)
        self.norm1 = nn.LayerNorm(dim)
        self.mlp = _Mlp(dim)
        self.norm2 = nn.LayerNorm(dim)


class _PatchMerging(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(2 * dim)


class _Stage(nn.Module):
    def __init__(self, dim, depth, heads, downsample):
        super().__init__()
        self.downsample = _PatchMerging(dim // 2) if downsample else nn.Identity()
        self.blocks = nn.ModuleList([_Block(dim, heads) for _ in range(depth)])


class _PatchEmbed(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.proj = nn.Conv2d(3, dim, 4, 4)
        self.norm = nn.LayerNorm(dim)


class SwinV2Params(nn.Module):
    """timm 0.9.16 `SwinTransformerV2(num_classes=0, global_pool='')` parameter tree.  Parameter containers only: their
    forward() is never used (the forward is vdk_swinv2_forward)."""

    def __init__(self, embed_dim, depths, num_heads, window_size, pretrained_window_sizes):
        super().__init__()
        self.embed_dim, self.depths, self.num_heads = int(embed_dim), tuple(depths), tuple(num_heads)
        self.window_size, self.pretrained_window_sizes = int(window_size), tuple(pretrained_window_sizes)
        self.patch_embed = _PatchEmbed(embed_dim)
        self.layers = nn.Sequential(*[_Stage(embed_dim << i, d, h, i > 0) for i, (d, h) in enumerate(zip(depths, num_heads))])
        self.norm = nn.LayerNorm(embed_dim << 3)
        # timm's init: trunc_normal(std .02) Linear weights, zero Linear biases, then every block's norm1 / norm2 zeroed
        # (_init_respostnorm)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        for blk in self.blocks():
            for n in (blk.norm1, blk.norm2):
                nn.init.zeros_(n.weight)
                nn.init.zeros_(n.bias)

    def blocks(self):
        return [b for stage in self.layers for b in stage.blocks]


class _SwinV2BlockC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("qkv_w", "qkv_b", "attn_scale", "attn_bias", "proj_w", "proj_b", "norm1_w", "norm1_b",
                                          "fc1_w", "fc1_b", "fc2_w", "fc2_b", "norm2_w", "norm2_b")]


MAX_BLOCKS = 24


class SwinV2NetC(C.Structure):
    """vdk_swinv2_net (include/vdk_b200.h)."""
    api = "vdk_swinv2"
    _fields_ = [
        ("image_size", C.c_int), ("feat_dim", C.c_int), ("embed_dim", C.c_int), ("depths", C.c_int * 4), ("window", C.c_int * 4),
        ("shift", C.c_int * 4), ("stem_w", C.c_void_p), ("stem_b", C.c_void_p), ("stem_ln_w", C.c_void_p),
        ("stem_ln_b", C.c_void_p), ("merge_w", C.c_void_p * 4), ("merge_ln_w", C.c_void_p * 4), ("merge_ln_b", C.c_void_p * 4),
        ("blocks", _SwinV2BlockC * MAX_BLOCKS), ("norm_w", C.c_void_p), ("norm_b", C.c_void_p), ("neck_w", C.c_void_p),
        ("neck_b", C.c_void_p),
    ]


def merge_weight_khkw(w: torch.Tensor) -> torch.Tensor:
    """timm's PatchMerging reduction weight [2C, 4C], K order (w-offset, h-offset, c), as the 2x2/s2 conv weight
    [2C, kh, kw, C] that vdk_conv2d contracts in (kh, kw, c) order."""
    cout, c = w.shape[0], w.shape[1] // 4
    return w.reshape(cout, 2, 2, c).permute(0, 2, 1, 3)


def fold_nhwc_neck(output_layer: nn.Sequential, h: int, wc: int, feat_dim: int, device):
    """The neck BatchNorm2d(h) over the h axis of an NHWC map -> Flatten in (h, w, c) order -> Linear -> BatchNorm1d (eval
    statistics) as one Linear over the (h, w, c) features: (weight [feat_dim, h * wc], bias [feat_dim]) in fp64."""
    w, bias = fold_neck(output_layer, device)
    return w.reshape(feat_dim, h * wc), bias


class SwinV2Wrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm Swin V2 backbone (eval / extract only)."""

    _dropped = ("head.fc.",)
    _rebuilt = ("relative_position_index", "relative_coords_table", "attn_mask")  # as timm's own checkpoint filter does

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, **kwargs):
        if model_name not in SWINV2_ARCHS:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; Swin V2 towers available: {sorted(SWINV2_ARCHS)}")
        if image_size != IMAGE_SIZE:
            raise ValueError(f"{model_name}: timm builds this tower at {IMAGE_SIZE}x{IMAGE_SIZE} (timm_wrapper.py passes no "
                             f"img_size), so image_size must be {IMAGE_SIZE} (got {image_size})")
        args = dict(SWINV2_ARCHS[model_name])
        if depths is not None:
            args["depths"] = tuple(depths)
        c_last, hw = args["embed_dim"] * 8, image_size // 32
        super().__init__(model_name, feat_dim, image_size, SwinV2Params(**args), cnn_neck(hw, hw * hw * c_last, feat_dim),
                         pretrained)

    def _build(self, p) -> SwinV2NetC:
        """Kernel-side layouts (include/vdk_b200.h), once per weight version: bf16 Linear weights, the qkv bias
        cat(q_bias, 0, v_bias), the clamped logit scales and 16 sigmoid(cpb_mlp(table)) bias tables in fp32, the merge weights
        in (kh, kw, c) order, the folded neck."""
        m = self.model
        if sum(m.depths) > MAX_BLOCKS:
            raise ValueError(f"{self.model_name}: at most {MAX_BLOCKS} blocks")
        net = SwinV2NetC()
        net.image_size, net.feat_dim, net.embed_dim = self.image_size, self.feat_dim, m.embed_dim
        windows = stage_windows(m.window_size, self.image_size)
        pe = m.patch_embed
        net.stem_w, net.stem_b = p.bf16(pe.proj.weight.reshape(m.embed_dim, 48)), p.f32(pe.proj.bias)
        net.stem_ln_w, net.stem_ln_b = p.f32(pe.norm.weight), p.f32(pe.norm.bias)
        blk = 0
        for i, stage in enumerate(m.layers):
            w, shift = windows[i]
            net.depths[i], net.window[i], net.shift[i] = m.depths[i], w, shift
            if i > 0:
                ds = stage.downsample
                net.merge_w[i] = p.bf16(merge_weight_khkw(ds.reduction.weight))
                net.merge_ln_w[i], net.merge_ln_b[i] = p.f32(ds.norm.weight), p.f32(ds.norm.bias)
            table = relative_coords_table(w, m.pretrained_window_sizes[i])
            for b in stage.blocks:
                dst, a = net.blocks[blk], b.attn
                blk += 1
                dst.qkv_w = p.bf16(a.qkv.weight)
                dst.qkv_b = p.f32(torch.cat([a.q_bias, torch.zeros_like(a.q_bias), a.v_bias]))
                dst.attn_scale = p.f32(torch.clamp(a.logit_scale, max=math.log(100.0)).exp().reshape(-1))
                dst.attn_bias = p.f32((16 * torch.sigmoid(a.cpb_mlp(table.to(a.logit_scale.device)))).t())
                dst.proj_w, dst.proj_b = p.bf16(a.proj.weight), p.f32(a.proj.bias)
                dst.norm1_w, dst.norm1_b = p.f32(b.norm1.weight), p.f32(b.norm1.bias)
                dst.fc1_w, dst.fc1_b = p.bf16(b.mlp.fc1.weight), p.f32(b.mlp.fc1.bias)
                dst.fc2_w, dst.fc2_b = p.bf16(b.mlp.fc2.weight), p.f32(b.mlp.fc2.bias)
                dst.norm2_w, dst.norm2_b = p.f32(b.norm2.weight), p.f32(b.norm2.bias)
        net.norm_w, net.norm_b = p.f32(m.norm.weight), p.f32(m.norm.bias)
        hw, c_last = self.image_size // 32, m.embed_dim * 8
        w, bias = fold_nhwc_neck(self.output_layer, hw, hw * c_last, self.feat_dim, p.device)
        net.neck_w, net.neck_b = p.bf16(w), p.f32(bias)
        return net
