"""fp32 oracle of timm 0.9.16's SwinTransformerV2 (swin_transformer_v2.py) with timm's state_dict keys, and the reference
TimmWrapper's neck rule around it (models/faceX/backbone/timm_wrapper.py:16-54).

The shifted-window attention is the literal form: torch.roll, window_partition / window_reverse, timm's slice-built attn_mask
and the log-spaced CPB coordinate table gathered by relative_position_index, so the kernel's index arithmetic is checked
against it.  timm itself is not installed: these hyperparameters and keys come from timm 0.9.16's source (unverified at
the timm boundary); tests/test_oracle_swinv2_cpu.py pins the oracle against HF transformers' Swinv2Model and torchvision's
SwinTransformer V2."""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

ARCHS = {
    "swinv2_base_window8_256": dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=8,
                                    pretrained_window_sizes=(0, 0, 0, 0)),
    "swinv2_large_window12to16_192to256": dict(embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window_size=16,
                                               pretrained_window_sizes=(12, 12, 12, 6)),
}


def window_partition(x, w):
    """[B, H, W, C] -> [B * H/w * W/w, w, w, C]"""
    B, H, W, C = x.shape
    return x.view(B, H // w, w, W // w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, w, w, C)


def window_reverse(windows, w, H, W):
    C = windows.shape[-1]
    return windows.view(-1, H // w, W // w, w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, H, W, C)


def attention_mask(H, W, w, s):
    """timm's attn_mask [nW, w*w, w*w]: 0 within a shift region, -100 across regions (slices (0:-w), (-w:-s), (-s:))."""
    img = torch.zeros(1, H, W, 1)
    cnt = 0
    for hs in (slice(0, -w), slice(-w, -s), slice(-s, None)):
        for ws in (slice(0, -w), slice(-w, -s), slice(-s, None)):
            img[:, hs, ws, :] = cnt
            cnt += 1
    mw = window_partition(img, w).view(-1, w * w)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def coords_table(w, pretrained_w):
    c = torch.arange(-(w - 1), w, dtype=torch.float32)
    t = torch.stack(torch.meshgrid([c, c], indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    d = (pretrained_w - 1) if pretrained_w > 0 else (w - 1)
    t[:, :, :, 0] /= d
    t[:, :, :, 1] /= d
    t *= 8
    return torch.sign(t) * torch.log2(torch.abs(t) + 1.0) / math.log2(8)


def position_index(w):
    coords = torch.stack(torch.meshgrid([torch.arange(w), torch.arange(w)], indexing="ij"))
    cf = torch.flatten(coords, 1)
    rel = (cf[:, :, None] - cf[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += w - 1
    rel[:, :, 1] += w - 1
    rel[:, :, 0] *= 2 * w - 1
    return rel.sum(-1)


class WindowAttention(nn.Module):
    def __init__(self, dim, window, heads, pretrained_window):
        super().__init__()
        self.window, self.heads = window, heads
        self.logit_scale = nn.Parameter(torch.log(10 * torch.ones(heads, 1, 1)))
        self.cpb_mlp = nn.Sequential(nn.Linear(2, 512), nn.ReLU(inplace=True), nn.Linear(512, heads, bias=False))
        self.register_buffer("relative_coords_table", coords_table(window, pretrained_window), persistent=False)
        self.register_buffer("relative_position_index", position_index(window), persistent=False)
        self.qkv = nn.Linear(dim, 3 * dim, bias=False)
        self.q_bias = nn.Parameter(torch.zeros(dim))
        self.register_buffer("k_bias", torch.zeros(dim), persistent=False)
        self.v_bias = nn.Parameter(torch.zeros(dim))
        self.proj = nn.Linear(dim, dim)

    def bias_table(self):
        """[heads, (2w-1)^2]: 16 sigmoid(cpb_mlp(relative_coords_table))"""
        return 16 * torch.sigmoid(self.cpb_mlp(self.relative_coords_table).view(-1, self.heads)).t()

    def forward(self, x, mask=None):
        B_, N, C = x.shape
        qkv = F.linear(x, self.qkv.weight, torch.cat((self.q_bias, self.k_bias, self.v_bias)))
        q, k, v = qkv.reshape(B_, N, 3, self.heads, -1).permute(2, 0, 3, 1, 4).unbind(0)
        attn = F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-2, -1)
        attn = attn * torch.clamp(self.logit_scale, max=math.log(1.0 / 0.01)).exp()
        table = self.cpb_mlp(self.relative_coords_table).view(-1, self.heads)
        bias = table[self.relative_position_index.view(-1)].view(N, N, -1).permute(2, 0, 1).contiguous()
        attn = attn + 16 * torch.sigmoid(bias).unsqueeze(0)
        if mask is not None:
            nW = mask.shape[0]
            attn = (attn.view(-1, nW, self.heads, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, self.heads, N, N)
        attn = attn.softmax(dim=-1)
        return self.proj((attn @ v).transpose(1, 2).reshape(B_, N, C))


class Mlp(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(dim, 4 * dim), nn.Linear(4 * dim, dim)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x)))


class Block(nn.Module):
    def __init__(self, dim, res, heads, window, shift, pretrained_window):
        super().__init__()
        # timm's _calc_window_shift: a map no larger than the window is one unshifted window
        self.window, self.shift = (res, 0) if res <= window else (window, shift)
        self.attn = WindowAttention(dim, self.window, heads, pretrained_window)
        self.norm1 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.register_buffer("attn_mask", attention_mask(res, res, self.window, self.shift) if self.shift else None,
                             persistent=False)

    def _attn(self, x):
        B, H, W, C = x.shape
        w, s = self.window, self.shift
        xs = torch.roll(x, shifts=(-s, -s), dims=(1, 2)) if s else x
        aw = self.attn(window_partition(xs, w).view(-1, w * w, C), mask=self.attn_mask).view(-1, w, w, C)
        xs = window_reverse(aw, w, H, W)
        return torch.roll(xs, shifts=(s, s), dims=(1, 2)) if s else xs

    def forward(self, x):
        B, H, W, C = x.shape
        x = x + self.norm1(self._attn(x))
        x = x.reshape(B, -1, C)
        x = x + self.norm2(self.mlp(x))
        return x.reshape(B, H, W, C)


class PatchMerging(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(2 * dim)

    def forward(self, x):
        B, H, W, C = x.shape
        x = x.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 4, 2, 5).flatten(3)
        return self.norm(self.reduction(x))


class Stage(nn.Module):
    def __init__(self, dim, res, depth, heads, window, pretrained_window, downsample):
        super().__init__()
        self.downsample = PatchMerging(dim // 2) if downsample else nn.Identity()
        self.blocks = nn.ModuleList([Block(dim, res, heads, window, 0 if i % 2 == 0 else window // 2, pretrained_window)
                                     for i in range(depth)])

    def forward(self, x):
        x = self.downsample(x)
        for b in self.blocks:
            x = b(x)
        return x


class PatchEmbed(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.proj = nn.Conv2d(3, dim, 4, 4)
        self.norm = nn.LayerNorm(dim)

    def forward(self, x):
        return self.norm(self.proj(x).permute(0, 2, 3, 1))


class SwinTransformerV2(nn.Module):
    """forward() = timm's forward_features + the identity head of num_classes=0, global_pool='': NHWC [B, S/32, S/32, 8C]."""

    def __init__(self, embed_dim, depths, num_heads, window_size, pretrained_window_sizes, img_size=256):
        super().__init__()
        self.patch_embed = PatchEmbed(embed_dim)
        grid = img_size // 4
        self.layers = nn.Sequential(*[Stage(embed_dim << i, grid >> i, d, h, window_size, pretrained_window_sizes[i], i > 0)
                                      for i, (d, h) in enumerate(zip(depths, num_heads))])
        self.norm = nn.LayerNorm(embed_dim << 3)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        for stage in self.layers:
            for b in stage.blocks:
                for n in (b.norm1, b.norm2):
                    nn.init.zeros_(n.weight)
                    nn.init.zeros_(n.bias)

    def forward(self, x):
        return self.norm(self.layers(self.patch_embed(x)))


def backbone(name, depths=None):
    args = dict(ARCHS[name])
    if depths is not None:
        args["depths"] = tuple(depths)
    return SwinTransformerV2(**args)


class WrapperOracle(nn.Module):
    """The reference TimmWrapper around the oracle tower: the neck is built by its rank rule from the tower's output on a
    zero image (timm_wrapper.py:23-49), so timm 0.9's NHWC map takes the CNN branch with channels = shape[1]."""

    def __init__(self, name, feat_dim, image_size=256, depths=None):
        super().__init__()
        self.model = backbone(name, depths)
        with torch.no_grad():
            out = self.model(torch.zeros(1, 3, image_size, image_size))
        if out.dim() == 4:
            _, channels, h, w = out.shape
            self.output_layer = nn.Sequential(nn.BatchNorm2d(channels), nn.Flatten(1), nn.Linear(channels * h * w, feat_dim),
                                              nn.BatchNorm1d(feat_dim))
        else:
            _, tokens, channels = out.shape
            self.output_layer = nn.Sequential(nn.LayerNorm(channels), nn.Flatten(1), nn.Linear(tokens * channels, feat_dim),
                                              nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))


@torch.no_grad()
def randomize_(m: nn.Module, seed: int) -> nn.Module:
    """Every parameter and BatchNorm statistic away from its init (the post-norms are zero at timm's init, which would make
    every block the identity): LayerNorm / BatchNorm affines around 1 / 0, exp(logit scales) in [2, 20] around timm's init
    value 10, CPB weights wide enough that the bias table varies.

    The scales stay below the ln 100 clamp on purpose: near it a cosine error of bf16 size moves a score by ~0.3 and the
    network stops being a well-conditioned function of its bf16 activations (rounding only the oracle's Linear / LayerNorm
    outputs and weights to bf16 moves its depth-(2, 2, 2, 2) embedding by relative L2 0.86 at scales up to 100, 0.009 at
    scales up to 20).  The clamp itself is checked at the kernel and packing level."""
    g = torch.Generator().manual_seed(seed)
    for name, p in m.named_parameters():
        r = torch.randn(p.shape, generator=g)
        if name.endswith("logit_scale"):
            p.copy_(torch.log(torch.empty(p.shape).uniform_(2.0, 20.0, generator=g)))
        elif "cpb_mlp" in name:
            p.copy_(r * (0.5 if name.endswith("0.weight") or name.endswith("0.bias") else 0.05))
        elif p.dim() == 1 and ("norm" in name or name.startswith("output_layer.0") or name.startswith("output_layer.3")):
            p.copy_((1.0 + 0.2 * r) if name.endswith("weight") else 0.1 * r)
        elif p.dim() == 1:
            p.copy_(0.02 * r)
        else:
            p.copy_(r * (1.0 / math.sqrt(p[0].numel())))
    for mod in m.modules():
        if isinstance(mod, (nn.BatchNorm1d, nn.BatchNorm2d)):
            mod.running_mean.copy_(0.1 * torch.randn(mod.running_mean.shape, generator=g))
            mod.running_var.copy_(torch.empty(mod.running_var.shape).uniform_(0.5, 2.0, generator=g))
    return m
