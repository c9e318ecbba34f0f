"""Oracle for the CBIR config's other Transformer towers (TEST INFRASTRUCTURE — see oracle/__init__.py).

The reference's CBIR config (configs/faceX/cbir.yaml:6-16) lists, besides the plain ViTs of oracle/vit.py, four timm
VisionTransformer entries that need three more options of timm 0.9.16's VisionTransformer (timm/models/vision_transformer.py):
an MLP width other than 4 * dim, no class token, and LayerScale.  This file restates that VisionTransformer with those options,
in plain PyTorch fp32 with timm's state_dict keys, reusing oracle/vit.py's Attention (head dim = dim / heads, scale
head_dim^-0.5) and PatchEmbed.  With every option at its default it is oracle/vit.py's model.

  vit_base_patch8_224            DINO ViT-B/8: the plain ViT at patch 8 (785 tokens).  Cross-check: HF ViTModel.
  vit_large_patch14_dinov2       DINOv2 ViT-L/14 at 518^2 (1370 tokens): `init_values=1e-5` -> LayerScale after attention and
                                 MLP, x + ls1.gamma * attn(norm1(x)), x + ls2.gamma * mlp(norm2(x)) (keys `blocks.{i}.ls1.gamma`,
                                 `ls2.gamma`).  Cross-check: HF Dinov2Model (layer_scale1/2.lambda1).
  vit_so400m_patch14_siglip_224  SigLIP So400m/14: width 1152, 16 heads of 72, MLP int(1152 * 3.7362) = 4304, `class_token=False`
                                 (timm sets cls_token to None, so there is no such key; pos_embed [1, 256, C]; the neck flattens
                                 256 tokens).  Registered WITHOUT an act_layer, so timm's default erf nn.GELU.  timm registers it
                                 with global_pool='map', but the reference passes global_pool='', which builds neither attn_pool
                                 nor fc_norm.  Cross-check: HF SiglipVisionModel with hidden_act="gelu" and no head.
  vit_huge_patch14_clip_224      CLIP ViT-H/14: oracle/vit.py's pre_norm tower at width 1280, 16 heads of 80.  Cross-check: HF
                                 CLIPVisionModel (hidden_act="gelu").

The HF cross-checks (tests/test_oracle_vit_archs_cpu.py) pin the architectures, not timm: the hyperparameters above, SigLIP's
erf GELU, the key names and the absent cls_token key are read from timm 0.9.16's source, which is not installed here — PARITY
UNPINNED at the timm boundary, like every ViT in oracle/vit.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from oracle.vit import VIT_ARCHS as _BASE_ARCHS, VIT_PRE_NORM as _BASE_PRE_NORM, Attention, PatchEmbed, randomize_  # noqa: F401

VIT_ARCHS = dict(_BASE_ARCHS)
VIT_ARCHS.update({
    # timm name -> (patch, embed_dim, depth, heads)
    "vit_base_patch8_224": (8, 768, 12, 12),
    "vit_large_patch14_dinov2": (14, 1024, 24, 16),
    "vit_so400m_patch14_siglip_224": (14, 1152, 27, 16),
    "vit_huge_patch14_clip_224": (14, 1280, 32, 16),
})
VIT_PRE_NORM = set(_BASE_PRE_NORM) | {"vit_huge_patch14_clip_224"}
VIT_MLP_DIM = {"vit_so400m_patch14_siglip_224": 4304}
VIT_NO_CLASS_TOKEN = {"vit_so400m_patch14_siglip_224"}
VIT_LAYER_SCALE = {"vit_large_patch14_dinov2"}
VIT_IMAGE_SIZE = {"vit_large_patch14_dinov2": 518, "vit_large_patch14_clip_336": 336}  # pretrained resolution (else 224)


class Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()  # erf form: timm's default act_layer
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class LayerScale(nn.Module):
    """timm's LayerScale: x * gamma (init_values 1e-5 for DINOv2)."""

    def __init__(self, dim, init_values=1e-5):
        super().__init__()
        self.gamma = nn.Parameter(init_values * torch.ones(dim))

    def forward(self, x):
        return x * self.gamma


class Block(nn.Module):
    def __init__(self, dim, heads, eps, mlp_dim, layer_scale):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = Attention(dim, heads)
        self.ls1 = LayerScale(dim) if layer_scale else nn.Identity()
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = Mlp(dim, mlp_dim)
        self.ls2 = LayerScale(dim) if layer_scale else nn.Identity()

    def forward(self, x):
        x = x + self.ls1(self.attn(self.norm1(x)))
        return x + self.ls2(self.mlp(self.norm2(x)))


class VisionTransformer(nn.Module):
    def __init__(self, image_size, patch, dim, depth, heads, pre_norm=False, mlp_dim=None, class_token=True, layer_scale=False):
        super().__init__()
        n = (image_size // patch) ** 2
        eps = 1e-5 if pre_norm else 1e-6  # timm: norm_layer=nn.LayerNorm for the clip entries, partial(LayerNorm, eps=1e-6) otherwise
        self.patch_embed = PatchEmbed(patch, dim, bias=not pre_norm)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, dim)) if class_token else None
        self.pos_embed = nn.Parameter(torch.randn(1, n + (1 if class_token else 0), dim) * 0.02)
        self.norm_pre = nn.LayerNorm(dim, eps=eps) if pre_norm else nn.Identity()
        self.blocks = nn.Sequential(*[Block(dim, heads, eps, mlp_dim or 4 * dim, layer_scale) for _ in range(depth)])
        self.norm = nn.LayerNorm(dim, eps=eps)

    def forward_tokens(self, x):
        """Tokens after the last block, BEFORE the final LayerNorm (what HF's `last_hidden_state` of a CLIP tower holds)."""
        x = self.patch_embed(x)
        if self.cls_token is not None:
            x = torch.cat([self.cls_token.expand(x.shape[0], -1, -1), x], dim=1)
        return self.blocks(self.norm_pre(x + self.pos_embed))

    def forward(self, x):
        return self.norm(self.forward_tokens(x))


class ViTWrapperOracle(nn.Module):
    """timm_wrapper.py TimmWrapper around one of these towers: `model` + the `[B,N,C]` neck (LayerNorm -> Flatten -> Linear ->
    BatchNorm1d, timm_wrapper.py:39-47) over every token the model outputs."""

    def __init__(self, model_name, feat_dim, image_size, patch=None, dim=None, depth=None, heads=None, pre_norm=None, mlp_dim=None,
                 class_token=None, layer_scale=None):
        super().__init__()
        if dim is None:
            patch, dim, depth, heads = VIT_ARCHS[model_name]
        if pre_norm is None:
            pre_norm = model_name in VIT_PRE_NORM
        if mlp_dim is None:
            mlp_dim = VIT_MLP_DIM.get(model_name)
        if class_token is None:
            class_token = model_name not in VIT_NO_CLASS_TOKEN
        if layer_scale is None:
            layer_scale = model_name in VIT_LAYER_SCALE
        assert image_size % patch == 0 and dim % heads == 0
        self.model = VisionTransformer(image_size, patch, dim, depth, heads, pre_norm=pre_norm, mlp_dim=mlp_dim, class_token=class_token,
                                       layer_scale=layer_scale)
        tokens = (image_size // patch) ** 2 + (1 if class_token else 0)
        self.output_layer = nn.Sequential(nn.LayerNorm(dim), nn.Flatten(1), nn.Linear(tokens * dim, feat_dim),
                                          nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))
