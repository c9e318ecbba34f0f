"""fp32 oracle of the EfficientNetV2 backbones + neck (test infrastructure, like oracle/).

An fp32 restatement of timm 0.9.16 timm/models/efficientnet.py `EfficientNet` for tf_efficientnetv2_s / _m / _l
(num_classes=0, global_pool=''), with the same state_dict keys:

  conv_stem Conv2dSame(3, stem, 3, s2) + bn1 + SiLU
  blocks.<stage>.<i>: ConvBnAct  {conv 3x3, bn1} SiLU, then + shortcut
                      EdgeResidual {conv_exp 3x3/s, bn1} SiLU, {conv_pwl 1x1, bn2} (+ shortcut)
                      InvertedResidual {conv_pw 1x1, bn1} SiLU, {conv_dw 3x3/s depthwise, bn2} SiLU,
                                       se.{conv_reduce SiLU, conv_expand sigmoid} gate, {conv_pwl, bn3} (+ shortcut)
  conv_head 1x1 + bn2 + SiLU;  every BatchNorm eps 1e-3, a shortcut when stride == 1 and in == out

Every 3x3 conv pads TensorFlow-"same" with an explicit F.pad: per axis total = max((ceil(H / s) - 1) s + k - H, 0),
low = total // 2.  timm is not installed here: the arch definitions and key names were read from timm's source; the block
structure, widths, depths, SE widths and BN eps are pinned against torchvision's efficientnet_v2_{s,m,l} in
tests/test_oracle_effnetv2_cpu.py.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from visiondk_b200.efficientnet import EFFNETV2_ARCHS, HEAD_CH  # noqa: F401  (arch table shared with the wrapper)

BN_EPS = 1e-3


def same_pad(x: torch.Tensor, k: int, s: int) -> torch.Tensor:
    """TF "same" zero padding of an NCHW map for a k x k / stride-s conv."""
    pads = []
    for size in (x.shape[3], x.shape[2]):  # F.pad order: (w_lo, w_hi, h_lo, h_hi)
        total = max((math.ceil(size / s) - 1) * s + k - size, 0)
        pads += [total // 2, total - total // 2]
    return F.pad(x, pads)


class Conv2dSame(nn.Conv2d):
    def forward(self, x):
        return F.conv2d(same_pad(x, self.kernel_size[0], self.stride[0]), self.weight, self.bias, self.stride, 0, 1, self.groups)


def bn(c):
    return nn.BatchNorm2d(c, eps=BN_EPS)


class SqueezeExcite(nn.Module):
    def __init__(self, chs, rd):
        super().__init__()
        self.conv_reduce = nn.Conv2d(chs, rd, 1)
        self.conv_expand = nn.Conv2d(rd, chs, 1)

    def forward(self, x):
        s = F.silu(self.conv_reduce(x.mean((2, 3), keepdim=True)))
        return x * torch.sigmoid(self.conv_expand(s))


class ConvBnAct(nn.Module):
    def __init__(self, cin, cout, stride, exp):
        super().__init__()
        self.conv = Conv2dSame(cin, cout, 3, stride, bias=False)
        self.bn1 = bn(cout)
        self.has_skip = stride == 1 and cin == cout

    def forward(self, x):
        y = F.silu(self.bn1(self.conv(x)))
        return y + x if self.has_skip else y


class EdgeResidual(nn.Module):
    def __init__(self, cin, cout, stride, exp):
        super().__init__()
        mid = cin * exp
        self.conv_exp = Conv2dSame(cin, mid, 3, stride, bias=False)
        self.bn1 = bn(mid)
        self.conv_pwl = nn.Conv2d(mid, cout, 1, bias=False)
        self.bn2 = bn(cout)
        self.has_skip = stride == 1 and cin == cout

    def forward(self, x):
        y = self.bn2(self.conv_pwl(F.silu(self.bn1(self.conv_exp(x)))))
        return y + x if self.has_skip else y


class InvertedResidual(nn.Module):
    def __init__(self, cin, cout, stride, exp):
        super().__init__()
        mid = cin * exp
        self.conv_pw = nn.Conv2d(cin, mid, 1, bias=False)
        self.bn1 = bn(mid)
        self.conv_dw = Conv2dSame(mid, mid, 3, stride, groups=mid, bias=False)
        self.bn2 = bn(mid)
        self.se = SqueezeExcite(mid, round(cin / 4))
        self.conv_pwl = nn.Conv2d(mid, cout, 1, bias=False)
        self.bn3 = bn(cout)
        self.has_skip = stride == 1 and cin == cout

    def forward(self, x):
        y = F.silu(self.bn1(self.conv_pw(x)))
        y = self.se(F.silu(self.bn2(self.conv_dw(y))))
        y = self.bn3(self.conv_pwl(y))
        return y + x if self.has_skip else y


BLOCKS = {"cn": ConvBnAct, "er": EdgeResidual, "ir": InvertedResidual}


class EfficientNetV2(nn.Module):
    def __init__(self, stem, stages, depths=None):
        super().__init__()
        self.conv_stem = Conv2dSame(3, stem, 3, 2, bias=False)
        self.bn1 = bn(stem)
        self.blocks = nn.Sequential()
        cin = stem
        for s, (kind, reps, stride, exp, cout) in enumerate(stages):
            n = reps if depths is None else depths[s]
            self.blocks.add_module(str(s), nn.Sequential(*[BLOCKS[kind](cin if i == 0 else cout, cout, stride if i == 0 else 1, exp)
                                                           for i in range(n)]))
            cin = cout
        self.conv_head = nn.Conv2d(cin, HEAD_CH, 1, bias=False)
        self.bn2 = bn(HEAD_CH)

    def forward(self, x):
        x = F.silu(self.bn1(self.conv_stem(x)))
        x = self.blocks(x)
        return F.silu(self.bn2(self.conv_head(x)))


def backbone(name, depths=None) -> EfficientNetV2:
    return EfficientNetV2(**EFFNETV2_ARCHS[name], depths=depths)


class WrapperOracle(nn.Module):
    """timm_wrapper.py:5-54 for these backbones: the un-pooled [B, 1280, S/32, S/32] map -> BN2d -> Flatten -> Linear -> BN1d
    (the rank rule's neck, sized from the tower's real output)."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int, depths=None):
        super().__init__()
        self.model = backbone(model_name, depths)
        with torch.no_grad():
            c, h, w = self.model.eval()(torch.zeros(1, 3, image_size, image_size)).shape[1:]
        self.output_layer = nn.Sequential(nn.BatchNorm2d(c), nn.Flatten(1), nn.Linear(c * h * w, feat_dim), nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))


def randomize_(module: nn.Module, seed: int = 0) -> nn.Module:
    """Random, well-conditioned weights and BatchNorm statistics / affine parameters for every BatchNorm.  The projection
    BatchNorms (bn2 of an EdgeResidual, bn3 of an InvertedResidual) are scaled by 0.3, as oracle/resnet.py does for bn3, so
    that the residual stream's growth stays moderate over L's 79 blocks."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, m in module.named_modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                parent = module.get_submodule(name.rsplit(".", 1)[0]) if "." in name else module
                proj = name.endswith("bn3") or (name.endswith("bn2") and hasattr(parent, "conv_exp"))  # EdgeResidual's bn2
                scale = 0.3 if proj else 1.0
                m.weight.copy_(scale * (0.5 + 0.5 * torch.rand(m.weight.shape, generator=g)))
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=g))
                m.running_var.copy_(0.5 + torch.rand(m.running_var.shape, generator=g))
            elif isinstance(m, (nn.Conv2d, nn.Linear)):
                fan_in = m.weight[0].numel()
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
                if m.bias is not None:
                    m.bias.copy_(0.05 * torch.randn(m.bias.shape, generator=g))
    return module
