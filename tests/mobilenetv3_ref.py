"""fp32 oracle of the MobileNetV3 backbones + neck (test infrastructure, like oracle/).

An fp32 restatement of timm 0.9.16 timm/models/mobilenetv3.py `MobileNetV3` (num_classes=0, global_pool='') for the six
width-1.0 entries of visiondk_b200.mobilenetv3.MOBILENETV3_ARCHS, with the same state_dict keys:

  conv_stem 3x3/s2 + bn1 + act
  blocks.<stage>.<i>: DepthwiseSeparableConv {conv_dw k/s, bn1} act, [se], {conv_pw 1x1, bn2} (+ shortcut)
                      InvertedResidual {conv_pw 1x1, bn1} act, {conv_dw k/s depthwise, bn2} act, [se], {conv_pwl, bn3} (+ shortcut)
                      ConvBnAct {conv 1x1, bn1} act
  se: conv_reduce -> ReLU -> conv_expand -> hard_sigmoid gate;  a shortcut when stride == 1 and in == out
  forward_head with global_pool='': conv_head 1x1 (with bias) + act on the unpooled map

act is hard-swish or ReLU per block (nre), ReLU throughout for the minimal variants.  The tf_* models pad every conv
TensorFlow-"same" (effnetv2_ref's Conv2dSame) with BatchNorm eps 1e-3; the others pad k // 2 with eps 1e-5.  timm is not
installed here: the arch strings, key names and block order were read from timm's source; the full models' bodies are
pinned against torchvision's mobilenet_v3_large / _small in tests/test_mobilenetv3_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from effnetv2_ref import Conv2dSame, randomize_  # noqa: F401  (randomize_ is re-exported for the GPU tests)
from visiondk_b200.mobilenetv3 import MOBILENETV3_ARCHS, STEM_CH, decode_blocks

ACT = {"relu": F.relu, "hard_swish": F.hardswish}


def conv(cin, cout, k, stride=1, groups=1, bias=False, tf=False):
    if tf:
        return Conv2dSame(cin, cout, k, stride, groups=groups, bias=bias)
    return nn.Conv2d(cin, cout, k, stride, k // 2, groups=groups, bias=bias)


class SqueezeExcite(nn.Module):
    def __init__(self, chs, rd):
        super().__init__()
        self.conv_reduce = nn.Conv2d(chs, rd, 1)
        self.conv_expand = nn.Conv2d(rd, chs, 1)

    def forward(self, x):
        s = F.relu(self.conv_reduce(x.mean((2, 3), keepdim=True)))
        return x * F.hardsigmoid(self.conv_expand(s))


class Block(nn.Module):
    def __init__(self, kind, cin, cout, k, stride, mid, act, se_rd, eps, tf):
        super().__init__()
        self.kind, self.act = kind, ACT[act]
        self.has_skip = kind != "cn" and stride == 1 and cin == cout
        if kind == "cn":
            self.conv = conv(cin, cout, k, stride, tf=tf)
            self.bn1 = nn.BatchNorm2d(cout, eps=eps)
            return
        if kind == "ir":
            self.conv_pw = conv(cin, mid, 1, tf=tf)
            self.bn1 = nn.BatchNorm2d(mid, eps=eps)
        self.conv_dw = conv(mid, mid, k, stride, groups=mid, tf=tf)
        if kind == "ds":
            self.bn1 = nn.BatchNorm2d(mid, eps=eps)
        else:
            self.bn2 = nn.BatchNorm2d(mid, eps=eps)
        self.se = SqueezeExcite(mid, se_rd) if se_rd else nn.Identity()
        if kind == "ds":
            self.conv_pw = conv(mid, cout, 1, tf=tf)
            self.bn2 = nn.BatchNorm2d(cout, eps=eps)
        else:
            self.conv_pwl = conv(mid, cout, 1, tf=tf)
            self.bn3 = nn.BatchNorm2d(cout, eps=eps)

    def forward(self, x):
        if self.kind == "cn":
            return self.act(self.bn1(self.conv(x)))
        if self.kind == "ds":
            y = self.se(self.act(self.bn1(self.conv_dw(x))))
            y = self.bn2(self.conv_pw(y))
        else:
            y = self.act(self.bn1(self.conv_pw(x)))
            y = self.se(self.act(self.bn2(self.conv_dw(y))))
            y = self.bn3(self.conv_pwl(y))
        return y + x if self.has_skip else y


class MobileNetV3(nn.Module):
    def __init__(self, arch, head, act, tf):
        super().__init__()
        eps = 1e-3 if tf else 1e-5
        self.act = ACT[act]
        self.conv_stem = conv(3, STEM_CH, 3, 2, tf=tf)
        self.bn1 = nn.BatchNorm2d(STEM_CH, eps=eps)
        stages = decode_blocks(arch, act)
        self.blocks = nn.Sequential(*[nn.Sequential(*[Block(*spec, eps, tf) for spec in stage]) for stage in stages])
        self.conv_head = conv(stages[-1][-1][2], head, 1, bias=True, tf=tf)

    def forward_features(self, x):
        return self.blocks(self.act(self.bn1(self.conv_stem(x))))

    def forward(self, x):
        return self.act(self.conv_head(self.forward_features(x)))


def backbone(name) -> MobileNetV3:
    return MobileNetV3(**MOBILENETV3_ARCHS[name])


class WrapperOracle(nn.Module):
    """timm_wrapper.py:5-54 for these backbones: the un-pooled [B, head, S/32, S/32] map -> BN2d -> Flatten -> Linear -> BN1d
    (the rank rule's neck, sized from the tower's real output)."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int):
        super().__init__()
        self.model = backbone(model_name)
        with torch.no_grad():
            c, h, w = self.model.eval()(torch.zeros(1, 3, image_size, image_size)).shape[1:]
        self.output_layer = nn.Sequential(nn.BatchNorm2d(c), nn.Flatten(1), nn.Linear(c * h * w, feat_dim), nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))
