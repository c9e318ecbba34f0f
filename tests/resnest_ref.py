"""fp32 oracle of the ResNeSt backbones + neck (test infrastructure, like oracle/).

An fp32 restatement of timm 0.9.16 timm/models/resnest.py (ResNestBottleneck) and timm/layers/split_attn.py (SplitAttn,
RadixSoftmax) on timm's ResNet with stem_type='deep', stem_width=32, avg_down=True, num_classes=0, global_pool='', with
the same state_dict keys:

  conv1.{0: Conv(3,32,3,s2), 1: BN, 3: Conv(32,32,3), 4: BN, 6: Conv(32,64,3)}, bn1, ReLU, MaxPool2d(3, 2, 1)
  layer{1-4}.{i}.{conv1 1x1, bn1, [avd_first], conv2 = SplitAttn.{conv, bn0, fc1, bn1, fc2}, [avd_last], conv3 1x1, bn3},
  ReLU after the residual add; downsample.{0: AvgPool2d(2, 2, ceil_mode, no pad count) or Identity, 1: Conv 1x1, 2: BN}

avd is AvgPool2d(3, stride, padding=1) (count_include_pad=True) on stride-2 blocks only: timm's make_blocks does not pass
is_first, so no stage-1 block has one.  timm is not installed here: the hyperparameters and key names were read from timm's
source; SplitAttn is checked against an independent per-(radix, cardinal group) formulation in tests/test_resnest_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.resnet import randomize_  # noqa: F401  (re-exported for the tests)

RESNEST_ARCHS = {
    "resnest14d": dict(depths=(1, 1, 1, 1), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest26d": dict(depths=(2, 2, 2, 2), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest50d": dict(depths=(3, 4, 6, 3), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest50d_1s4x24d": dict(depths=(3, 4, 6, 3), radix=1, cardinality=4, base_width=24, avd_first=True),
    "resnest50d_4s2x40d": dict(depths=(3, 4, 6, 3), radix=4, cardinality=2, base_width=40, avd_first=True),
}


def make_divisible(v, divisor=8, min_value=None, round_limit=0.9):
    min_value = min_value or divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < round_limit * v:
        new_v += divisor
    return new_v


class RadixSoftmax(nn.Module):
    def __init__(self, radix, cardinality):
        super().__init__()
        self.radix, self.cardinality = radix, cardinality

    def forward(self, x):
        batch = x.size(0)
        if self.radix > 1:
            x = x.view(batch, self.cardinality, self.radix, -1).transpose(1, 2)
            x = F.softmax(x, dim=1)
            x = x.reshape(batch, -1)
        else:
            x = torch.sigmoid(x)
        return x


class SplitAttn(nn.Module):
    def __init__(self, in_channels, out_channels=None, kernel_size=3, stride=1, padding=1, groups=1, radix=2, rd_ratio=0.25,
                 rd_divisor=8):
        super().__init__()
        out_channels = out_channels or in_channels
        self.radix = radix
        mid_chs = out_channels * radix
        attn_chs = make_divisible(in_channels * radix * rd_ratio, min_value=32, divisor=rd_divisor)
        self.conv = nn.Conv2d(in_channels, mid_chs, kernel_size, stride, padding, groups=groups * radix, bias=False)
        self.bn0 = nn.BatchNorm2d(mid_chs)
        self.act0 = nn.ReLU(inplace=True)
        self.fc1 = nn.Conv2d(out_channels, attn_chs, 1, groups=groups)
        self.bn1 = nn.BatchNorm2d(attn_chs)
        self.act1 = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(attn_chs, mid_chs, 1, groups=groups)
        self.rsoftmax = RadixSoftmax(radix, groups)

    def forward(self, x):
        x = self.act0(self.bn0(self.conv(x)))
        B, RC, H, W = x.shape
        if self.radix > 1:
            x = x.reshape((B, self.radix, RC // self.radix, H, W))
            x_gap = x.sum(dim=1)
        else:
            x_gap = x
        x_gap = x_gap.mean((2, 3), keepdim=True)
        x_attn = self.fc2(self.act1(self.bn1(self.fc1(x_gap))))
        x_attn = self.rsoftmax(x_attn).view(B, -1, 1, 1)
        if self.radix > 1:
            out = (x * x_attn.reshape((B, self.radix, RC // self.radix, 1, 1))).sum(dim=1)
        else:
            out = x * x_attn
        return out.contiguous()


class ResNestBottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, radix=1, cardinality=1, base_width=64, avd=True,
                 avd_first=False):
        super().__init__()
        group_width = int(planes * (base_width / 64.0)) * cardinality
        if avd and stride > 1:
            avd_stride, stride = stride, 1
        else:
            avd_stride = 0
        self.radix = radix
        self.conv1 = nn.Conv2d(inplanes, group_width, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(group_width)
        self.act1 = nn.ReLU(inplace=True)
        self.avd_first = nn.AvgPool2d(3, avd_stride, padding=1) if avd_stride > 0 and avd_first else None
        self.conv2 = SplitAttn(group_width, group_width, kernel_size=3, stride=stride, padding=1, groups=cardinality, radix=radix)
        self.avd_last = nn.AvgPool2d(3, avd_stride, padding=1) if avd_stride > 0 and not avd_first else None
        self.conv3 = nn.Conv2d(group_width, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.act3 = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        shortcut = x
        out = self.act1(self.bn1(self.conv1(x)))
        if self.avd_first is not None:
            out = self.avd_first(out)
        out = self.conv2(out)
        if self.avd_last is not None:
            out = self.avd_last(out)
        out = self.bn3(self.conv3(out))
        if self.downsample is not None:
            shortcut = self.downsample(x)
        return self.act3(out + shortcut)


class ResNeSt(nn.Module):
    def __init__(self, depths, radix, cardinality, base_width, avd_first):
        super().__init__()
        self.conv1 = nn.Sequential(
            nn.Conv2d(3, 32, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
            nn.Conv2d(32, 32, 3, stride=1, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
            nn.Conv2d(32, 64, 3, stride=1, padding=1, bias=False))
        self.bn1 = nn.BatchNorm2d(64)
        self.act1 = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        inplanes = 64
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride, blocks = (1 if i == 0 else 2), []
            for j in range(depth):
                down = None
                if j == 0 and (stride != 1 or inplanes != planes * 4):
                    pool = nn.AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False) if stride != 1 else nn.Identity()
                    down = nn.Sequential(pool, nn.Conv2d(inplanes, planes * 4, 1, bias=False), nn.BatchNorm2d(planes * 4))
                blocks.append(ResNestBottleneck(inplanes, planes, stride if j == 0 else 1, down, radix, cardinality, base_width,
                                                avd_first=avd_first))
                inplanes = planes * 4
            setattr(self, f"layer{i + 1}", nn.Sequential(*blocks))

    def forward(self, x):
        x = self.maxpool(self.act1(self.bn1(self.conv1(x))))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))


def backbone(name, depths=None) -> ResNeSt:
    kw = dict(RESNEST_ARCHS[name])
    if depths is not None:
        kw["depths"] = tuple(depths)
    return ResNeSt(**kw)


class WrapperOracle(nn.Module):
    """timm_wrapper.py:5-54 for a ResNeSt backbone: un-pooled features -> BN2d -> Flatten -> Linear -> BN1d."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int, depths=None):
        super().__init__()
        self.model = backbone(model_name, depths)
        hw = image_size // 32
        self.output_layer = nn.Sequential(nn.BatchNorm2d(2048), nn.Flatten(1), nn.Linear(2048 * hw * hw, feat_dim),
                                          nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))
