"""Oracle for the ResNet backbones + neck (TEST INFRASTRUCTURE — see oracle/__init__.py).

An fp32 restatement of timm 0.9.16's Bottleneck ResNet (timm/models/resnet.py: ResNet, Bottleneck, create_aa-free
downsample_conv / downsample_avg, the 'deep' stem) with the SAME state_dict keys, built with num_classes=0,
global_pool='' so that forward returns the un-pooled [B, 2048, H/32, W/32] map the reference's neck flattens
(timm_wrapper.py:30-38):

  conv1 Conv2d(3,64,7,s2,p3)  |  deep stem: conv1.{0: Conv(3,32,3,s2), 1: BN, 3: Conv(32,32,3), 4: BN, 6: Conv(32,64,3)}
  bn1, ReLU, MaxPool2d(3, 2, 1)
  layer{1-4}.{i}.{conv1 1x1, bn1, conv2 3x3/stride, bn2, conv3 1x1 (x4), bn3}, ReLU after the residual add
  downsample.{0: Conv 1x1/stride, 1: BN}  |  avg_down: downsample.{0: AvgPool2d(2, 2, ceil_mode, no pad count) or
                                                           Identity (stride 1), 1: Conv 1x1, 2: BN}
  output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear(2048*h*w, feat_dim), 3: BatchNorm1d}

timm is not installed here.  resnet50 / resnet101 / wide_resnet50_2 are pinned against torchvision's ResNets, which
share these keys (tests/test_oracle_resnet_cpu.py); the -D variants' hyperparameters (stem_width=32, stem_type='deep',
avg_down=True) and key names were read from timm's source and are unverified beyond the module-by-module check there.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

RESNET_ARCHS = {
    # timm name -> ResNet kwargs (timm 0.9.16 model_args)
    "resnet50": dict(depths=(3, 4, 6, 3)),
    "resnet101": dict(depths=(3, 4, 23, 3)),
    "resnet152": dict(depths=(3, 8, 36, 3)),
    "resnet50d": dict(depths=(3, 4, 6, 3), stem_width=32, stem_type="deep", avg_down=True),
    "resnet101d": dict(depths=(3, 4, 23, 3), stem_width=32, stem_type="deep", avg_down=True),
    "resnet152d": dict(depths=(3, 8, 36, 3), stem_width=32, stem_type="deep", avg_down=True),
    "wide_resnet50_2": dict(depths=(3, 4, 6, 3), base_width=128),
    "wide_resnet101_2": dict(depths=(3, 4, 23, 3), base_width=128),
}


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, base_width=64):
        super().__init__()
        width = int(math.floor(planes * (base_width / 64)))
        outplanes = planes * self.expansion
        self.conv1 = nn.Conv2d(inplanes, width, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.act1 = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(width, width, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.act2 = nn.ReLU(inplace=True)
        self.conv3 = nn.Conv2d(width, outplanes, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(outplanes)
        self.act3 = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        shortcut = x
        x = self.act1(self.bn1(self.conv1(x)))
        x = self.act2(self.bn2(self.conv2(x)))
        x = self.bn3(self.conv3(x))
        if self.downsample is not None:
            shortcut = self.downsample(shortcut)
        return self.act3(x + shortcut)


def downsample_conv(in_chs, out_chs, stride):
    return nn.Sequential(nn.Conv2d(in_chs, out_chs, 1, stride=stride, bias=False), nn.BatchNorm2d(out_chs))


def downsample_avg(in_chs, out_chs, stride):
    pool = nn.AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False) if stride != 1 else nn.Identity()
    return nn.Sequential(pool, nn.Conv2d(in_chs, out_chs, 1, stride=1, bias=False), nn.BatchNorm2d(out_chs))


class ResNet(nn.Module):
    def __init__(self, depths, base_width=64, stem_width=64, stem_type="", avg_down=False):
        super().__init__()
        deep = "deep" in stem_type
        inplanes = stem_width * 2 if deep else 64
        if deep:
            self.conv1 = nn.Sequential(
                nn.Conv2d(3, stem_width, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(stem_width), nn.ReLU(inplace=True),
                nn.Conv2d(stem_width, stem_width, 3, stride=1, padding=1, bias=False), nn.BatchNorm2d(stem_width),
                nn.ReLU(inplace=True), nn.Conv2d(stem_width, inplanes, 3, stride=1, padding=1, bias=False))
        else:
            self.conv1 = nn.Conv2d(3, inplanes, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(inplanes)
        self.act1 = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride = 1 if i == 0 else 2
            blocks = []
            for j in range(depth):
                down = None
                if j == 0 and (stride != 1 or inplanes != planes * 4):
                    down = (downsample_avg if avg_down else downsample_conv)(inplanes, planes * 4, stride)
                blocks.append(Bottleneck(inplanes, planes, stride if j == 0 else 1, down, base_width))
                inplanes = planes * 4
            setattr(self, f"layer{i + 1}", nn.Sequential(*blocks))

    def forward(self, x):
        x = self.maxpool(self.act1(self.bn1(self.conv1(x))))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))


class ResNetWrapperOracle(nn.Module):
    """timm_wrapper.py:5-54 for a ResNet backbone: un-pooled features -> BN2d -> Flatten -> Linear -> BN1d."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int, depths=None):
        super().__init__()
        kw = dict(RESNET_ARCHS[model_name])
        if depths is not None:
            kw["depths"] = tuple(depths)
        self.model = ResNet(**kw)
        hw = image_size // 32
        self.output_layer = nn.Sequential(nn.BatchNorm2d(2048), nn.Flatten(1), nn.Linear(2048 * hw * hw, feat_dim),
                                          nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))


def randomize_(module: nn.Module, seed: int = 0) -> nn.Module:
    """Random, well-conditioned weights and BatchNorm statistics / affine parameters — every BatchNorm, bn3 included
    (timm zero-initialises bn3.weight, which would silence every residual branch)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, m in module.named_modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                scale = 0.3 if name.endswith("bn3") else 1.0  # keeps the residual stream's growth moderate over 50 blocks
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
