"""fp32 oracles of the ResNeXt and legacy SENet backbones + neck (test infrastructure, like oracle/).

ResNeXt: timm 0.9.16 resnet.py with cardinality > 1 is oracle/resnet.py's ResNet whose Bottleneck width is
floor(planes * base_width / 64) * cardinality and whose 3x3 conv has `cardinality` groups.  It is built here from
oracle.resnet.ResNet (base_width * cardinality gives the same widths), with each conv2 swapped for the grouped conv in place,
so the state_dict keys and their order stay timm's.  It is pinned against torchvision's ResNeXts, which share the keys.

Legacy SENet: an fp32 restatement of timm 0.9.16 timm/models/senet.py (SEModule, SEResNetBottleneck, SEResNeXtBottleneck,
SENet with num_classes=0, global_pool='') with the same state_dict keys:

  layer0.{conv1 Conv2d(3,64,7,s2,p3), bn1, relu1}, pool0 MaxPool2d(3, 2, ceil_mode=True)
  layer{1-4}.{i}.{conv1, bn1, conv2 (groups), bn2, conv3, bn3, se_module.{fc1, fc2} (1x1 convs with bias)}, ReLU after
  se_module(bn3(conv3)) + shortcut; downsample.{0: Conv 1x1/stride, 1: BN}

timm is not installed here: the legacy SENet hyperparameters (reduction 16, stride on conv1 for SE-ResNet and on conv2 for
SE-ResNeXt, base width 4) and key names were read from timm's source and are unverified beyond the module-by-module checks
in tests/test_resnext_senet_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from oracle.resnet import ResNet, randomize_  # noqa: F401  (randomize_ re-exported for the tests)

RESNEXT_ARCHS = {
    "resnext50_32x4d": dict(depths=(3, 4, 6, 3), cardinality=32, base_width=4),
    "resnext50d_32x4d": dict(depths=(3, 4, 6, 3), cardinality=32, base_width=4, stem_width=32, stem_type="deep", avg_down=True),
    "resnext101_32x8d": dict(depths=(3, 4, 23, 3), cardinality=32, base_width=8),
    "resnext101_64x4d": dict(depths=(3, 4, 23, 3), cardinality=64, base_width=4),
}

SENET_ARCHS = {
    "legacy_seresnet50": dict(block="seresnet", depths=(3, 4, 6, 3), groups=1),
    "legacy_seresnet101": dict(block="seresnet", depths=(3, 4, 23, 3), groups=1),
    "legacy_seresnet152": dict(block="seresnet", depths=(3, 8, 36, 3), groups=1),
    "legacy_seresnext26_32x4d": dict(block="seresnext", depths=(2, 2, 2, 2), groups=32),
    "legacy_seresnext50_32x4d": dict(block="seresnext", depths=(3, 4, 6, 3), groups=32),
    "legacy_seresnext101_32x4d": dict(block="seresnext", depths=(3, 4, 23, 3), groups=32),
}


def resnext(depths, cardinality, base_width, **kw) -> ResNet:
    m = ResNet(depths, base_width=base_width * cardinality, **kw)
    for i in range(4):
        for blk in getattr(m, f"layer{i + 1}"):
            c = blk.conv2
            blk.conv2 = nn.Conv2d(c.in_channels, c.out_channels, 3, stride=c.stride, padding=1, groups=cardinality, bias=False)
    return m


class SEModule(nn.Module):
    def __init__(self, channels, reduction):
        super().__init__()
        self.fc1 = nn.Conv2d(channels, channels // reduction, kernel_size=1)
        self.relu = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(channels // reduction, channels, kernel_size=1)
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        s = x.mean((2, 3), keepdim=True)
        return x * self.sigmoid(self.fc2(self.relu(self.fc1(s))))


class SEBottleneck(nn.Module):
    """SEResNetBottleneck (width planes, stride on conv1) / SEResNeXtBottleneck (width floor(planes * 4 / 64) * groups,
    stride on conv2); expansion 4, reduction 16."""

    def __init__(self, block, inplanes, planes, groups, reduction, stride=1, downsample=None):
        super().__init__()
        resnext = block == "seresnext"
        width = (planes * 4 // 64) * groups if resnext else planes
        self.conv1 = nn.Conv2d(inplanes, width, kernel_size=1, bias=False, stride=1 if resnext else stride)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, kernel_size=3, stride=stride if resnext else 1, padding=1, groups=groups, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.se_module = SEModule(planes * 4, reduction=reduction)
        self.downsample = downsample

    def forward(self, x):
        shortcut = x
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        if self.downsample is not None:
            shortcut = self.downsample(x)
        return self.relu(self.se_module(out) + shortcut)


class SENet(nn.Module):
    def __init__(self, block, depths, groups, reduction=16):
        super().__init__()
        self.layer0 = nn.Sequential()
        self.layer0.add_module("conv1", nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False))
        self.layer0.add_module("bn1", nn.BatchNorm2d(64))
        self.layer0.add_module("relu1", nn.ReLU(inplace=True))
        self.pool0 = nn.MaxPool2d(3, stride=2, ceil_mode=True)
        inplanes = 64
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride = 1 if i == 0 else 2
            down = None
            if stride != 1 or inplanes != planes * 4:
                down = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False), nn.BatchNorm2d(planes * 4))
            layers = [SEBottleneck(block, inplanes, planes, groups, reduction, stride, down)]
            inplanes = planes * 4
            layers += [SEBottleneck(block, inplanes, planes, groups, reduction) for _ in range(1, depth)]
            setattr(self, f"layer{i + 1}", nn.Sequential(*layers))

    def forward(self, x):
        x = self.pool0(self.layer0(x))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))


def backbone(name, depths=None) -> nn.Module:
    if name in RESNEXT_ARCHS:
        kw = dict(RESNEXT_ARCHS[name])
        if depths is not None:
            kw["depths"] = tuple(depths)
        return resnext(**kw)
    kw = dict(SENET_ARCHS[name])
    if depths is not None:
        kw["depths"] = tuple(depths)
    return SENet(**kw)


class WrapperOracle(nn.Module):
    """timm_wrapper.py:5-54 for these backbones: un-pooled features -> BN2d -> Flatten -> Linear -> BN1d."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int, depths=None):
        super().__init__()
        self.model = backbone(model_name, depths)
        hw = image_size // 32
        self.output_layer = nn.Sequential(nn.BatchNorm2d(2048), nn.Flatten(1), nn.Linear(2048 * hw * hw, feat_dim),
                                          nn.BatchNorm1d(feat_dim))

    def forward(self, x):
        return self.output_layer(self.model(x))


def block_diagonal(w: torch.Tensor) -> torch.Tensor:
    """Grouped weight [Cout, cg, k, k] -> the dense [Cout, k, k, Cout] weight that is zero outside each output channel's
    group: a dense conv with it is exactly the grouped conv."""
    cout, cg, k = w.shape[0], w.shape[1], w.shape[2]
    dense = w.new_zeros(cout, k, k, cout)
    for g in range(cout // cg):
        dense[g * cg:(g + 1) * cg, :, :, g * cg:(g + 1) * cg] = w[g * cg:(g + 1) * cg].permute(0, 2, 3, 1)
    return dense
