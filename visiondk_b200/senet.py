"""Legacy SENet backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 timm/models/senet.py).

`SENetWrapper` is the reference's TimmWrapper for a `timm-legacy_seresnet*` / `timm-legacy_seresnext*` backbone
(models/faceX/backbone/timm_wrapper.py:16-54): the legacy SENet built with num_classes=0, global_pool='' under `model.`
and the CNN neck `output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear, 3: BatchNorm1d}`.  Parameter names and shapes are
timm's legacy ones (`layer0.conv1`, `layerN.i.se_module.fc1`, `downsample.0/1`), so timm checkpoints load with strict=True.
The arithmetic is csrc/resnet.cu (vdk_bottleneck_forward): every eval BatchNorm folded into its convolution, the grouped
3x3 convs of the SE-ResNeXts on vdk_conv2d_grouped, the SE gate in fp32.  Extraction only: a train-mode forward raises
NotImplementedError.
"""
from __future__ import annotations

import torch.nn as nn

from .resnet import STEM_POOL_CEIL, BottleneckNetC, pack_grouped
from .wrapper import BackboneWrapper, cnn_neck, fold_bn

# timm 0.9.16 senet.py model_args (reduction 16; SE-ResNet: stride on the 1x1 conv1, SE-ResNeXt: on the 3x3 conv2)
SENET_ARCHS = {
    "legacy_seresnet50": dict(block="seresnet", depths=(3, 4, 6, 3), groups=1),
    "legacy_seresnet101": dict(block="seresnet", depths=(3, 4, 23, 3), groups=1),
    "legacy_seresnet152": dict(block="seresnet", depths=(3, 8, 36, 3), groups=1),
    "legacy_seresnext26_32x4d": dict(block="seresnext", depths=(2, 2, 2, 2), groups=32),
    "legacy_seresnext50_32x4d": dict(block="seresnext", depths=(3, 4, 6, 3), groups=32),
    "legacy_seresnext101_32x4d": dict(block="seresnext", depths=(3, 4, 23, 3), groups=32),
}
SE_REDUCTION = 16


class _SEModule(nn.Module):
    def __init__(self, channels, reduction):
        super().__init__()
        self.fc1 = nn.Conv2d(channels, channels // reduction, 1)
        self.fc2 = nn.Conv2d(channels // reduction, channels, 1)


class _SEBottleneck(nn.Module):
    """SEResNetBottleneck (block='seresnet': width = planes, stride on conv1) or SEResNeXtBottleneck (block='seresnext':
    width = floor(planes * 4 / 64) * groups, stride on conv2)."""

    def __init__(self, block, inplanes, planes, groups, stride, downsample):
        super().__init__()
        resnext = block == "seresnext"
        width = (planes * 4 // 64) * groups if resnext else planes
        self.stride = stride
        self.conv1 = nn.Conv2d(inplanes, width, 1, bias=False, stride=1 if resnext else stride)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, 3, stride=stride if resnext else 1, padding=1, groups=groups, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.se_module = _SEModule(planes * 4, SE_REDUCTION)
        self.downsample = downsample


class SENetParams(nn.Module):
    """timm 0.9.16 legacy `SENet(block, layers, groups, reduction=16, num_classes=0, global_pool='')` parameter tree:
    layer0.{conv1 7x7/s2, bn1}, pool0 = MaxPool2d(3, 2, ceil_mode=True), layer1-4 of SE Bottlenecks whose first block has
    downsample.{0: Conv 1x1/stride, 1: BN}.  Parameter containers only: the forward is vdk_bottleneck_forward."""

    def __init__(self, block, depths, groups):
        super().__init__()
        self.block, self.depths, self.groups = block, tuple(depths), int(groups)
        self.layer0 = nn.Sequential()
        self.layer0.add_module("conv1", nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False))
        self.layer0.add_module("bn1", nn.BatchNorm2d(64))
        self.layer0.add_module("relu1", nn.ReLU())
        inplanes = 64
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride, blocks = (1 if i == 0 else 2), []
            for j in range(depth):
                down = None
                if j == 0 and (stride != 1 or inplanes != planes * 4):
                    down = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False), nn.BatchNorm2d(planes * 4))
                blocks.append(_SEBottleneck(block, inplanes, planes, groups, stride if j == 0 else 1, down))
                inplanes = planes * 4
            setattr(self, f"layer{i + 1}", nn.Sequential(*blocks))
        for m in self.modules():  # timm senet.py _weight_init
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def blocks(self):
        return [b for i in range(4) for b in getattr(self, f"layer{i + 1}")]


class SENetWrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm legacy SENet backbone (eval / extract only)."""

    _dropped = ("last_linear.",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, **kwargs):
        if model_name not in SENET_ARCHS:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; legacy SENets available: {sorted(SENET_ARCHS)}")
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        args = dict(SENET_ARCHS[model_name])
        if depths is not None:
            args["depths"] = tuple(depths)
        hw = image_size // 32
        super().__init__(model_name, feat_dim, image_size, SENetParams(**args), cnn_neck(2048, 2048 * hw * hw, feat_dim),
                         pretrained)

    def _build(self, p) -> BottleneckNetC:
        """vdk_bottleneck_net: BatchNorms folded once per weight version, bf16 conv weights [Cout, kh, kw, Cin] (grouped ones
        block-diagonal), the stem as zero-padded (kh, kw, c) patch rows, fp32 SE weights, the folded neck in (h, w, c) order."""
        m, net = self.model, BottleneckNetC()
        net.image_size, net.feat_dim = self.image_size, self.feat_dim
        for i in range(4):
            net.depths[i] = m.depths[i]
        resnext = m.block == "seresnext"
        net.width = (64 * 4 // 64) * m.groups if resnext else 64
        net.cardinality, net.stride_on_conv1, net.stem_pool = m.groups, int(not resnext), STEM_POOL_CEIL
        net.deep_stem, net.avg_down, net.se_reduction = 0, 0, SE_REDUCTION
        net.stem[0].w, net.stem[0].b = p.stem_rows(*fold_bn(m.layer0.conv1, m.layer0.bn1), 64)
        for i, blk in enumerate(m.blocks()):
            c = net.blocks[i]
            for dst, cv, bn in ((c.conv1, blk.conv1, blk.bn1), (c.conv2, blk.conv2, blk.bn2), (c.conv3, blk.conv3, blk.bn3)):
                w, b = fold_bn(cv, bn)
                w = pack_grouped(w) if cv.groups > 1 else w.permute(0, 2, 3, 1)
                dst.w, dst.b = p.bf16(w), p.f32(b)
            if blk.downsample is not None:
                w, b = fold_bn(blk.downsample[0], blk.downsample[1])
                c.down.w, c.down.b = p.bf16(w.permute(0, 2, 3, 1)), p.f32(b)
            se = blk.se_module
            c.se_fc1_w, c.se_fc1_b = p.f32(se.fc1.weight.flatten(1)), p.f32(se.fc1.bias)
            c.se_fc2_w, c.se_fc2_b = p.f32(se.fc2.weight.flatten(1)), p.f32(se.fc2.bias)
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net
