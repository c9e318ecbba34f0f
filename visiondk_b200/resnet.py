"""ResNet backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 Bottleneck ResNets and ResNeXts).

`ResNetWrapper` is the reference's TimmWrapper for a `timm-resnet*` / `timm-wide_resnet*` / `timm-resnext*` backbone
(models/faceX/backbone/timm_wrapper.py:16-54): the timm ResNet built with num_classes=0, global_pool='' under `model.`
and the CNN neck `output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear, 3: BatchNorm1d}`; parameter names and shapes are
timm's, so timm checkpoints load with strict=True.  The arithmetic is csrc/resnet.cu (vdk_resnet_forward): every eval
BatchNorm folded into its convolution, the convolutions on the wgmma GEMM (implicit GEMM with TMA im2col tiles).  ResNeXts
run through vdk_bottleneck_forward, their grouped 3x3 convs on vdk_conv2d_grouped with block-diagonal weights.
Extraction only: a train-mode forward raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from .wrapper import BackboneWrapper, cnn_neck, fold_bn

# timm 0.9.16 resnet.py model_args; all Bottleneck (stride on the 3x3 conv, expansion 4)
RESNET_ARCHS = {
    "resnet50": dict(depths=(3, 4, 6, 3)),
    "resnet101": dict(depths=(3, 4, 23, 3)),
    "resnet152": dict(depths=(3, 8, 36, 3)),
    "resnet50d": dict(depths=(3, 4, 6, 3), stem_width=32, stem_type="deep", avg_down=True),
    "resnet101d": dict(depths=(3, 4, 23, 3), stem_width=32, stem_type="deep", avg_down=True),
    "resnet152d": dict(depths=(3, 8, 36, 3), stem_width=32, stem_type="deep", avg_down=True),
    "wide_resnet50_2": dict(depths=(3, 4, 6, 3), base_width=128),
    "wide_resnet101_2": dict(depths=(3, 4, 23, 3), base_width=128),
}
# timm 0.9.16 resnet.py ResNeXt model_args: the 3x3 conv has `cardinality` groups of `base_width` * 2^stage channels
RESNEXT_ARCHS = {
    "resnext50_32x4d": dict(depths=(3, 4, 6, 3), cardinality=32, base_width=4),
    "resnext50d_32x4d": dict(depths=(3, 4, 6, 3), cardinality=32, base_width=4, stem_width=32, stem_type="deep", avg_down=True),
    "resnext101_32x8d": dict(depths=(3, 4, 23, 3), cardinality=32, base_width=8),
    "resnext101_64x4d": dict(depths=(3, 4, 23, 3), cardinality=64, base_width=4),
}


class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, downsample, base_width, cardinality=1):
        super().__init__()
        width = int(math.floor(planes * (base_width / 64)) * cardinality)
        self.stride = stride
        self.conv1 = nn.Conv2d(inplanes, width, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, 3, stride=stride, padding=1, groups=cardinality, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample


class ResNetParams(nn.Module):
    """timm 0.9.16 `ResNet(Bottleneck, ..., num_classes=0, global_pool='')` parameter tree.  Parameter containers only:
    their forward() is never used (the forward is vdk_resnet_forward)."""

    def __init__(self, depths, base_width=64, stem_width=64, stem_type="", avg_down=False, cardinality=1):
        super().__init__()
        self.depths, self.base_width, self.avg_down = tuple(depths), int(base_width), bool(avg_down)
        self.cardinality = int(cardinality)
        self.deep_stem = "deep" in stem_type
        inplanes = stem_width * 2 if self.deep_stem else 64
        if self.deep_stem:
            self.conv1 = nn.Sequential(
                nn.Conv2d(3, stem_width, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(stem_width), nn.ReLU(),
                nn.Conv2d(stem_width, stem_width, 3, padding=1, bias=False), nn.BatchNorm2d(stem_width), nn.ReLU(),
                nn.Conv2d(stem_width, inplanes, 3, padding=1, bias=False))
        else:
            self.conv1 = nn.Conv2d(3, inplanes, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(inplanes)
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride, blocks = (1 if i == 0 else 2), []
            for j in range(depth):
                down = None
                if j == 0 and (stride != 1 or inplanes != planes * 4):
                    conv, bn = nn.Conv2d(inplanes, planes * 4, 1, stride=1 if avg_down else stride, bias=False), nn.BatchNorm2d(planes * 4)
                    if avg_down:
                        pool = nn.AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False) if stride != 1 else nn.Identity()
                        down = nn.Sequential(pool, conv, bn)
                    else:
                        down = nn.Sequential(conv, bn)
                blocks.append(_Bottleneck(inplanes, planes, stride if j == 0 else 1, down, base_width, cardinality))
                inplanes = planes * 4
            setattr(self, f"layer{i + 1}", nn.Sequential(*blocks))
        # timm's init: kaiming_normal(fan_out, relu) convs, unit BatchNorms, bn3.weight zeroed (zero_init_last)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        for blk in self.blocks():
            nn.init.zeros_(blk.bn3.weight)

    def blocks(self):
        return [b for i in range(4) for b in getattr(self, f"layer{i + 1}")]


class _ConvC(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p)]


class _ResBlockC(C.Structure):
    _fields_ = [("conv1", _ConvC), ("conv2", _ConvC), ("conv3", _ConvC), ("down", _ConvC)]


class ResNetNetC(C.Structure):
    """vdk_resnet_net (include/vdk_b200.h)."""
    api = "vdk_resnet"  # prefix of the network's workspace / forward entry points
    _fields_ = [
        ("image_size", C.c_int), ("feat_dim", C.c_int), ("depths", C.c_int * 4), ("base_width", C.c_int),
        ("deep_stem", C.c_int), ("avg_down", C.c_int), ("stem", _ConvC * 3), ("blocks", _ResBlockC * 64),
        ("neck_w", C.c_void_p), ("neck_b", C.c_void_p),
    ]


class _BottleneckBlockC(C.Structure):
    _fields_ = [("conv1", _ConvC), ("conv2", _ConvC), ("conv3", _ConvC), ("down", _ConvC),
                ("se_fc1_w", C.c_void_p), ("se_fc1_b", C.c_void_p), ("se_fc2_w", C.c_void_p), ("se_fc2_b", C.c_void_p)]


class BottleneckNetC(C.Structure):
    """vdk_bottleneck_net (include/vdk_b200.h)."""
    api = "vdk_bottleneck"
    _fields_ = [
        ("image_size", C.c_int), ("feat_dim", C.c_int), ("depths", C.c_int * 4), ("width", C.c_int), ("cardinality", C.c_int),
        ("stride_on_conv1", C.c_int), ("stem_pool", C.c_int), ("deep_stem", C.c_int), ("avg_down", C.c_int),
        ("se_reduction", C.c_int), ("stem", _ConvC * 3), ("blocks", _BottleneckBlockC * 64), ("neck_w", C.c_void_p),
        ("neck_b", C.c_void_p),
    ]


STEM_POOL_PAD1, STEM_POOL_CEIL = 0, 1


def pack_grouped(w: torch.Tensor) -> torch.Tensor:
    """timm's grouped conv weight [Cout, Cout / groups, k, k] -> vdk_conv2d_grouped's block-diagonal [Cout, k, k, 128]:
    output channel n of group g = n // cg sits in the 128-channel tile t = n // 128, and its cg input channels go to tile
    columns g*cg - 128*t .. + cg; every other column is zero."""
    cout, cg, k = w.shape[0], w.shape[1], w.shape[2]
    start = (torch.arange(cout, device=w.device) // cg * cg) % 128
    cols = (start[:, None] + torch.arange(cg, device=w.device)[None, :])[:, None, :].expand(cout, k * k, cg)
    out = w.new_zeros(cout, k * k, 128)
    out.scatter_(2, cols, w.permute(0, 2, 3, 1).reshape(cout, k * k, cg))
    return out.view(cout, k, k, 128)


class ResNetWrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm ResNet backbone (eval / extract only)."""

    _dropped = ("fc.",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, **kwargs):
        archs = {**RESNET_ARCHS, **RESNEXT_ARCHS}
        if model_name not in archs:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; ResNets available: {sorted(archs)}")
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        args = dict(archs[model_name])
        if depths is not None:
            args["depths"] = tuple(depths)
        hw = image_size // 32
        super().__init__(model_name, feat_dim, image_size, ResNetParams(**args), cnn_neck(2048, 2048 * hw * hw, feat_dim),
                         pretrained)

    def _build(self, p) -> ResNetNetC:
        """Kernel-side layouts (include/vdk_b200.h): BatchNorms folded once per weight version, bf16 conv weights
        [Cout, kh, kw, Cin], stem weights as zero-padded (kh, kw, c) patch rows, the folded neck in (h, w, c) order."""
        def conv(dst, w, b, pool2=False):
            w = w.permute(0, 2, 3, 1)  # [Cout, kh, kw, Cin]
            if pool2:  # AvgPool2d(2, 2) then the 1x1 conv == a 2x2/s2 conv with w / 4 at every tap
                w = w.expand(-1, 2, 2, -1) / 4
            dst.w, dst.b = p.bf16(w), p.f32(b)

        m = self.model
        net = ResNetNetC() if m.cardinality == 1 else BottleneckNetC()
        net.image_size, net.feat_dim = self.image_size, self.feat_dim
        for i in range(4):
            net.depths[i] = m.depths[i]
        net.deep_stem, net.avg_down = int(m.deep_stem), int(m.avg_down)
        if m.cardinality == 1:
            net.base_width = m.base_width
        else:
            net.width, net.cardinality, net.stem_pool = m.base_width * m.cardinality, m.cardinality, STEM_POOL_PAD1
        if m.deep_stem:
            net.stem[0].w, net.stem[0].b = p.stem_rows(*fold_bn(m.conv1[0], m.conv1[1]), 64)
            net.stem[1].w, net.stem[1].b = p.stem_rows(*fold_bn(m.conv1[3], m.conv1[4]), 64)
            net.stem[2].w, net.stem[2].b = p.stem_rows(*fold_bn(m.conv1[6], m.bn1), 64)
        else:
            net.stem[0].w, net.stem[0].b = p.stem_rows(*fold_bn(m.conv1, m.bn1), 64)
        for i, blk in enumerate(m.blocks()):
            b = net.blocks[i]
            conv(b.conv1, *fold_bn(blk.conv1, blk.bn1))
            if m.cardinality == 1:
                conv(b.conv2, *fold_bn(blk.conv2, blk.bn2))
            else:
                w, bias = fold_bn(blk.conv2, blk.bn2)
                b.conv2.w, b.conv2.b = p.bf16(pack_grouped(w)), p.f32(bias)
            conv(b.conv3, *fold_bn(blk.conv3, blk.bn3))
            if blk.downsample is not None:
                if m.avg_down:
                    conv(b.down, *fold_bn(blk.downsample[1], blk.downsample[2]), pool2=blk.stride == 2)
                else:
                    conv(b.down, *fold_bn(blk.downsample[0], blk.downsample[1]))
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net
