"""ResNeSt backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 timm/models/resnest.py, timm/layers/split_attn.py).

`ResNeStWrapper` is the reference's TimmWrapper for a `timm-resnest*` backbone (models/faceX/backbone/timm_wrapper.py:16-54):
the timm ResNet with ResNestBottleneck blocks built with num_classes=0, global_pool='' under `model.` and the CNN neck
`output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear, 3: BatchNorm1d}`.  Parameter names and shapes are timm's
(`layerN.i.conv2.{conv, bn0, fc1, bn1, fc2}`, the deep stem `conv1.{0,1,3,4,6}`, avg_down `downsample.{1,2}`), so timm
checkpoints load with strict=True.  The arithmetic is csrc/resnest.cu (vdk_resnest_forward): every eval BatchNorm folded
into the conv before it (bn1 of the attention into fc1), the split conv on vdk_conv2d_grouped_ex, the split-attention gate
in fp32.  Extraction only: a train-mode forward raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .resnet import _ConvC
from .wrapper import BackboneWrapper, cnn_neck, fold_bn

# timm 0.9.16 resnest.py model_args: deep stem of width 32, avg_down shortcuts, avd (the stride-2 3x3 average pool)
RESNEST_ARCHS = {
    "resnest14d": dict(depths=(1, 1, 1, 1), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest26d": dict(depths=(2, 2, 2, 2), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest50d": dict(depths=(3, 4, 6, 3), radix=2, cardinality=1, base_width=64, avd_first=False),
    "resnest50d_1s4x24d": dict(depths=(3, 4, 6, 3), radix=1, cardinality=4, base_width=24, avd_first=True),
    "resnest50d_4s2x40d": dict(depths=(3, 4, 6, 3), radix=4, cardinality=2, base_width=40, avd_first=True),
}


def make_divisible(v, divisor=8, min_value=None, round_limit=0.9):
    """timm/layers/helpers.py make_divisible: the SplitAttn attention width."""
    min_value = min_value or divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < round_limit * v:
        new_v += divisor
    return new_v


def group_width(planes, base_width, cardinality):
    return int(planes * (base_width / 64.0)) * cardinality


def attn_width(gw, radix):
    return make_divisible(gw * radix * 0.25, min_value=32, divisor=8)


def split_tile_start(n0, cgi, cgo):
    """First input channel c_lo of the output tile at n0: its first group's, rounded down to a multiple of 8 (16 bytes)."""
    return n0 // cgo * cgi // 8 * 8


def split_conv_blocks(cin, cout, groups):
    """64-channel blocks per tap of vdk_conv2d_grouped_ex's packed weight (include/vdk_b200.h): the widest input-channel
    span, from c_lo, of the groups one 128-channel output tile covers."""
    cgi, cgo = cin // groups, cout // groups
    return max(-(-(((min(n0 + 128, cout) - 1) // cgo + 1) * cgi - split_tile_start(n0, cgi, cgo)) // 64)
               for n0 in range(0, cout, 128))


def pack_split(w: torch.Tensor, groups: int) -> torch.Tensor:
    """timm's grouped conv weight [Cout, Cin / groups, k, k] -> vdk_conv2d_grouped_ex's [Cout, k, k, cpb * 64]: output
    channel n of group g = n // cgo in tile t = n // 128 holds its cgi input channels at columns g cgi - c_lo(t) ..
    (split_tile_start); every other column is zero."""
    cout, cgi, k = w.shape[0], w.shape[1], w.shape[2]
    cgo = cout // groups
    cpb = split_conv_blocks(cgi * groups, cout, groups)
    n = torch.arange(cout, device=w.device)
    start = n // cgo * cgi - split_tile_start(n // 128 * 128, cgi, cgo)
    cols = (start[:, None] + torch.arange(cgi, device=w.device)[None, :])[:, None, :].expand(cout, k * k, cgi)
    out = w.new_zeros(cout, k * k, cpb * 64)
    out.scatter_(2, cols, w.permute(0, 2, 3, 1).reshape(cout, k * k, cgi))
    return out.view(cout, k, k, cpb * 64)


class _SplitAttn(nn.Module):
    def __init__(self, gw, radix, cardinality):
        super().__init__()
        attn = attn_width(gw, radix)
        self.radix, self.cardinality = radix, cardinality
        self.conv = nn.Conv2d(gw, gw * radix, 3, padding=1, groups=cardinality * radix, bias=False)
        self.bn0 = nn.BatchNorm2d(gw * radix)
        self.fc1 = nn.Conv2d(gw, attn, 1, groups=cardinality)
        self.bn1 = nn.BatchNorm2d(attn)
        self.fc2 = nn.Conv2d(attn, gw * radix, 1, groups=cardinality)


class _ResNestBottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, downsample, radix, cardinality, base_width):
        super().__init__()
        gw = group_width(planes, base_width, cardinality)
        self.stride = stride
        self.conv1 = nn.Conv2d(inplanes, gw, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(gw)
        self.conv2 = _SplitAttn(gw, radix, cardinality)
        self.conv3 = nn.Conv2d(gw, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample


class ResNeStParams(nn.Module):
    """timm 0.9.16 `ResNet(ResNestBottleneck, ..., stem_type='deep', stem_width=32, avg_down=True, num_classes=0,
    global_pool='')` parameter tree.  Parameter containers only: the forward is vdk_resnest_forward."""

    def __init__(self, depths, radix, cardinality, base_width, avd_first):
        super().__init__()
        self.depths, self.radix, self.cardinality = tuple(depths), int(radix), int(cardinality)
        self.base_width, self.avd_first = int(base_width), bool(avd_first)
        self.conv1 = nn.Sequential(
            nn.Conv2d(3, 32, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(),
            nn.Conv2d(32, 32, 3, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(),
            nn.Conv2d(32, 64, 3, padding=1, bias=False))
        self.bn1 = nn.BatchNorm2d(64)
        inplanes = 64
        for i, (planes, depth) in enumerate(zip((64, 128, 256, 512), depths)):
            stride, blocks = (1 if i == 0 else 2), []
            for j in range(depth):
                down = None
                if j == 0 and (stride != 1 or inplanes != planes * 4):
                    pool = nn.AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False) if stride != 1 else nn.Identity()
                    down = nn.Sequential(pool, nn.Conv2d(inplanes, planes * 4, 1, bias=False), nn.BatchNorm2d(planes * 4))
                blocks.append(_ResNestBottleneck(inplanes, planes, stride if j == 0 else 1, down, radix, cardinality, base_width))
                inplanes = planes * 4
            setattr(self, f"layer{i + 1}", nn.Sequential(*blocks))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def blocks(self):
        return [b for i in range(4) for b in getattr(self, f"layer{i + 1}")]


class _ResNestBlockC(C.Structure):
    _fields_ = [("conv1", _ConvC), ("conv2", _ConvC), ("fc1_w", C.c_void_p), ("fc1_b", C.c_void_p), ("fc2_w", C.c_void_p),
                ("fc2_b", C.c_void_p), ("conv3", _ConvC), ("down", _ConvC)]


class ResNeStNetC(C.Structure):
    """vdk_resnest_net (include/vdk_b200.h)."""
    api = "vdk_resnest"
    _fields_ = [
        ("image_size", C.c_int), ("feat_dim", C.c_int), ("depths", C.c_int * 4), ("radix", C.c_int), ("cardinality", C.c_int),
        ("base_width", C.c_int), ("avd_first", C.c_int), ("attn", C.c_int * 4), ("stem", _ConvC * 3),
        ("blocks", _ResNestBlockC * 64), ("neck_w", C.c_void_p), ("neck_b", C.c_void_p),
    ]


class ResNeStWrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm ResNeSt backbone (eval / extract only)."""

    _dropped = ("fc.",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, **kwargs):
        if model_name not in RESNEST_ARCHS:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; ResNeSts available: {sorted(RESNEST_ARCHS)}")
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        args = dict(RESNEST_ARCHS[model_name])
        if depths is not None:
            args["depths"] = tuple(depths)
        hw = image_size // 32
        super().__init__(model_name, feat_dim, image_size, ResNeStParams(**args), cnn_neck(2048, 2048 * hw * hw, feat_dim),
                         pretrained)

    def _build(self, p) -> ResNeStNetC:
        """vdk_resnest_net: BatchNorms folded in fp32 once per weight version, bf16 conv weights [Cout, kh, kw, Cin] (the split
        conv in vdk_conv2d_grouped_ex's layout), the deep stem as zero-padded (kh, kw, c) patch rows, fp32 attention weights,
        the folded neck in (h, w, c) order."""
        m, net = self.model, ResNeStNetC()
        net.image_size, net.feat_dim = self.image_size, self.feat_dim
        net.radix, net.cardinality, net.base_width, net.avd_first = m.radix, m.cardinality, m.base_width, int(m.avd_first)
        for i in range(4):
            net.depths[i] = m.depths[i]
            net.attn[i] = attn_width(group_width(64 << i, m.base_width, m.cardinality), m.radix)
        net.stem[0].w, net.stem[0].b = p.stem_rows(*fold_bn(m.conv1[0], m.conv1[1]), 64)
        net.stem[1].w, net.stem[1].b = p.stem_rows(*fold_bn(m.conv1[3], m.conv1[4]), 64)
        net.stem[2].w, net.stem[2].b = p.stem_rows(*fold_bn(m.conv1[6], m.bn1), 64)
        for i, blk in enumerate(m.blocks()):
            c, sa = net.blocks[i], blk.conv2
            w, b = fold_bn(blk.conv1, blk.bn1)
            c.conv1.w, c.conv1.b = p.bf16(w.flatten(1)), p.f32(b)
            w, b = fold_bn(sa.conv, sa.bn0)
            c.conv2.w, c.conv2.b = p.bf16(pack_split(w, sa.conv.groups)), p.f32(b)
            s = sa.bn1.weight.detach().float() / torch.sqrt(sa.bn1.running_var.detach().float() + sa.bn1.eps)
            c.fc1_w = p.f32(sa.fc1.weight.detach().float().flatten(1) * s[:, None])
            c.fc1_b = p.f32((sa.fc1.bias.detach().float() - sa.bn1.running_mean.detach().float()) * s + sa.bn1.bias.detach().float())
            c.fc2_w, c.fc2_b = p.f32(sa.fc2.weight.flatten(1)), p.f32(sa.fc2.bias)
            w, b = fold_bn(blk.conv3, blk.bn3)
            c.conv3.w, c.conv3.b = p.bf16(w.flatten(1)), p.f32(b)
            if blk.downsample is not None:
                w, b = fold_bn(blk.downsample[1], blk.downsample[2])
                w = w.permute(0, 2, 3, 1)
                if blk.stride == 2:  # AvgPool2d(2, 2) then the 1x1 conv == a 2x2/s2 conv with w / 4 at every tap
                    w = w.expand(-1, 2, 2, -1) / 4
                c.down.w, c.down.b = p.bf16(w), p.f32(b)
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net
