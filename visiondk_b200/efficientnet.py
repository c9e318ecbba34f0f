"""EfficientNetV2 backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 tf_efficientnetv2_s / _m / _l).

`EfficientNetV2Wrapper` is the reference's TimmWrapper for a `timm-tf_efficientnetv2_*` backbone
(models/faceX/backbone/timm_wrapper.py:16-54): timm's EfficientNet built with num_classes=0, global_pool='' under `model.`
and the CNN neck `output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear, 3: BatchNorm1d}`.  Parameter names and shapes are
timm's (`conv_stem`, `bn1`, `blocks.<stage>.<i>.{conv, conv_exp, conv_pw, conv_dw, se.conv_reduce, se.conv_expand,
conv_pwl, bn1-3}`, `conv_head`, `bn2`), so timm checkpoints load with strict=True.  The arithmetic is csrc/effnet.cu
(vdk_effnetv2_forward): every eval BatchNorm folded into its convolution, the dense convolutions on vdk_conv2d_ex with
TF-"same" padding, the depthwise convs and SE gates on their own kernels.  Extraction only: a train-mode forward raises
NotImplementedError.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .resnet import _ConvC
from .wrapper import BackboneWrapper, cnn_neck, fold_bn

# timm 0.9.16 efficientnet.py _gen_efficientnetv2_{s,m,l} arch_def: per stage (kind, repeats, stride, expansion, out
# channels); every `ir` stage has se0.25 of the block's input width.  stem width, conv_head width 1280, BN eps 1e-3.
EFFNETV2_ARCHS = {
    "tf_efficientnetv2_s": dict(stem=24, stages=(("cn", 2, 1, 1, 24), ("er", 4, 2, 4, 48), ("er", 4, 2, 4, 64),
                                                 ("ir", 6, 2, 4, 128), ("ir", 9, 1, 6, 160), ("ir", 15, 2, 6, 256))),
    "tf_efficientnetv2_m": dict(stem=24, stages=(("cn", 3, 1, 1, 24), ("er", 5, 2, 4, 48), ("er", 5, 2, 4, 80),
                                                 ("ir", 7, 2, 4, 160), ("ir", 14, 1, 6, 176), ("ir", 18, 2, 6, 304),
                                                 ("ir", 5, 1, 6, 512))),
    "tf_efficientnetv2_l": dict(stem=32, stages=(("cn", 4, 1, 1, 32), ("er", 7, 2, 4, 64), ("er", 7, 2, 4, 96),
                                                 ("ir", 10, 2, 4, 192), ("ir", 19, 1, 6, 224), ("ir", 25, 2, 6, 384),
                                                 ("ir", 7, 1, 6, 640))),
}
HEAD_CH = 1280
BN_EPS = 1e-3
KINDS = {"cn": 0, "er": 1, "ir": 2}  # VDK_EFFNET_CN / _ER / _IR


def _bn(c):
    return nn.BatchNorm2d(c, eps=BN_EPS)


class _SqueezeExcite(nn.Module):
    def __init__(self, chs, rd):
        super().__init__()
        self.conv_reduce = nn.Conv2d(chs, rd, 1)
        self.conv_expand = nn.Conv2d(rd, chs, 1)


class _Block(nn.Module):
    """timm ConvBnAct ('cn'), EdgeResidual ('er') or InvertedResidual ('ir') parameter containers."""

    def __init__(self, kind, cin, cout, stride, exp):
        super().__init__()
        self.kind, self.cin, self.cout, self.stride = kind, cin, cout, stride
        self.mid = cin * exp if kind != "cn" else cout
        self.has_skip = stride == 1 and cin == cout
        if kind == "cn":
            self.conv = nn.Conv2d(cin, cout, 3, stride, bias=False)
            self.bn1 = _bn(cout)
        elif kind == "er":
            self.conv_exp = nn.Conv2d(cin, self.mid, 3, stride, bias=False)
            self.bn1 = _bn(self.mid)
            self.conv_pwl = nn.Conv2d(self.mid, cout, 1, bias=False)
            self.bn2 = _bn(cout)
        else:
            self.conv_pw = nn.Conv2d(cin, self.mid, 1, bias=False)
            self.bn1 = _bn(self.mid)
            self.conv_dw = nn.Conv2d(self.mid, self.mid, 3, stride, groups=self.mid, bias=False)
            self.bn2 = _bn(self.mid)
            self.se = _SqueezeExcite(self.mid, round(cin / 4))
            self.conv_pwl = nn.Conv2d(self.mid, cout, 1, bias=False)
            self.bn3 = _bn(cout)


def build_blocks(stem, stages, depths=None) -> nn.Sequential:
    """timm's `blocks` Sequential of stage Sequentials; `depths` overrides the repeats (toy-depth tests)."""
    cin, out = stem, nn.Sequential()
    for s, (kind, reps, stride, exp, cout) in enumerate(stages):
        n = reps if depths is None else depths[s]
        stage = nn.Sequential(*[_Block(kind, cin if i == 0 else cout, cout, stride if i == 0 else 1, exp) for i in range(n)])
        out.add_module(str(s), stage)
        cin = cout
    return out


class EfficientNetV2Params(nn.Module):
    """timm 0.9.16 `EfficientNet` (tf_efficientnetv2_*, num_classes=0, global_pool='') parameter tree.  Parameter containers
    only: the forward is vdk_effnetv2_forward."""

    def __init__(self, stem, stages, depths=None):
        super().__init__()
        self.stem_ch, self.stages = stem, stages
        self.conv_stem = nn.Conv2d(3, stem, 3, 2, bias=False)
        self.bn1 = _bn(stem)
        self.blocks = build_blocks(stem, stages, depths)
        self.conv_head = nn.Conv2d(stages[-1][4], HEAD_CH, 1, bias=False)
        self.bn2 = _bn(HEAD_CH)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")


class _EffBlockC(C.Structure):
    _fields_ = [("kind", C.c_int), ("stride", C.c_int), ("cin", C.c_int), ("cout", C.c_int), ("mid", C.c_int),
                ("se_rd", C.c_int), ("conv", _ConvC), ("dw_w", C.c_void_p), ("dw_b", C.c_void_p), ("se_w1", C.c_void_p),
                ("se_b1", C.c_void_p), ("se_w2", C.c_void_p), ("se_b2", C.c_void_p), ("conv_pwl", _ConvC)]


MAX_BLOCKS = 80


class EffNetV2NetC(C.Structure):
    """vdk_effnetv2_net (include/vdk_b200.h)."""
    api = "vdk_effnetv2"
    _fields_ = [("image_size", C.c_int), ("feat_dim", C.c_int), ("num_blocks", C.c_int), ("stem_ch", C.c_int),
                ("head_ch", C.c_int), ("stem", _ConvC), ("blocks", _EffBlockC * MAX_BLOCKS), ("head", _ConvC),
                ("neck_w", C.c_void_p), ("neck_b", C.c_void_p)]


class ConvExDesc(C.Structure):
    """vdk_conv_ex_desc (include/vdk_b200.h)."""
    _fields_ = [("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("residual", C.c_void_p), ("y", C.c_void_p),
                ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("Cout", C.c_int), ("kernel", C.c_int),
                ("stride", C.c_int), ("pad_h_lo", C.c_int), ("pad_h_hi", C.c_int), ("pad_w_lo", C.c_int),
                ("pad_w_hi", C.c_int), ("epilogue", C.c_int)]


def pack_conv_ex(w: torch.Tensor) -> torch.Tensor:
    """Conv weight [Cout, Cin, k, k] -> vdk_conv2d_ex's layout: [Cout, Cin] for 1x1, else [Cout, k, k, Cinp] with the
    channels zero-padded to Cinp = Cin rounded up to 64."""
    cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
    if k == 1:
        return w.reshape(cout, cin)
    cinp = (cin + 63) // 64 * 64
    out = w.new_zeros(cout, k, k, cinp)
    out[..., :cin] = w.permute(0, 2, 3, 1)
    return out


class EfficientNetV2Wrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm tf_efficientnetv2 backbone (eval /
    extract only)."""

    _dropped = ("classifier.",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, **kwargs):
        if model_name not in EFFNETV2_ARCHS:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; EfficientNetV2s available: {sorted(EFFNETV2_ARCHS)}")
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        hw = image_size // 32
        super().__init__(model_name, feat_dim, image_size, EfficientNetV2Params(**EFFNETV2_ARCHS[model_name], depths=depths),
                         cnn_neck(HEAD_CH, HEAD_CH * hw * hw, feat_dim), pretrained)

    def _build(self, p) -> EffNetV2NetC:
        """vdk_effnetv2_net: BatchNorms folded once per weight version; bf16 conv weights in vdk_conv2d_ex's layouts, the stem
        as zero-padded (kh, kw, c) patch rows [stem, 64], fp32 depthwise taps [9, mid] and SE weights, the folded neck in
        (h, w, c) order."""
        def conv(dst, w, b):
            dst.w, dst.b = p.bf16(pack_conv_ex(w)), p.f32(b)

        m, net = self.model, EffNetV2NetC()
        net.image_size, net.feat_dim, net.stem_ch, net.head_ch = self.image_size, self.feat_dim, m.stem_ch, HEAD_CH
        net.stem.w, net.stem.b = p.stem_rows(*fold_bn(m.conv_stem, m.bn1), 64)
        blocks = [blk for stage in m.blocks for blk in stage]
        if len(blocks) > MAX_BLOCKS:
            raise ValueError(f"{len(blocks)} blocks exceed vdk_effnetv2_net's {MAX_BLOCKS}")
        net.num_blocks = len(blocks)
        for i, blk in enumerate(blocks):
            c = net.blocks[i]
            c.kind, c.stride, c.cin, c.cout, c.mid = KINDS[blk.kind], blk.stride, blk.cin, blk.cout, blk.mid
            if blk.kind == "cn":
                conv(c.conv, *fold_bn(blk.conv, blk.bn1))
            elif blk.kind == "er":
                conv(c.conv, *fold_bn(blk.conv_exp, blk.bn1))
                conv(c.conv_pwl, *fold_bn(blk.conv_pwl, blk.bn2))
            else:
                conv(c.conv, *fold_bn(blk.conv_pw, blk.bn1))
                w, b = fold_bn(blk.conv_dw, blk.bn2)
                c.dw_w, c.dw_b = p.f32(w.reshape(blk.mid, 9).t()), p.f32(b)
                se = blk.se
                c.se_rd = se.conv_reduce.out_channels
                c.se_w1, c.se_b1 = p.f32(se.conv_reduce.weight.flatten(1)), p.f32(se.conv_reduce.bias)
                c.se_w2, c.se_b2 = p.f32(se.conv_expand.weight.flatten(1)), p.f32(se.conv_expand.bias)
                conv(c.conv_pwl, *fold_bn(blk.conv_pwl, blk.bn3))
        conv(net.head, *fold_bn(m.conv_head, m.bn2))
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net
