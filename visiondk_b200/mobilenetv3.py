"""MobileNetV3 backbones of the faceX / CBIR extract path on H100 (timm 0.9.16 mobilenetv3_large_100 / _small_100 and the
TF-ported tf_mobilenetv3_large_100 / _small_100 / _large_minimal_100 / _small_minimal_100).

`MobileNetV3Wrapper` is the reference's TimmWrapper for a `timm-[tf_]mobilenetv3_*` backbone
(models/faceX/backbone/timm_wrapper.py:16-54): timm's MobileNetV3 built with num_classes=0, global_pool='' under `model.`
and the CNN neck `output_layer.{0: BatchNorm2d, 1: Flatten, 2: Linear, 3: BatchNorm1d}`.  With global_pool='' timm's
forward_head still applies conv_head (1x1, with bias) and act2 to the unpooled map, so the neck sees [B, 1280 | 1024,
S/32, S/32].  Parameter names and shapes are timm's (`conv_stem`, `bn1`, `blocks.<stage>.<i>.{conv_dw, conv_pw, conv_pwl,
conv, se.conv_reduce, se.conv_expand, bn1-3}`, `conv_head.{weight,bias}`), so timm checkpoints load with strict=True.  The
arithmetic is csrc/mobilenetv3.cu (vdk_mobilenetv3_forward): every eval BatchNorm folded into its convolution, the 1x1
convolutions on vdk_conv2d_ex's ReLU / hard-swish epilogues, the depthwise convs and SE gates on their own kernels.
Extraction only: a train-mode forward raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C

import torch.nn as nn

from .resnet import _ConvC
from .wrapper import BackboneWrapper, cnn_neck, fold_bn

# timm 0.9.16 mobilenetv3.py _gen_mobilenet_v3 arch_def, one tuple of block strings per stage (timm's
# _efficientnet_builder._decode_block_str: kind, r repeats, k kernel, s stride, e expansion, c out channels, se ratio, nre:
# ReLU instead of the model's activation).  The minimal variants take k3 everywhere, no SE and ReLU throughout.
LARGE = (("ds_r1_k3_s1_e1_c16_nre",),
         ("ir_r1_k3_s2_e4_c24_nre", "ir_r1_k3_s1_e3_c24_nre"),
         ("ir_r3_k5_s2_e3_c40_se0.25_nre",),
         ("ir_r1_k3_s2_e6_c80", "ir_r1_k3_s1_e2.5_c80", "ir_r2_k3_s1_e2.3_c80"),
         ("ir_r2_k3_s1_e6_c112_se0.25",),
         ("ir_r3_k5_s2_e6_c160_se0.25",),
         ("cn_r1_k1_s1_c960",))
SMALL = (("ds_r1_k3_s2_e1_c16_se0.25_nre",),
         ("ir_r1_k3_s2_e4.5_c24_nre", "ir_r1_k3_s1_e3.67_c24_nre"),
         ("ir_r1_k5_s2_e4_c40_se0.25", "ir_r2_k5_s1_e6_c40_se0.25"),
         ("ir_r2_k5_s1_e3_c48_se0.25",),
         ("ir_r3_k5_s2_e6_c96_se0.25",),
         ("cn_r1_k1_s1_c576",))


def _minimal(arch):
    return tuple(tuple(b.replace("_k5", "_k3").replace("_se0.25", "") for b in stage) for stage in arch)


# stem width 16; conv_head width; the model's activation; TF "same" padding with BN eps 1e-3, or symmetric k // 2 with 1e-5
MOBILENETV3_ARCHS = {
    "tf_mobilenetv3_large_minimal_100": dict(arch=_minimal(LARGE), head=1280, act="relu", tf=True),
    "tf_mobilenetv3_large_100": dict(arch=LARGE, head=1280, act="hard_swish", tf=True),
    "tf_mobilenetv3_small_100": dict(arch=SMALL, head=1024, act="hard_swish", tf=True),
    "tf_mobilenetv3_small_minimal_100": dict(arch=_minimal(SMALL), head=1024, act="relu", tf=True),
    "mobilenetv3_large_100": dict(arch=LARGE, head=1280, act="hard_swish", tf=False),
    "mobilenetv3_small_100": dict(arch=SMALL, head=1024, act="hard_swish", tf=False),
}
STEM_CH = 16
KINDS = {"ds": 0, "ir": 1, "cn": 2}  # VDK_MNV3_DS / _IR / _CN
ACTS = {"relu": 0, "hard_swish": 1}  # VDK_ACT_RELU / _HARDSWISH


def make_divisible(v, divisor=8, round_limit=0.9):
    """timm.layers.make_divisible: the nearest multiple of `divisor`, not below 90 % of v."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < round_limit * v else new_v


def decode_blocks(arch, model_act):
    """Per block (kind, cin, cout, kernel, stride, mid, act, se_rd) in timm's order, from the stem's 16 channels."""
    out, cin = [], STEM_CH
    for stage in arch:
        specs = []
        for s in stage:
            tok = s.split("_")
            opt = {t[:2] if t.startswith("se") else t[0]: t[2:] if t.startswith("se") else t[1:] for t in tok[1:] if t != "nre"}
            act = "relu" if "nre" in tok else model_act
            for i in range(int(opt["r"])):
                cout, k, stride = int(opt["c"]), int(opt["k"]), int(opt["s"]) if i == 0 else 1
                if tok[0] == "cn":
                    mid = cout
                elif tok[0] == "ds":
                    mid = cin
                else:
                    mid = make_divisible(cin * float(opt["e"]))
                se_rd = make_divisible(mid * float(opt["se"])) if "se" in opt else 0  # se_from_exp: of the depthwise width
                specs.append((tok[0], cin, cout, k, stride, mid, act, se_rd))
                cin = cout
        out.append(specs)
    return out


class _SqueezeExcite(nn.Module):
    def __init__(self, chs, rd):
        super().__init__()
        self.conv_reduce = nn.Conv2d(chs, rd, 1)
        self.conv_expand = nn.Conv2d(rd, chs, 1)


class _Block(nn.Module):
    """timm DepthwiseSeparableConv ('ds'), InvertedResidual ('ir') or ConvBnAct ('cn') parameter containers."""

    def __init__(self, kind, cin, cout, k, stride, mid, act, se_rd, eps):
        super().__init__()
        self.kind, self.cin, self.cout, self.k, self.stride, self.mid, self.act, self.se_rd = kind, cin, cout, k, stride, mid, act, se_rd
        if kind == "cn":
            self.conv = nn.Conv2d(cin, cout, k, stride, bias=False)
            self.bn1 = nn.BatchNorm2d(cout, eps=eps)
            return
        if kind == "ir":
            self.conv_pw = nn.Conv2d(cin, mid, 1, bias=False)
            self.bn1 = nn.BatchNorm2d(mid, eps=eps)
        self.conv_dw = nn.Conv2d(mid, mid, k, stride, groups=mid, bias=False)
        if kind == "ds":
            self.bn1 = nn.BatchNorm2d(mid, eps=eps)
        else:
            self.bn2 = nn.BatchNorm2d(mid, eps=eps)
        if se_rd:
            self.se = _SqueezeExcite(mid, se_rd)
        if kind == "ds":
            self.conv_pw = nn.Conv2d(mid, cout, 1, bias=False)
            self.bn2 = nn.BatchNorm2d(cout, eps=eps)
        else:
            self.conv_pwl = nn.Conv2d(mid, cout, 1, bias=False)
            self.bn3 = nn.BatchNorm2d(cout, eps=eps)


class MobileNetV3Params(nn.Module):
    """timm 0.9.16 `MobileNetV3` (num_classes=0, global_pool='') parameter tree.  Parameter containers only: the forward is
    vdk_mobilenetv3_forward."""

    def __init__(self, arch, head, act, tf):
        super().__init__()
        eps = 1e-3 if tf else 1e-5
        self.head_ch, self.act, self.tf = head, act, tf
        self.conv_stem = nn.Conv2d(3, STEM_CH, 3, 2, bias=False)
        self.bn1 = nn.BatchNorm2d(STEM_CH, eps=eps)
        stages = decode_blocks(arch, act)
        self.blocks = nn.Sequential(*[nn.Sequential(*[_Block(*spec, eps) for spec in stage]) for stage in stages])
        self.conv_head = nn.Conv2d(stages[-1][-1][2], head, 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)


class _Mnv3BlockC(C.Structure):
    _fields_ = [("kind", C.c_int), ("kernel", C.c_int), ("stride", C.c_int), ("cin", C.c_int), ("mid", C.c_int),
                ("cout", C.c_int), ("act", C.c_int), ("se_rd", C.c_int), ("conv", _ConvC), ("dw_w", C.c_void_p),
                ("dw_b", C.c_void_p), ("se_w1", C.c_void_p), ("se_b1", C.c_void_p), ("se_w2", C.c_void_p),
                ("se_b2", C.c_void_p), ("conv_pwl", _ConvC)]


MAX_BLOCKS = 24


class MobileNetV3NetC(C.Structure):
    """vdk_mobilenetv3_net (include/vdk_b200.h)."""
    api = "vdk_mobilenetv3"
    _fields_ = [("image_size", C.c_int), ("feat_dim", C.c_int), ("num_blocks", C.c_int), ("pad", C.c_int),
                ("stem_ch", C.c_int), ("stem_act", C.c_int), ("head_ch", C.c_int), ("head_act", C.c_int), ("stem", _ConvC),
                ("blocks", _Mnv3BlockC * MAX_BLOCKS), ("head", _ConvC), ("neck_w", C.c_void_p), ("neck_b", C.c_void_p)]


class MobileNetV3Wrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper with a timm MobileNetV3 backbone (eval / extract
    only)."""

    _dropped = ("classifier.",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, **kwargs):
        if model_name not in MOBILENETV3_ARCHS:
            raise ValueError(f"backbone '{model_name}' is not built for H100 yet; MobileNetV3s available: {sorted(MOBILENETV3_ARCHS)}")
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        hw, head = image_size // 32, MOBILENETV3_ARCHS[model_name]["head"]
        super().__init__(model_name, feat_dim, image_size, MobileNetV3Params(**MOBILENETV3_ARCHS[model_name]),
                         cnn_neck(head, head * hw * hw, feat_dim), pretrained)

    def _build(self, p) -> MobileNetV3NetC:
        """vdk_mobilenetv3_net: BatchNorms folded once per weight version; bf16 1x1 weights [out, in], the stem as zero-padded
        (kh, kw, c) patch rows [16, 64], fp32 depthwise taps [k*k, mid] and SE weights, the folded neck in (h, w, c) order."""
        def conv(dst, w, b):
            dst.w, dst.b = p.bf16(w.reshape(w.shape[0], -1)), p.f32(b)

        m, net = self.model, MobileNetV3NetC()
        net.image_size, net.feat_dim, net.pad = self.image_size, self.feat_dim, 0 if m.tf else 1
        net.stem_ch, net.head_ch, net.stem_act = STEM_CH, m.head_ch, ACTS[m.act]
        net.head_act = ACTS[m.act]
        net.stem.w, net.stem.b = p.stem_rows(*fold_bn(m.conv_stem, m.bn1), 64)
        blocks = [blk for stage in m.blocks for blk in stage]
        if len(blocks) > MAX_BLOCKS:
            raise ValueError(f"{len(blocks)} blocks exceed vdk_mobilenetv3_net's {MAX_BLOCKS}")
        net.num_blocks = len(blocks)
        for i, blk in enumerate(blocks):
            c = net.blocks[i]
            c.kind, c.kernel, c.stride, c.cin, c.mid, c.cout = KINDS[blk.kind], blk.k, blk.stride, blk.cin, blk.mid, blk.cout
            c.act, c.se_rd = ACTS[blk.act], blk.se_rd
            if blk.kind == "cn":
                conv(c.conv, *fold_bn(blk.conv, blk.bn1))
                continue
            if blk.kind == "ir":
                conv(c.conv, *fold_bn(blk.conv_pw, blk.bn1))
                w, b = fold_bn(blk.conv_dw, blk.bn2)
                conv(c.conv_pwl, *fold_bn(blk.conv_pwl, blk.bn3))
            else:
                w, b = fold_bn(blk.conv_dw, blk.bn1)
                conv(c.conv_pwl, *fold_bn(blk.conv_pw, blk.bn2))
            c.dw_w, c.dw_b = p.f32(w.reshape(blk.mid, blk.k * blk.k).t()), p.f32(b)
            if blk.se_rd:
                se = blk.se
                c.se_w1, c.se_b1 = p.f32(se.conv_reduce.weight.flatten(1)), p.f32(se.conv_reduce.bias)
                c.se_w2, c.se_b2 = p.f32(se.conv_expand.weight.flatten(1)), p.f32(se.conv_expand.bias)
        conv(net.head, m.conv_head.weight.detach().float(), m.conv_head.bias.detach().float())
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net
