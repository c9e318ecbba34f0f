"""Backbone seam of the faceX / CBIR path on H100 (SURVEY.md §8b, Seam 1).

The reference builds `TimmWrapper(model_name, feat_dim, image_size, pretrained)` in
models/faceX/backbone/backbone_def.py:16-26 (config key `timm-<name>`), i.e. a timm backbone created with
num_classes=0 / global_pool='' plus the neck BatchNorm2d -> Flatten -> Linear -> BatchNorm1d
(models/faceX/backbone/timm_wrapper.py:16-49), `forward(x[B,3,S,S]) -> [B, feat_dim]` (:51-54) and
state_dict prefixes `model.` / `output_layer.`.

This module keeps exactly that surface (constructor arguments, parameter names and shapes — timm 0.9.16
ConvNeXt checkpoints and the reference's Epoch_N.pt `state_dict` / `ema` entries load with strict=True) but the
arithmetic is the hand-written sm_90a path: vdk_convnext_forward in csrc/convnext.cu (wgmma GEMMs with fused
LayerNorm / GELU / layer-scale+residual epilogues, NHWC bf16 activations).  The nn.Module children below are
parameter containers only; their own forward() is never used on the hot path, and there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .wrapper import BackboneWrapper, cnn_neck

CONVNEXT_ARCHS = {
    "convnext_atto": ((2, 2, 6, 2), (40, 80, 160, 320)),
    "convnext_femto": ((2, 2, 6, 2), (48, 96, 192, 384)),
    "convnext_pico": ((2, 2, 6, 2), (64, 128, 256, 512)),
    "convnext_nano": ((2, 2, 8, 2), (80, 160, 320, 640)),
    "convnext_tiny": ((3, 3, 9, 3), (96, 192, 384, 768)),
    "convnext_small": ((3, 3, 27, 3), (96, 192, 384, 768)),
    "convnext_base": ((3, 3, 27, 3), (128, 256, 512, 1024)),
    "convnext_large": ((3, 3, 27, 3), (192, 384, 768, 1536)),
}


class _LayerNorm2d(nn.LayerNorm):
    """Parameter container named like timm.layers.LayerNorm2d (weight, bias over channels)."""


class _Mlp(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.fc1 = nn.Linear(dim, 4 * dim)
        self.fc2 = nn.Linear(4 * dim, dim)


class _Block(nn.Module):
    def __init__(self, dim: int, ls_init_value: float = 1e-6):
        super().__init__()
        self.conv_dw = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _Mlp(dim)
        self.gamma = nn.Parameter(ls_init_value * torch.ones(dim))


class _Stage(nn.Module):
    def __init__(self, in_chs: int, out_chs: int, depth: int, downsample: bool):
        super().__init__()
        if downsample:
            self.downsample = nn.Sequential(_LayerNorm2d(in_chs, eps=1e-6), nn.Conv2d(in_chs, out_chs, kernel_size=2, stride=2))
        else:
            self.downsample = nn.Identity()
        self.blocks = nn.Sequential(*[_Block(out_chs) for _ in range(depth)])


class _Head(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.norm = _LayerNorm2d(dim, eps=1e-6)


class ConvNeXtParams(nn.Module):
    """timm 0.9.16 `ConvNeXt(num_classes=0, global_pool='')` parameter tree (timm/models/convnext.py)."""

    def __init__(self, depths, dims):
        super().__init__()
        self.depths, self.dims = tuple(depths), tuple(dims)
        self.stem = nn.Sequential(nn.Conv2d(3, dims[0], kernel_size=4, stride=4), _LayerNorm2d(dims[0], eps=1e-6))
        stages, prev = [], dims[0]
        for i, (d, c) in enumerate(zip(depths, dims)):
            stages.append(_Stage(prev, c, d, downsample=i > 0))
            prev = c
        self.stages = nn.Sequential(*stages)
        self.head = _Head(prev)
        # timm's init: trunc_normal(std .02) weights, zero biases (convnext.py _init_weights)
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)


class _BlockC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("dw_w", "dw_b", "ln_w", "ln_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "gamma",
                                          "dw_w_flip", "fc2_wg")]


class _BlockTensorsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("dw_w", "dw_b", "ln_w", "ln_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "gamma")]


class _DownTensorsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("ln_w", "ln_b", "conv_w", "conv_b")]


class ConvNeXtTensorsC(C.Structure):
    """vdk_convnext_tensors: fp32 tensors in timm layouts (parameters, or their gradients)."""
    _fields_ = [
        ("stem_w", C.c_void_p), ("stem_b", C.c_void_p), ("stem_ln_w", C.c_void_p), ("stem_ln_b", C.c_void_p),
        ("down", _DownTensorsC * 4), ("blocks", _BlockTensorsC * 64),
        ("head_ln_w", C.c_void_p), ("head_ln_b", C.c_void_p),
        ("bn2_w", C.c_void_p), ("bn2_b", C.c_void_p), ("bn2_running_mean", C.c_void_p), ("bn2_running_var", C.c_void_p),
        ("lin_w", C.c_void_p), ("lin_b", C.c_void_p),
        ("bn1_w", C.c_void_p), ("bn1_b", C.c_void_p), ("bn1_running_mean", C.c_void_p), ("bn1_running_var", C.c_void_p),
    ]


class _DownC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("ln_w", "ln_b", "conv_w", "conv_b")]


class ConvNeXtNetC(C.Structure):
    api = "vdk_convnext"
    _fields_ = [
        ("image_size", C.c_int), ("feat_dim", C.c_int), ("depths", C.c_int * 4), ("dims", C.c_int * 4),
        ("stem_w", C.c_void_p), ("stem_b", C.c_void_p), ("stem_ln_w", C.c_void_p), ("stem_ln_b", C.c_void_p),
        ("down", _DownC * 4), ("blocks", _BlockC * 64),
        ("head_ln_w", C.c_void_p), ("head_ln_b", C.c_void_p), ("neck_w", C.c_void_p), ("neck_b", C.c_void_p),
    ]


class TimmWrapper(BackboneWrapper):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper (ConvNeXt family)."""

    _dropped = ("head.fc",)

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, depths=None, dims=None,
                 **kwargs):
        if depths is None:
            if model_name not in CONVNEXT_ARCHS:
                raise ValueError(f"backbone '{model_name}' is not built for H100 yet; available: {sorted(CONVNEXT_ARCHS)}")
            depths, dims = CONVNEXT_ARCHS[model_name]
        if image_size % 32 != 0:
            raise ValueError("image_size must be a multiple of 32")
        hw = image_size // 32
        super().__init__(model_name, feat_dim, image_size, ConvNeXtParams(depths, dims),
                         cnn_neck(dims[-1], dims[-1] * hw * hw, feat_dim), pretrained)

    def _train_refusal(self) -> str:
        return ""

    # ---- training path (csrc/convnext_train.cu) ------------------------------------------------------
    def _tensors_struct(self, get) -> ConvNeXtTensorsC:
        """vdk_convnext_tensors whose pointers are `get(name)` for every parameter / BN buffer name."""
        t = ConvNeXtTensorsC()
        t.stem_w, t.stem_b = get("model.stem.0.weight"), get("model.stem.0.bias")
        t.stem_ln_w, t.stem_ln_b = get("model.stem.1.weight"), get("model.stem.1.bias")
        bi = 0
        for si, depth in enumerate(self.model.depths):
            if si > 0:
                d = t.down[si]
                d.ln_w, d.ln_b = get(f"model.stages.{si}.downsample.0.weight"), get(f"model.stages.{si}.downsample.0.bias")
                d.conv_w, d.conv_b = get(f"model.stages.{si}.downsample.1.weight"), get(f"model.stages.{si}.downsample.1.bias")
            for j in range(depth):
                pre, b = f"model.stages.{si}.blocks.{j}", t.blocks[bi]
                b.dw_w, b.dw_b = get(f"{pre}.conv_dw.weight"), get(f"{pre}.conv_dw.bias")
                b.ln_w, b.ln_b = get(f"{pre}.norm.weight"), get(f"{pre}.norm.bias")
                b.fc1_w, b.fc1_b = get(f"{pre}.mlp.fc1.weight"), get(f"{pre}.mlp.fc1.bias")
                b.fc2_w, b.fc2_b = get(f"{pre}.mlp.fc2.weight"), get(f"{pre}.mlp.fc2.bias")
                b.gamma = get(f"{pre}.gamma")
                bi += 1
        t.head_ln_w, t.head_ln_b = get("model.head.norm.weight"), get("model.head.norm.bias")
        t.bn2_w, t.bn2_b = get("output_layer.0.weight"), get("output_layer.0.bias")
        t.bn2_running_mean, t.bn2_running_var = get("output_layer.0.running_mean"), get("output_layer.0.running_var")
        t.lin_w, t.lin_b = get("output_layer.2.weight"), get("output_layer.2.bias")
        t.bn1_w, t.bn1_b = get("output_layer.3.weight"), get("output_layer.3.bias")
        t.bn1_running_mean, t.bn1_running_var = get("output_layer.3.running_mean"), get("output_layer.3.running_var")
        return t

    def _train_state(self, device):
        """Packed-weight buffers (allocated once) + the net struct whose fp32 vector fields alias the master params."""
        st = self._train
        if st is not None and st["device"] == device:
            return st
        m = self.model
        bf = lambda *shape: torch.empty(shape, dtype=torch.bfloat16, device=device)
        f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=device)
        hw = self.image_size // 32
        bufs = {"stem_w": bf(m.dims[0], 48), "neck_w": bf(self.feat_dim, hw * hw * m.dims[-1]), "blocks": [], "down": {}}
        for si, (d, c) in enumerate(zip(m.depths, m.dims)):
            if si > 0:
                bufs["down"][si] = bf(c, 4 * m.dims[si - 1])
            for _ in range(d):
                bufs["blocks"].append({"dw_w": f32(49, c), "dw_w_flip": f32(49, c), "fc1_w": bf(4 * c, c), "fc2_w": bf(c, 4 * c),
                                       "fc2_wg": bf(c, 4 * c)})
        self._train = {"device": device, "bufs": bufs, "ws": None, "gflat": None}
        return self._train

    def _train_structs(self, device):
        st = self._train_state(device)
        params = self._master_tensors(device)
        bufs, m = st["bufs"], self.model
        net = ConvNeXtNetC()
        net.image_size, net.feat_dim = self.image_size, self.feat_dim
        for i in range(4):
            net.depths[i], net.dims[i] = m.depths[i], m.dims[i]
        net.stem_w = bufs["stem_w"].data_ptr()
        net.stem_b, net.stem_ln_w, net.stem_ln_b = params.stem_b, params.stem_ln_w, params.stem_ln_b
        bi = 0
        for si, depth in enumerate(m.depths):
            if si > 0:
                net.down[si].ln_w, net.down[si].ln_b = params.down[si].ln_w, params.down[si].ln_b
                net.down[si].conv_w, net.down[si].conv_b = bufs["down"][si].data_ptr(), params.down[si].conv_b
            for _ in range(depth):
                b, pb, bb = net.blocks[bi], params.blocks[bi], bufs["blocks"][bi]
                b.dw_w, b.dw_w_flip = bb["dw_w"].data_ptr(), bb["dw_w_flip"].data_ptr()
                b.fc1_w, b.fc2_w, b.fc2_wg = bb["fc1_w"].data_ptr(), bb["fc2_w"].data_ptr(), bb["fc2_wg"].data_ptr()
                b.dw_b, b.ln_w, b.ln_b, b.fc1_b, b.fc2_b, b.gamma = pb.dw_b, pb.ln_w, pb.ln_b, pb.fc1_b, pb.fc2_b, pb.gamma
                bi += 1
        net.head_ln_w, net.head_ln_b = params.head_ln_w, params.head_ln_b
        net.neck_w, net.neck_b = bufs["neck_w"].data_ptr(), params.lin_b
        return st, net, params

    def _train_forward(self, x: torch.Tensor) -> torch.Tensor:
        lib = _lib.load()
        if x.device.type != "cuda":
            raise RuntimeError("visiondk_b200.TimmWrapper runs on CUDA (sm_90a) only; there is no CPU fallback")
        x = x.contiguous().float()
        B = x.shape[0]
        st, net, params = self._train_structs(x.device)
        need = lib.vdk_convnext_train_workspace_bytes(C.byref(net), B)
        if st["ws"] is None or st["ws"].numel() < need:
            st["ws"] = torch.empty((need,), dtype=torch.uint8, device=x.device)
        out = torch.empty((B, self.feat_dim), dtype=torch.float32, device=x.device)
        bn = self.output_layer[0]
        with torch.cuda.device(x.device):
            s = _lib.stream_ptr()
            # fp32 masters -> kernel layouts (bf16 weights, [49][C] taps and their reversal, gamma-scaled fc2): batched per stage
            _lib.check(lib.vdk_convnext_pack(C.byref(params), C.byref(net), s), "vdk_convnext_pack")
            _lib.check(lib.vdk_convnext_train_forward(C.byref(net), C.byref(params), x.data_ptr(), B, float(bn.momentum),
                                                      out.data_ptr(), st["ws"].data_ptr(), st["ws"].numel(), s),
                       "vdk_convnext_train_forward")
        for m in (self.output_layer[0], self.output_layer[3]):
            m.num_batches_tracked += 1
        st["last"] = (net, params, B)
        return out

    def backward_sections(self):
        """[((unit_begin, unit_end), [parameter names whose gradients are final after that range]), ...] in execution order
        (units: include/vdk_b200.h, vdk_convnext_train_backward_range).  Four ranges: neck + head norm + stage 4; the second
        half of stage 3's blocks; the rest of stage 3; stages 2, 1 and the stem — each a contiguous run of named_parameters()."""
        d = self.model.depths
        names = [n for n, _ in self.named_parameters()]

        def pick(pred):
            return [n for n in names if pred(n)]

        def block_id(n, stage):
            pre = f"model.stages.{stage}.blocks."
            return int(n[len(pre):].split(".")[0]) if n.startswith(pre) else None

        half = d[2] // 2
        u_a = 1 + d[3] + 1                  # neck, stage-4 blocks, stage-4 downsample
        u_b = u_a + (d[2] - half)           # blocks d[2]-1 .. half of stage 3
        u_c = u_a + d[2] + 1                # remaining blocks + stage-3 downsample
        u_end = 1 + sum(d) + 4
        sec = [
            ((0, u_a), pick(lambda n: n.startswith("output_layer.") or n.startswith("model.head.") or n.startswith("model.stages.3."))),
            ((u_a, u_b), pick(lambda n: (block_id(n, 2) is not None and block_id(n, 2) >= half))),
            ((u_b, u_c), pick(lambda n: n.startswith("model.stages.2.") and not (block_id(n, 2) is not None and block_id(n, 2) >= half))),
            ((u_c, u_end), pick(lambda n: n.startswith("model.stem.") or n.startswith("model.stages.0.") or n.startswith("model.stages.1."))),
        ]
        covered = sum(len(ns) for _, ns in sec)
        if covered != len(names):
            raise RuntimeError(f"backward_sections: {len(names) - covered} parameters not assigned to a section")
        return [x for x in sec if x[0][0] < x[0][1]]

    # ---- weight packing --------------------------------------------------------------------------
    def _build(self, p) -> ConvNeXtNetC:
        """Kernel-side layouts (include/vdk_b200.h): bf16 GEMM weights, fp32 vectors, depthwise taps [49][C],
        downsample conv K order (kh,kw,cin), neck with BN2d/BN1d eval statistics folded and K order (h,w,c)."""
        m, net = self.model, ConvNeXtNetC()
        net.image_size, net.feat_dim = self.image_size, self.feat_dim
        for i in range(4):
            net.depths[i], net.dims[i] = m.depths[i], m.dims[i]
        net.stem_w = p.bf16(m.stem[0].weight.reshape(m.dims[0], 48))
        net.stem_b, net.stem_ln_w, net.stem_ln_b = p.f32(m.stem[0].bias), p.f32(m.stem[1].weight), p.f32(m.stem[1].bias)
        bi = 0
        for si, stage in enumerate(m.stages):
            if si > 0:
                ln, conv = stage.downsample[0], stage.downsample[1]
                net.down[si].ln_w, net.down[si].ln_b = p.f32(ln.weight), p.f32(ln.bias)
                net.down[si].conv_w = p.bf16(conv.weight.permute(0, 2, 3, 1).reshape(conv.weight.shape[0], -1))
                net.down[si].conv_b = p.f32(conv.bias)
            for blk in stage.blocks:
                b = net.blocks[bi]
                c = blk.conv_dw.weight.shape[0]
                b.dw_w = p.f32(blk.conv_dw.weight.reshape(c, 49).t())
                b.dw_b, b.ln_w, b.ln_b = p.f32(blk.conv_dw.bias), p.f32(blk.norm.weight), p.f32(blk.norm.bias)
                b.fc1_w, b.fc1_b = p.bf16(blk.mlp.fc1.weight), p.f32(blk.mlp.fc1.bias)
                b.fc2_w, b.fc2_b = p.bf16(blk.mlp.fc2.weight), p.f32(blk.mlp.fc2.bias)
                b.gamma = p.f32(blk.gamma)
                bi += 1
        net.head_ln_w, net.head_ln_b = p.f32(m.head.norm.weight), p.f32(m.head.norm.bias)
        net.neck_w, net.neck_b = self._pack_cnn_neck(p)
        return net


class BackboneFactory:
    """models/faceX/backbone/backbone_def.py:5-26: `{'timm-<name>': {pretrained, image_size, feat_dim}}`."""

    def __init__(self, backbone_config: dict):
        for k, v in backbone_config.items():
            self.backbone_type, self.backbone_param = k, v

    def get_backbone(self) -> nn.Module:
        if not self.backbone_type.startswith("timm-"):
            raise ValueError(f"Unsupported backbone type: {self.backbone_type}. Only timm models are supported.")
        model_name = self.backbone_type[5:].split(".")[0]  # timm's "<architecture>.<pretrained tag>": the tag names weights only
        if model_name.startswith("vit_"):  # Transformer backbones: eval / extract path (visiondk_b200/vit.py)
            from .vit import ViTWrapper
            return ViTWrapper(model_name=model_name, **self.backbone_param)
        from .resnet import RESNET_ARCHS, RESNEXT_ARCHS, ResNetWrapper
        if model_name in RESNET_ARCHS or model_name in RESNEXT_ARCHS:  # Bottleneck ResNets / ResNeXts: eval / extract path
            return ResNetWrapper(model_name=model_name, **self.backbone_param)  # (visiondk_b200/resnet.py)
        from .senet import SENET_ARCHS, SENetWrapper
        if model_name in SENET_ARCHS:  # legacy SE-ResNets / SE-ResNeXts: eval / extract path (visiondk_b200/senet.py)
            return SENetWrapper(model_name=model_name, **self.backbone_param)
        from .resnest import RESNEST_ARCHS, ResNeStWrapper
        if model_name in RESNEST_ARCHS:  # ResNeSts: eval / extract path (visiondk_b200/resnest.py)
            return ResNeStWrapper(model_name=model_name, **self.backbone_param)
        if model_name.startswith("swinv2_"):  # Swin V2 towers: eval / extract path (visiondk_b200/swin.py); other variants refused
            from .swin import SwinV2Wrapper
            return SwinV2Wrapper(model_name=model_name, **self.backbone_param)
        if model_name.startswith("tf_efficientnetv2_"):  # EfficientNetV2: eval / extract path (visiondk_b200/efficientnet.py)
            from .efficientnet import EfficientNetV2Wrapper
            return EfficientNetV2Wrapper(model_name=model_name, **self.backbone_param)
        if model_name.startswith(("mobilenetv3_", "tf_mobilenetv3_")):  # MobileNetV3: eval / extract path
            from .mobilenetv3 import MobileNetV3Wrapper  # (visiondk_b200/mobilenetv3.py); other widths / variants refused
            return MobileNetV3Wrapper(model_name=model_name, **self.backbone_param)
        return TimmWrapper(model_name=model_name, **self.backbone_param)
