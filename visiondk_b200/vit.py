"""ViT backbones for the CBIR extract path (inference) on the H100 kernels.

Mirrors what `TimmWrapper(model_name='vit_*', feat_dim, image_size)` builds in the reference
(models/faceX/backbone/timm_wrapper.py:16-21 + the Transformer neck of :39-47): the parameter tree and state_dict keys of
timm 0.9.16's VisionTransformer (`model.patch_embed.proj`, `model.cls_token`, `model.pos_embed`, `model.blocks.{i}.{norm1,
attn.qkv, attn.proj, norm2, mlp.fc1, mlp.fc2}`, `model.norm`) and `output_layer.{0: LayerNorm, 2: Linear, 3: BatchNorm1d}`,
so reference checkpoints load with `strict=True`.  The eval forward runs in `vdk_vit_forward`, the train-mode forward and
backward (BASELINE config 3) in `vdk_vit_train_forward` / `vdk_vit_train_backward` (csrc/vit.cu) as ONE autograd node;
training needs 3*patch^2 % 8 == 0 and at most 208 tokens (ViT-*/16 at 224^2).

The CBIR configs' self-supervised and contrastive towers (DINO ViT-B/8, DINOv2 ViT-L/14, SigLIP So400m/14, CLIP ViT-H/14) add
head dims 72 and 80, a model without a class token (`model.cls_token` absent, pos_embed [N, dim]), LayerScale
(`model.blocks.{i}.ls1.gamma`, `ls2.gamma`) and an MLP width other than 4 * dim.  Those are built for extraction only.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .wrapper import BackboneWrapper, fold_bn1d

VIT_ARCHS = {
    # timm name -> (patch, embed_dim, depth, heads)
    "vit_tiny_patch16_224": (16, 192, 12, 3),
    "vit_small_patch16_224": (16, 384, 12, 6),
    "vit_base_patch16_224": (16, 768, 12, 12),
    "vit_large_patch16_224": (16, 1024, 24, 16),
    "vit_base_patch16_clip_224": (16, 768, 12, 12),
    "vit_large_patch14_clip_224": (14, 1024, 24, 16),
    "vit_large_patch14_clip_336": (14, 1024, 24, 16),
    "vit_base_patch8_224": (8, 768, 12, 12),                # DINO ViT-B/8 (.dino)
    "vit_large_patch14_dinov2": (14, 1024, 24, 16),        # DINOv2 ViT-L/14 (.lvd142m), 518^2
    "vit_so400m_patch14_siglip_224": (14, 1152, 27, 16),   # SigLIP So400m/14 (.webli): head dim 72
    "vit_huge_patch14_clip_224": (14, 1280, 32, 16),       # CLIP ViT-H/14 (.laion2b_ft_in12k_in1k): head dim 80
}
# timm 0.9.16 `vit_*_clip_*` (the CLIP image towers; BASELINE config 5's ViT-L/14 at 336^2): VisionTransformer(pre_norm=True,
# norm_layer=nn.LayerNorm): a `norm_pre` LayerNorm after cls / position, NO bias in patch_embed.proj, LayerNorm eps 1e-5,
# standard GELU (the `*_clip_quickgelu_*` architectures are separate timm entries and are not built).
VIT_PRE_NORM = {"vit_base_patch16_clip_224", "vit_large_patch14_clip_224", "vit_large_patch14_clip_336", "vit_huge_patch14_clip_224"}
# timm 0.9.16 side attributes of the entries above (absent: 4 * dim MLP, a class token, no LayerScale):
VIT_MLP_DIM = {"vit_so400m_patch14_siglip_224": 4304}          # mlp_ratio 3.7362 -> int(1152 * 3.7362)
VIT_NO_CLASS_TOKEN = {"vit_so400m_patch14_siglip_224"}         # class_token=False: no cls_token parameter at all
VIT_LAYER_SCALE = {"vit_large_patch14_dinov2"}                 # init_values=1e-5: blocks.{i}.ls1.gamma, ls2.gamma
VIT_IMAGE_SIZE = {"vit_large_patch14_dinov2": 518, "vit_large_patch14_clip_336": 336}  # pretrained resolution (else 224)
VIT_HEAD_DIMS = (64, 72, 80)
MAX_BLOCKS = 48


class _Attention(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim, bias=True)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _LayerScale(nn.Module):
    def __init__(self, dim, init_values=1e-5):
        super().__init__()
        self.gamma = nn.Parameter(init_values * torch.ones(dim))


class _Block(nn.Module):
    def __init__(self, dim, eps=1e-6, mlp_dim=None, layer_scale=False):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = _Attention(dim)
        if layer_scale:
            self.ls1 = _LayerScale(dim)
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = _Mlp(dim, mlp_dim or 4 * dim)
        if layer_scale:
            self.ls2 = _LayerScale(dim)


class _PatchEmbed(nn.Module):
    def __init__(self, patch, dim, bias=True):
        super().__init__()
        self.proj = nn.Conv2d(3, dim, kernel_size=patch, stride=patch, bias=bias)


class ViTParams(nn.Module):
    """timm 0.9.16 `VisionTransformer(num_classes=0, global_pool='')` parameter tree (timm/models/vision_transformer.py)."""

    def __init__(self, image_size, patch, dim, depth, heads, pre_norm=False, mlp_dim=None, class_token=True, layer_scale=False):
        super().__init__()
        self.image_size, self.patch, self.dim, self.depth, self.heads = image_size, patch, dim, depth, heads
        self.pre_norm = bool(pre_norm)
        self.mlp_dim = int(mlp_dim or 4 * dim)
        self.class_token, self.layer_scale = bool(class_token), bool(layer_scale)
        self.ln_eps = 1e-5 if pre_norm else 1e-6
        n = (image_size // patch) ** 2
        self.tokens = n + (1 if class_token else 0)
        self.patch_embed = _PatchEmbed(patch, dim, bias=not pre_norm)
        if class_token:
            self.cls_token = nn.Parameter(torch.zeros(1, 1, dim))
        self.pos_embed = nn.Parameter(torch.randn(1, self.tokens, dim) * 0.02)
        if pre_norm:
            self.norm_pre = nn.LayerNorm(dim, eps=self.ln_eps)
        self.blocks = nn.Sequential(*[_Block(dim, self.ln_eps, self.mlp_dim, layer_scale) for _ in range(depth)])
        self.norm = nn.LayerNorm(dim, eps=self.ln_eps)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)
        if class_token:
            nn.init.normal_(self.cls_token, std=1e-6)

    def inference_only_features(self):
        """Names of what this model has that the training kernels do not implement (empty: trainable)."""
        f = []
        if self.pre_norm:
            f.append("pre_norm (CLIP towers)")
        if self.dim != 64 * self.heads:
            f.append(f"head dim {self.dim // self.heads}")
        if not self.class_token:
            f.append("no class token")
        if self.layer_scale:
            f.append("LayerScale")
        if self.mlp_dim != 4 * self.dim:
            f.append(f"MLP width {self.mlp_dim}")
        if self.tokens > 208:  # the attention backward keeps one head's probability matrix in shared memory
            f.append(f"{self.tokens} tokens (training takes at most 208)")
        return f


class _VitBlockC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("ln1_w", "ln1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "ln2_w", "ln2_b", "fc1_w", "fc1_b",
                                          "fc2_w", "fc2_b", "ls1", "ls2")]


class _VitBlockTensorsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("ln1_w", "ln1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "ln2_w", "ln2_b", "fc1_w", "fc1_b",
                                          "fc2_w", "fc2_b")]


class VitTensorsC(C.Structure):
    """vdk_vit_tensors: fp32 tensors in timm layouts (parameters, or their gradients)."""
    _fields_ = [("patch_w", C.c_void_p), ("patch_b", C.c_void_p), ("cls_token", C.c_void_p), ("pos_embed", C.c_void_p),
                ("blocks", _VitBlockTensorsC * MAX_BLOCKS),
                ("norm_w", C.c_void_p), ("norm_b", C.c_void_p), ("neck_ln_w", C.c_void_p), ("neck_ln_b", C.c_void_p),
                ("lin_w", C.c_void_p), ("lin_b", C.c_void_p),
                ("bn1_w", C.c_void_p), ("bn1_b", C.c_void_p), ("bn1_running_mean", C.c_void_p), ("bn1_running_var", C.c_void_p)]


class VitNetC(C.Structure):
    """vdk_vit_net (include/vdk_b200.h)."""
    api = "vdk_vit"
    _fields_ = [("image_size", C.c_int), ("patch", C.c_int), ("dim", C.c_int), ("depth", C.c_int), ("heads", C.c_int),
                ("feat_dim", C.c_int),
                ("patch_w", C.c_void_p), ("patch_b", C.c_void_p), ("cls_token", C.c_void_p), ("pos_embed", C.c_void_p),
                ("ones", C.c_void_p), ("blocks", _VitBlockC * MAX_BLOCKS),
                ("norm_w", C.c_void_p), ("norm_b", C.c_void_p), ("neck_ln_w", C.c_void_p), ("neck_ln_b", C.c_void_p),
                ("neck_w", C.c_void_p), ("neck_b", C.c_void_p),
                ("norm_pre_w", C.c_void_p), ("norm_pre_b", C.c_void_p), ("ln_eps", C.c_float), ("mlp_dim", C.c_int)]


class ViTWrapper(BackboneWrapper):
    """Drop-in for the reference's TimmWrapper when the timm model is a VisionTransformer (eval / extract path)."""

    def __init__(self, model_name: str, feat_dim: int, image_size: int, pretrained: bool = True, patch=None, dim=None, depth=None,
                 heads=None, pre_norm=None, mlp_dim=None, class_token=None, layer_scale=None, **kwargs):
        if dim is None:
            if model_name not in VIT_ARCHS:
                raise ValueError(f"backbone '{model_name}' is not built for H100 yet; available: {sorted(VIT_ARCHS)}")
            patch, dim, depth, heads = VIT_ARCHS[model_name]
        if pre_norm is None:
            pre_norm = model_name in VIT_PRE_NORM
        if mlp_dim is None:
            mlp_dim = VIT_MLP_DIM.get(model_name, 4 * dim)
        if class_token is None:
            class_token = model_name not in VIT_NO_CLASS_TOKEN
        if layer_scale is None:
            layer_scale = model_name in VIT_LAYER_SCALE
        if (image_size % patch != 0 or dim % heads != 0 or dim // heads not in VIT_HEAD_DIMS or depth > MAX_BLOCKS or
                mlp_dim % 8 != 0):
            raise ValueError("ViT on H100: image_size must be a multiple of patch, head_dim 64, 72 or 80, depth <= 48, mlp_dim a "
                             "multiple of 8")
        if pretrained:
            raise RuntimeError("pretrained timm weights cannot be downloaded here (no network): pass pretrained=False and "
                               "load a checkpoint with load_state_dict (keys are timm's)")
        model = ViTParams(image_size, patch, dim, depth, heads, pre_norm=pre_norm, mlp_dim=mlp_dim, class_token=class_token,
                          layer_scale=layer_scale)
        output_layer = nn.Sequential(nn.LayerNorm(dim), nn.Flatten(1), nn.Linear(model.tokens * dim, feat_dim),
                                     nn.BatchNorm1d(feat_dim))
        super().__init__(model_name, feat_dim, image_size, model, output_layer, pretrained=False)

    def _train_refusal(self) -> str:
        features = self.model.inference_only_features()
        return f"{', '.join(features)}: built for inference / extraction only" if features else ""

    # ---- training path (csrc/vit.cu: vdk_vit_train_forward / vdk_vit_train_backward) -------------------------------------
    def _tensors_struct(self, get) -> VitTensorsC:
        t = VitTensorsC()
        t.patch_w, t.patch_b = get("model.patch_embed.proj.weight"), get("model.patch_embed.proj.bias")
        t.cls_token, t.pos_embed = get("model.cls_token"), get("model.pos_embed")
        for i in range(self.model.depth):
            b, pre = t.blocks[i], f"model.blocks.{i}."
            b.ln1_w, b.ln1_b = get(pre + "norm1.weight"), get(pre + "norm1.bias")
            b.qkv_w, b.qkv_b = get(pre + "attn.qkv.weight"), get(pre + "attn.qkv.bias")
            b.proj_w, b.proj_b = get(pre + "attn.proj.weight"), get(pre + "attn.proj.bias")
            b.ln2_w, b.ln2_b = get(pre + "norm2.weight"), get(pre + "norm2.bias")
            b.fc1_w, b.fc1_b = get(pre + "mlp.fc1.weight"), get(pre + "mlp.fc1.bias")
            b.fc2_w, b.fc2_b = get(pre + "mlp.fc2.weight"), get(pre + "mlp.fc2.bias")
        t.norm_w, t.norm_b = get("model.norm.weight"), get("model.norm.bias")
        t.neck_ln_w, t.neck_ln_b = get("output_layer.0.weight"), get("output_layer.0.bias")
        t.lin_w, t.lin_b = get("output_layer.2.weight"), get("output_layer.2.bias")
        t.bn1_w, t.bn1_b = get("output_layer.3.weight"), get("output_layer.3.bias")
        t.bn1_running_mean, t.bn1_running_var = get("output_layer.3.running_mean"), get("output_layer.3.running_var")
        return t

    def backward_sections(self):
        """[((unit_begin, unit_end), [parameter names final after that range]), ...]: neck + final norm + the last third of the
        blocks; the middle third; the first third + patch / cls / position embeddings — each a contiguous run of named_parameters()."""
        d = self.model.depth
        names = [n for n, _ in self.named_parameters()]

        def blk(n):
            return int(n.split(".")[2]) if n.startswith("model.blocks.") else None

        c1, c2 = d - d // 3, d - 2 * (d // 3)  # blocks >= c1 | c2 <= blocks < c1 | blocks < c2
        sec = [
            ((0, 1 + (d - c1)), [n for n in names if n.startswith("output_layer.") or n.startswith("model.norm.") or
                                 (blk(n) is not None and blk(n) >= c1)]),
            ((1 + (d - c1), 1 + (d - c2)), [n for n in names if blk(n) is not None and c2 <= blk(n) < c1]),
            ((1 + (d - c2), d + 2), [n for n in names if (blk(n) is not None and blk(n) < c2) or n in ("model.cls_token", "model.pos_embed")
                                     or n.startswith("model.patch_embed.")]),
        ]
        if sum(len(ns) for _, ns in sec) != len(names):
            raise RuntimeError("backward_sections: parameters not covered exactly once")
        return [x for x in sec if x[0][0] < x[0][1] and x[1]]

    def _train_structs(self, device):
        m = self.model
        if self._train is None or self._train["device"] != device:
            def buf(*shape):
                return torch.empty(shape, dtype=torch.bfloat16, device=device)
            tokens = (m.image_size // m.patch) ** 2 + 1
            self._train = {"device": device, "ws": None, "gflat": None, "last": None,
                           "patch_w": buf(m.dim, 3 * m.patch * m.patch),
                           "blocks": [{"qkv_w": buf(3 * m.dim, m.dim), "proj_w": buf(m.dim, m.dim), "fc1_w": buf(4 * m.dim, m.dim),
                                       "fc2_w": buf(m.dim, 4 * m.dim)} for _ in range(m.depth)],
                           "neck_w": buf(self.feat_dim, tokens * m.dim),
                           "ones": torch.ones(m.dim, dtype=torch.float32, device=device)}
        st = self._train
        params = self._master_tensors(device)
        net = VitNetC()
        net.image_size, net.patch, net.dim, net.depth, net.heads, net.feat_dim = (m.image_size, m.patch, m.dim, m.depth, m.heads,
                                                                                 self.feat_dim)
        net.patch_w, net.patch_b = st["patch_w"].data_ptr(), params.patch_b
        net.cls_token, net.pos_embed, net.ones = params.cls_token, params.pos_embed, st["ones"].data_ptr()
        for i in range(m.depth):
            b, pb, bb = net.blocks[i], params.blocks[i], st["blocks"][i]
            b.ln1_w, b.ln1_b, b.qkv_b, b.proj_b = pb.ln1_w, pb.ln1_b, pb.qkv_b, pb.proj_b
            b.ln2_w, b.ln2_b, b.fc1_b, b.fc2_b = pb.ln2_w, pb.ln2_b, pb.fc1_b, pb.fc2_b
            b.qkv_w, b.proj_w = bb["qkv_w"].data_ptr(), bb["proj_w"].data_ptr()
            b.fc1_w, b.fc2_w = bb["fc1_w"].data_ptr(), bb["fc2_w"].data_ptr()
        net.norm_w, net.norm_b, net.neck_ln_w, net.neck_ln_b = params.norm_w, params.norm_b, params.neck_ln_w, params.neck_ln_b
        net.neck_w, net.neck_b = st["neck_w"].data_ptr(), params.lin_b
        return st, net, params

    def _train_forward(self, x: torch.Tensor) -> torch.Tensor:
        lib = _lib.load()
        if x.device.type != "cuda":
            raise RuntimeError("visiondk_b200.ViTWrapper runs on CUDA (sm_90a) only; there is no CPU fallback")
        x = x.contiguous().float()
        B = x.shape[0]
        st, net, params = self._train_structs(x.device)
        need = lib.vdk_vit_train_workspace_bytes(C.byref(net), B)
        if need == 0:
            raise RuntimeError("vdk_vit_train_workspace_bytes: " + _lib.last_error())
        if st["ws"] is None or st["ws"].numel() < need:
            st["ws"] = torch.empty((need,), dtype=torch.uint8, device=x.device)
        out = torch.empty((B, self.feat_dim), dtype=torch.float32, device=x.device)
        bn = self.output_layer[3]
        with torch.cuda.device(x.device):
            s = _lib.stream_ptr()
            _lib.check(lib.vdk_vit_pack(C.byref(params), C.byref(net), s), "vdk_vit_pack")
            _lib.check(lib.vdk_vit_train_forward(C.byref(net), C.byref(params), x.data_ptr(), B, float(bn.momentum), out.data_ptr(),
                                                 st["ws"].data_ptr(), st["ws"].numel(), s), "vdk_vit_train_forward")
        bn.num_batches_tracked += 1
        st["last"] = (net, params, B)
        return out

    def _build(self, p) -> VitNetC:
        m, net = self.model, VitNetC()
        net.image_size, net.patch, net.dim, net.depth, net.heads, net.feat_dim = (m.image_size, m.patch, m.dim, m.depth, m.heads,
                                                                                 self.feat_dim)
        k = 3 * m.patch * m.patch
        kp = (k + 7) // 8 * 8
        w = m.patch_embed.proj.weight.detach().reshape(m.dim, k)  # (c, kh, kw) order
        if kp != k:
            w = torch.cat([w, torch.zeros(m.dim, kp - k, dtype=w.dtype, device=w.device)], dim=1)
        net.patch_w = p.bf16(w)
        net.patch_b = p.f32(m.patch_embed.proj.bias) if m.patch_embed.proj.bias is not None else 0
        if m.pre_norm:
            net.norm_pre_w, net.norm_pre_b = p.f32(m.norm_pre.weight), p.f32(m.norm_pre.bias)
        net.ln_eps = float(m.ln_eps)
        net.mlp_dim = m.mlp_dim
        net.cls_token = p.f32(m.cls_token.reshape(-1)) if m.class_token else 0
        net.pos_embed = p.f32(m.pos_embed.reshape(-1, m.dim))
        net.ones = p.f32(torch.ones(m.dim))
        for i, blk in enumerate(m.blocks):
            b = net.blocks[i]
            b.ln1_w, b.ln1_b = p.f32(blk.norm1.weight), p.f32(blk.norm1.bias)
            b.qkv_w, b.qkv_b = p.bf16(blk.attn.qkv.weight), p.f32(blk.attn.qkv.bias)
            b.proj_w, b.proj_b = p.bf16(blk.attn.proj.weight), p.f32(blk.attn.proj.bias)
            b.ln2_w, b.ln2_b = p.f32(blk.norm2.weight), p.f32(blk.norm2.bias)
            b.fc1_w, b.fc1_b = p.bf16(blk.mlp.fc1.weight), p.f32(blk.mlp.fc1.bias)
            b.fc2_w, b.fc2_b = p.bf16(blk.mlp.fc2.weight), p.f32(blk.mlp.fc2.bias)
            if m.layer_scale:
                b.ls1, b.ls2 = p.f32(blk.ls1.gamma), p.f32(blk.ls2.gamma)
        net.norm_w, net.norm_b = p.f32(m.norm.weight), p.f32(m.norm.bias)
        ln, lin = self.output_layer[0], self.output_layer[2]
        net.neck_ln_w, net.neck_ln_b = p.f32(ln.weight), p.f32(ln.bias)
        w, bias = fold_bn1d(lin.weight.detach().double(), lin.bias.detach().double(), self.output_layer[3])
        net.neck_w, net.neck_b = p.bf16(w), p.f32(bias)
        return net
