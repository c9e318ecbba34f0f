"""What every extraction backbone wrapper shares (ConvNeXt, ViT, ResNet / ResNeXt, SENet, ResNeSt, EfficientNetV2, MobileNetV3,
Swin V2).

`BackboneWrapper` keeps the reference TimmWrapper's surface (`model.` / `output_layer.` parameters, `forward(x) -> [B,
feat_dim]`) and owns the host side around the family's kernels: the weight-pack cache, `embed`, the checkpoint load and, for
the families that train, the one autograd node.  A family supplies its parameter tree, its `*NetC` struct (with `api`, the
prefix of its C entry points) and `_build(packer)`, which fills that struct from the parameters.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings

import torch
import torch.nn as nn

from . import _lib


class Packer:
    """Converts tensors to their kernel-side dtype on one device, keeps the results alive, and returns their pointers."""

    def __init__(self, device):
        self.device, self.keep = device, []

    def f32(self, t: torch.Tensor) -> int:
        t = t.detach().to(self.device, torch.float32).contiguous()
        self.keep.append(t)
        return t.data_ptr()

    def bf16(self, t: torch.Tensor) -> int:
        t = t.detach().to(self.device, torch.float32).contiguous().to(torch.bfloat16)
        self.keep.append(t)
        return t.data_ptr()

    def stem_rows(self, w: torch.Tensor, b: torch.Tensor, multiple: int):
        """A stem conv [Cout, Cin, kh, kw] as bf16 (kh, kw, c) patch rows zero-padded to a multiple of `multiple`, and its
        fp32 bias: (weight pointer, bias pointer)."""
        k = w[0].numel()
        rows = w.permute(0, 2, 3, 1).reshape(w.shape[0], k)
        kp = -(-k // multiple) * multiple
        return self.bf16(torch.cat([rows, rows.new_zeros(w.shape[0], kp - k)], dim=1)), self.f32(b)


def fold_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d):
    """Eval BatchNorm folded into the bias-free conv before it, in fp32: w * g / sqrt(var + eps), b - mean * g / sqrt(var + eps)."""
    s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    w = conv.weight.detach().float() * s.view(-1, 1, 1, 1)
    return w, bn.bias.detach().float() - bn.running_mean.detach().float() * s


@torch.no_grad()
def fold_bn1d(w: torch.Tensor, b: torch.Tensor, bn: nn.BatchNorm1d):
    """Eval BatchNorm1d folded into the fp64 Linear (w [out, ...], b) before it, on w's device: y = s (W x + b - mean) + beta
    with s = gamma / sqrt(var + eps)."""
    s = (bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)).to(w.device)
    return w * s.view(-1, *(1,) * (w.dim() - 1)), s * (b - bn.running_mean.double().to(w.device)) + bn.bias.double().to(w.device)


@torch.no_grad()
def fold_neck(output_layer: nn.Sequential, device):
    """The neck BatchNorm2d(n) -> Flatten -> Linear -> BatchNorm1d (eval statistics) as one Linear over the flattened
    features, in fp64 on `device`: (weight [feat_dim, n, in_features / n], bias [feat_dim])."""
    bn2, lin = output_layer[0], output_layer[2]
    s2 = (bn2.weight.double() / torch.sqrt(bn2.running_var.double() + bn2.eps)).to(device)
    t2 = bn2.bias.double().to(device) - bn2.running_mean.double().to(device) * s2
    w = lin.weight.detach().double().to(device).reshape(lin.out_features, bn2.num_features, -1)
    bias = lin.bias.detach().double().to(device) + (w * t2.view(1, -1, 1)).sum(dim=(1, 2))
    return fold_bn1d(w * s2.view(1, -1, 1), bias, output_layer[3])


def cnn_neck(channels: int, in_features: int, feat_dim: int) -> nn.Sequential:
    """The reference wrapper's neck for a 4-D backbone output: BatchNorm2d(shape[1]) -> Flatten -> Linear -> BatchNorm1d."""
    return nn.Sequential(nn.BatchNorm2d(channels), nn.Flatten(1), nn.Linear(in_features, feat_dim), nn.BatchNorm1d(feat_dim))


class BackboneWrapper(nn.Module):
    """Drop-in for models/faceX/backbone/timm_wrapper.py::TimmWrapper, running on the sm_90a kernels of one family."""

    _dropped = ()  # checkpoint key prefixes not loaded: timm's classifier (num_classes=0)
    _rebuilt = ()  # checkpoint key suffixes not loaded: buffers the family rebuilds

    def __init__(self, model_name: str, feat_dim: int, image_size: int, model: nn.Module, output_layer: nn.Sequential,
                 pretrained: bool):
        super().__init__()
        self.model_name, self.feat_dim, self.image_size = model_name, int(feat_dim), int(image_size)
        self.model, self.output_layer = model, output_layer
        self._packed = None  # {"key", "net", "keep"}: the packed struct and the tensors its pointers point into
        self._ws = None
        self._train = None
        if pretrained:
            self._load_pretrained()

    # ---- reference surface -----------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self.training:
            return self.embed(x, l2_normalize=False)
        refusal = self._train_refusal()
        if refusal:
            raise NotImplementedError(f"{self.model_name}: {refusal} (call .eval() first)")
        return _TrainFn.apply(self, x, *self.parameters())

    def _train_refusal(self) -> str:
        """Why a train-mode forward is refused; empty for a family with a train path."""
        return f"{type(self).__name__} is extraction-only on H100"

    @torch.no_grad()
    def embed(self, x: torch.Tensor, l2_normalize: bool = False) -> torch.Tensor:
        """[B,3,S,S] fp32 NCHW (normalised like the reference's transforms) -> fp32 [B, feat_dim] (TimmWrapper.forward in eval
        mode; optionally F.normalize fused)."""
        if x.device.type != "cuda":
            raise RuntimeError(f"visiondk_b200.{type(self).__name__} runs on CUDA (sm_90a) only; there is no CPU fallback")
        lib = _lib.load()
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != self.image_size or x.shape[3] != self.image_size:
            raise ValueError(f"expected [B,3,{self.image_size},{self.image_size}], got {tuple(x.shape)}")
        x = x.contiguous().float()
        net = self._pack(x.device)
        B = x.shape[0]
        out = torch.empty((B, self.feat_dim), dtype=torch.float32, device=x.device)
        api = net.api
        need = getattr(lib, f"{api}_workspace_bytes")(C.byref(net), B)
        if need == 0:
            raise RuntimeError(f"{api}_workspace_bytes: {_lib.last_error()}")
        if self._ws is None or self._ws.numel() < need or self._ws.device != x.device:
            self._ws = torch.empty((need,), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(getattr(lib, f"{api}_forward")(C.byref(net), x.data_ptr(), B, int(l2_normalize), out.data_ptr(),
                                                      self._ws.data_ptr(), self._ws.numel(), _lib.stream_ptr()), f"{api}_forward")
        return out

    # ---- weight packing --------------------------------------------------------------------------
    def _pack(self, device):
        """The family's `*NetC` over kernel-side copies of the weights, rebuilt by `_build` when the device or the `_version`
        of any parameter or buffer has changed since the last build."""
        key = (str(device),) + tuple(int(t._version) for t in list(self.parameters()) + list(self.buffers()))
        if self._packed is None or self._packed["key"] != key:
            packer = Packer(device)
            with torch.no_grad():
                net = self._build(packer)
            self._packed = {"key": key, "net": net, "keep": packer.keep}
        return self._packed["net"]

    def invalidate_pack(self) -> None:
        """Drop the packed weights: writes through raw pointers (the fused optimizer's) do not bump `_version`."""
        self._packed = None

    def _pack_cnn_neck(self, p: Packer):
        """The folded CNN neck over the final NHWC map: bf16 weight with K in (h, w, c) order, fp32 bias."""
        w, bias = fold_neck(self.output_layer, p.device)
        return p.bf16(w.transpose(1, 2).reshape(self.feat_dim, -1)), p.f32(bias)

    def _load_pretrained(self) -> None:
        """The reference downloads timm weights (timm_wrapper.py:16-21); this package reads a timm state_dict from
        $VDK_PRETRAINED_DIR/<model_name>.pth when present, without the keys num_classes=0 or the family's rebuilt buffers drop."""
        root = os.environ.get("VDK_PRETRAINED_DIR")
        path = os.path.join(root, f"{self.model_name}.pth") if root else None
        if path and os.path.exists(path):
            sd = torch.load(path, map_location="cpu")
            sd = {k: v for k, v in sd.items() if not k.startswith(self._dropped) and not k.endswith(self._rebuilt)}
            self.model.load_state_dict(sd, strict=True)
        else:
            warnings.warn(f"pretrained weights for '{self.model_name}' not found (set VDK_PRETRAINED_DIR); using random init")

    # ---- training (families with `_tensors_struct`, `_train_forward` and `backward_sections`) ---------
    def _master_tensors(self, device):
        """The family's `*TensorsC` over the fp32 master parameters and BatchNorm buffers, which the train kernels read and
        update in place."""
        named = dict(self.named_parameters())
        named.update(dict(self.named_buffers()))
        for n, t in named.items():
            if t.is_floating_point() and (t.device != device or t.dtype != torch.float32 or not t.is_contiguous()):
                raise RuntimeError(f"{n}: training needs contiguous fp32 parameters on {device}")
        return self._tensors_struct(lambda n: named[n].data_ptr())

    def _train_backward(self, dout: torch.Tensor):
        """Gradients of every parameter.  When the parameters already own fp32 `.grad` buffers (the fused optimizer
        re-points them into its flat gradient buffer) the kernels accumulate straight into those and autograd receives
        None; otherwise the gradients are produced in a scratch buffer and returned."""
        lib = _lib.load()
        st = self._train
        net, params, B = st["last"]
        plist = list(self.named_parameters())
        direct = all(p.grad is not None and p.grad.dtype == torch.float32 and p.grad.is_contiguous() and
                     p.grad.device == dout.device for _, p in plist)
        if direct:
            ptrs = {n: p.grad.data_ptr() for n, p in plist}
        else:
            total = sum(p.numel() for _, p in plist)
            if st["gflat"] is None or st["gflat"].numel() != total:
                st["gflat"] = torch.empty((total,), dtype=torch.float32, device=dout.device)
            gflat = st["gflat"]
            gflat.zero_()
            offs, off = {}, 0
            for n, p in plist:
                offs[n] = off
                off += p.numel()
            ptrs = {n: gflat.data_ptr() + 4 * offs[n] for n, _ in plist}
        grads = self._tensors_struct(lambda n: ptrs.get(n, 0))
        dout = dout.contiguous().float()
        hook = getattr(self, "grad_section_hook", None)
        api = net.api
        with torch.cuda.device(dout.device):
            args = (C.byref(net), C.byref(params), C.byref(grads), dout.data_ptr(), B, st["ws"].data_ptr(), st["ws"].numel(),
                    _lib.stream_ptr())
            if hook is not None and direct:
                # DDP overlap: the backward runs in a few unit ranges; after each one the parameters whose gradients are now
                # final are handed to the hook (FaceTrainer starts their all-reduce while the next range computes)
                for (u0, u1), names in self.backward_sections():
                    _lib.check(getattr(lib, f"{api}_train_backward_range")(*args, u0, u1), f"{api}_train_backward_range")
                    hook(names)
            else:
                _lib.check(getattr(lib, f"{api}_train_backward")(*args), f"{api}_train_backward")
        if direct:
            return [None] * len(plist)
        return [gflat[offs[n]:offs[n] + p.numel()].view_as(p) for n, p in plist]


class _TrainFn(torch.autograd.Function):
    """Train-mode forward / backward of the whole backbone + neck as one autograd node."""

    @staticmethod
    def forward(ctx, module, x, *params):
        ctx.module = module
        return module._train_forward(x)

    @staticmethod
    def backward(ctx, dout):
        return (None, None, *ctx.module._train_backward(dout))
