"""Training-time image augmentation on the device: the reference's `data.train.augment` list (dataset/transforms.py:403-555,
configs/faceX/{face,cbir}.yaml) for a batch of decoded RGB images of different sizes.

    spec = parse_train_augment(cfg["data"]["train"]["augment"])
    aug = TrainAugmenter(spec, device="cuda")
    batch = aug(images, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))   # fp32 [n, 3, S, S]

The host draws every random parameter in the order and from the stream the reference's `T.Compose` draws it (Python
`random`: RandomChoice, RandomColorJitter's prob, Cutout, ResizeAndPadding2Square(training=True); numpy: the cutout centres;
torch's CPU generator: torchvision's `get_params` and RandomApply / RandomHorizontalFlip / RandomAdjustSharpness coins), so a
generator seeded like the reference's globals gives the reference's decisions.  The outcome is one vdk_aug_plan per image;
csrc/augment.cu applies it bit-exactly with Pillow (the blur within one unit of torch's CPU convolution).  No CPU fallback."""
from __future__ import annotations

import math
import random as _random
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .jpeg import DecodedBatch
from .preprocess import IMAGENET_MEAN, IMAGENET_STD, ImagePreprocessor

PIXEL_OPS = ("random_color_jitter", "random_cutout", "random_gaussianblur", "random_rotate", "random_adjustsharpness",
             "random_horizonflip")
RESIZE_OPS = ("resize_and_padding", "random_crop_and_resize")


@dataclass(frozen=True)
class Transform:
    name: str
    params: dict


@dataclass(frozen=True)
class Choice:
    options: Tuple[Transform, ...]
    p: Optional[Tuple[float, ...]]


@dataclass(frozen=True)
class TrainAugment:
    stages: Tuple[object, ...]   # Transform or Choice, the source-resolution stages then the resize stage, in list order
    size: int
    mean: Tuple[float, ...]
    std: Tuple[float, ...]


def _jitter_range(value, center: float, bound: Optional[Tuple[float, float]] = None, clip_zero: bool = True):
    """torchvision ColorJitter._check_input: a number v -> [center - v, center + v] (clipped at 0), a pair as given; the
    neutral range -> None (no draw)."""
    if isinstance(value, (int, float)):
        if value < 0:
            raise ValueError(f"color jitter value {value} must be non-negative")
        lo, hi = center - float(value), center + float(value)
        if clip_zero:
            lo = max(lo, 0.0)
    else:
        lo, hi = (float(v) for v in value)
    if bound is not None and not (bound[0] <= lo <= hi <= bound[1]):
        raise ValueError(f"color jitter range {(lo, hi)} outside {bound}")
    return None if lo == hi == center else (lo, hi)


def _pair(v, neg: bool = False) -> Tuple[float, float]:
    if isinstance(v, (int, float)):
        return (-float(v), float(v)) if neg else (float(v), float(v))
    a, b = v
    return float(a), float(b)


def _transform(name: str, params) -> Transform:
    """One registered transform with the defaults of its registration (dataset/transforms.py:402-528)."""
    kw = {} if params == "no_params" else dict(params)
    if name == "random_color_jitter":
        kw = {"prob": float(kw.get("prob", 0.5)),
              "brightness": _jitter_range(kw.get("brightness", 0), 1.0),
              "contrast": _jitter_range(kw.get("contrast", 0), 1.0),
              "saturation": _jitter_range(kw.get("saturation", 0), 1.0),
              "hue": _jitter_range(kw.get("hue", 0), 0.0, (-0.5, 0.5), clip_zero=False)}
    elif name == "random_cutout":
        kw = {"n_holes": int(kw.get("n_holes", 1)), "length": int(kw.get("length", 200)), "ratio": float(kw.get("ratio", 0.2)),
              "h_range": kw.get("h_range"), "w_range": kw.get("w_range"), "prob": float(kw.get("prob", 0.5)),
              "color": tuple(int(c) for c in kw.get("color", (0, 0)))}
        if kw["n_holes"] > _lib.AUG_MAX_HOLES:
            raise NotImplementedError(f"random_cutout: at most {_lib.AUG_MAX_HOLES} holes")
    elif name == "random_gaussianblur":
        ks = kw.get("kernel_size", 3)
        ks = (ks, ks) if isinstance(ks, int) else tuple(ks)
        if ks[0] != ks[1] or ks[0] % 2 == 0 or ks[0] > _lib.AUG_MAX_KERNEL:
            raise NotImplementedError(f"random_gaussianblur: kernel_size {ks}: square, odd and at most {_lib.AUG_MAX_KERNEL}")
        kw = {"prob": float(kw.get("prob", 0.5)), "kernel_size": int(ks[0]), "sigma": _pair(kw.get("sigma", (0.1, 2.0)))}
    elif name == "random_rotate":
        kw = {"degrees": _pair(kw["degrees"], neg=True)}
    elif name == "random_adjustsharpness":
        kw = {"sharpness_factor": float(kw.get("sharpness_factor", 2)), "p": float(kw.get("p", 0.5))}
    elif name == "random_horizonflip":
        kw = {"p": float(kw.get("p", 0.5))}
    elif name == "resize_and_padding":
        kw = {"size": int(kw.get("size", 224)), "training": bool(kw.get("training", False))}
    elif name == "random_crop_and_resize":
        kw = {"size": int(kw["size"]), "scale": _pair(kw.get("scale", (0.08, 1.0))),
              "ratio": _pair(kw.get("ratio", (3.0 / 4.0, 4.0 / 3.0)))}
    else:
        raise NotImplementedError(f"train.augment: {name!r} is not built for the device pipeline (supported: "
                                  f"{', '.join(PIXEL_OPS + RESIZE_OPS)}, random_choice, to_tensor, normalize)")
    return Transform(name, kw)


def parse_train_augment(augment: Sequence[dict], base_aug=None, class_aug=None, common_aug=None) -> TrainAugment:
    """data.train.augment (a list of one-key dicts, dataset/transforms.py:530-555) -> the typed plan of the supported list:
    source-resolution stages, one resize stage (or a random_choice of them), to_tensor, normalize."""
    for key, v in (("base_aug", base_aug), ("class_aug", class_aug), ("common_aug", common_aug)):
        if v is not None:
            raise NotImplementedError(f"train.{key}: class-wise augmentation is not built for the device pipeline")
    items = [next(iter(a.items())) for a in augment]
    names = [k for k, _ in items]
    if len(items) < 3 or names[-2:] != ["to_tensor", "normalize"]:
        for k in names:
            if k not in PIXEL_OPS + RESIZE_OPS + ("random_choice", "to_tensor", "normalize"):
                _transform(k, {})
        raise NotImplementedError(f"train.augment {names}: the device pipeline ends in a resize stage -> to_tensor -> normalize")
    stages: List[object] = []
    for name, params in items[:-2]:
        if name == "random_choice":
            opts = tuple(_transform(*next(iter(t.items()))) for t in params["transforms"])
            p = params.get("p")
            if p is not None and (not isinstance(p, (list, tuple)) or len(p) != len(opts)):
                raise ValueError("random_choice: p must list one weight per transform")
            stages.append(Choice(opts, None if p is None else tuple(float(x) for x in p)))
        else:
            stages.append(_transform(name, params))
    kinds = []
    for st in stages:
        opts = st.options if isinstance(st, Choice) else (st,)
        resize = {t.name in RESIZE_OPS for t in opts}
        if len(resize) != 1:
            raise NotImplementedError("random_choice mixes resize stages with source-resolution stages")
        kinds.append(resize.pop())
    if kinds.count(True) != 1 or not kinds[-1]:
        raise NotImplementedError("train.augment: the device pipeline needs exactly one resize stage "
                                  "(resize_and_padding / random_crop_and_resize), after every other stage")
    last = stages[-1]
    sizes = {t.params["size"] for t in (last.options if isinstance(last, Choice) else (last,))}
    if len(sizes) != 1:
        raise NotImplementedError(f"train.augment: resize stages of different sizes {sorted(sizes)}")
    norm = items[-1][1]
    mean = IMAGENET_MEAN if norm == "no_params" else tuple(float(v) for v in norm.get("mean", IMAGENET_MEAN))
    std = IMAGENET_STD if norm == "no_params" else tuple(float(v) for v in norm.get("std", IMAGENET_STD))
    return TrainAugment(tuple(stages), sizes.pop(), mean, std)


# ---- the per-image draws --------------------------------------------------------------------------------------------


def gaussian_kernel1d(kernel_size: int, sigma: float) -> torch.Tensor:
    """torchvision _functional_tensor._get_gaussian_kernel1d in fp32."""
    half = (kernel_size - 1) * 0.5
    x = torch.linspace(-half, half, steps=kernel_size, dtype=torch.float32)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    return pdf / pdf.sum()


def rotate_matrix(angle: float, w: int, h: int) -> List[float]:
    """PIL Image.rotate's affine matrix (no expand, centre (w / 2, h / 2)): output pixel centre -> input position."""
    ang = -math.radians(angle % 360.0)
    cx, cy = w / 2.0, h / 2.0
    m = [round(math.cos(ang), 15), round(math.sin(ang), 15), 0.0, round(-math.sin(ang), 15), round(math.cos(ang), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return m


@dataclass
class ImagePlan:
    ops: List[tuple]                # (kind, params dict) in application order
    resize: int                     # _lib.AUG_RESIZE_PAD_BILINEAR / _NEAREST / AUG_CROP_RESIZE
    crop: Tuple[int, int, int, int] = (0, 0, 0, 0)   # CROP_RESIZE: left, top, width, height


def _resize_and_padding(training: bool, py: _random.Random) -> int:
    if training:  # transforms.py:337-338
        return _lib.AUG_RESIZE_PAD_BILINEAR if py.random() < 0.5 else _lib.AUG_RESIZE_PAD_NEAREST
    return _lib.AUG_RESIZE_PAD_BILINEAR


def _resized_crop_params(w: int, h: int, scale, ratio, g: torch.Generator):
    """torchvision RandomResizedCrop.get_params: 10 attempts, then the centre crop."""
    area = h * w
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1], generator=g).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1], generator=g)).item()
        cw = int(round(math.sqrt(target_area * aspect_ratio)))
        ch = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < cw <= w and 0 < ch <= h:
            i = torch.randint(0, h - ch + 1, size=(1,), generator=g).item()
            j = torch.randint(0, w - cw + 1, size=(1,), generator=g).item()
            return j, i, cw, ch
    in_ratio = float(w) / float(h)
    if in_ratio < min(ratio):
        cw, ch = w, int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        ch, cw = h, int(round(h * max(ratio)))
    else:
        cw, ch = w, h
    return (w - cw) // 2, (h - ch) // 2, cw, ch


def sample_plan(spec: TrainAugment, w: int, h: int, py: _random.Random, nprs: np.random.RandomState,
                g: torch.Generator) -> ImagePlan:
    """One image's draws, in the order the reference's T.Compose makes them."""
    ops: List[tuple] = []
    plan = None
    for st in spec.stages:
        if isinstance(st, Choice):  # torchvision RandomChoice: random.choices(transforms, weights=p)[0]
            t = py.choices(st.options, weights=st.p)[0]
        else:
            t = st
        k = t.params
        if t.name == "random_color_jitter":  # transforms.py:170-179 + torchvision ColorJitter
            if not py.random() < k["prob"]:
                continue
            order = torch.randperm(4, generator=g).tolist()
            f = [None if k[n] is None else float(torch.empty(1).uniform_(k[n][0], k[n][1], generator=g))
                 for n in ("brightness", "contrast", "saturation", "hue")]
            for fn in order:
                if f[fn] is None:
                    continue
                if fn == 3:
                    ops.append((_lib.AUG_HUE, {"hue_shift": int(np.int32(f[3] * 255).astype(np.uint8))}))
                else:
                    ops.append(((_lib.AUG_BRIGHTNESS, _lib.AUG_CONTRAST, _lib.AUG_SATURATION)[fn], {"alpha": f[fn]}))
        elif t.name == "random_cutout":  # transforms.py:80-109
            if py.random() > k["prob"]:
                continue
            hr = k["h_range"] if k["h_range"] is not None else [0, h]
            wr = k["w_range"] if k["w_range"] is not None else [0, w]
            mask_w = int(py.uniform(1 - k["ratio"], 1 + k["ratio"]) * k["length"])
            mask_h = k["length"]
            boxes, colors = [], []
            for _ in range(k["n_holes"]):
                colors.append((py.randint(*k["color"]), py.randint(*k["color"]), py.randint(*k["color"])))
                y = int(nprs.randint(*hr))
                x = int(nprs.randint(*wr))
                boxes.append((max(0, x - k["length"] // 2), max(0, y - k["length"] // 2), mask_w, mask_h))
            ops.append((_lib.AUG_CUTOUT, {"boxes": boxes, "colors": colors}))
        elif t.name == "random_gaussianblur":  # T.RandomApply([T.GaussianBlur]) (transforms.py:510-512)
            if k["prob"] < torch.rand(1, generator=g):
                continue
            sigma = torch.empty(1).uniform_(k["sigma"][0], k["sigma"][1], generator=g).item()
            if k["kernel_size"] // 2 >= min(w, h):
                raise ValueError(f"random_gaussianblur: reflect padding {k['kernel_size'] // 2} needs both sides of the "
                                 f"{w} x {h} image to be larger")
            ops.append((_lib.AUG_BLUR, {"kernel": gaussian_kernel1d(k["kernel_size"], sigma).tolist()}))
        elif t.name == "random_rotate":  # T.RandomRotation(BILINEAR) (transforms.py:463-465)
            angle = float(torch.empty(1).uniform_(k["degrees"][0], k["degrees"][1], generator=g).item())
            if angle % 360.0 != 0.0:
                ops.append((_lib.AUG_ROTATE, {"matrix": rotate_matrix(angle, w, h)}))
        elif t.name == "random_adjustsharpness":  # T.RandomAdjustSharpness
            if torch.rand(1, generator=g).item() < k["p"]:
                ops.append((_lib.AUG_SHARPNESS, {"alpha": k["sharpness_factor"]}))
        elif t.name == "random_horizonflip":  # T.RandomHorizontalFlip
            if torch.rand(1, generator=g) < k["p"]:
                ops.append((_lib.AUG_HFLIP, {}))
        elif t.name == "resize_and_padding":
            plan = ImagePlan(ops, _resize_and_padding(k["training"], py))
        else:  # random_crop_and_resize (transforms.py:390-400)
            if max(h / w, w / h) > 1.5:
                plan = ImagePlan(ops, _resize_and_padding(True, py))
            else:
                plan = ImagePlan(ops, _lib.AUG_CROP_RESIZE, _resized_crop_params(w, h, k["scale"], k["ratio"], g))
    if len(plan.ops) > _lib.AUG_MAX_OPS:
        raise NotImplementedError(f"{len(plan.ops)} source-resolution stages for one image (at most {_lib.AUG_MAX_OPS})")
    return plan


def pack_plans(plans: Sequence[ImagePlan]):
    """ImagePlan list -> ctypes array of vdk_aug_plan."""
    arr = (_lib.AugPlan * len(plans))()
    for rec, p in zip(arr, plans):
        rec.n_ops, rec.resize = len(p.ops), p.resize
        rec.crop[:] = list(p.crop)
        for op, (kind, a) in zip(rec.ops, p.ops):
            op.kind = kind
            if "alpha" in a:
                op.alpha = a["alpha"]
            if "hue_shift" in a:
                op.hue_shift = a["hue_shift"]
            if "matrix" in a:
                op.matrix[:] = a["matrix"]
            if "kernel" in a:
                op.n = len(a["kernel"])
                op.kernel[:op.n] = a["kernel"]
            if "boxes" in a:
                op.n = len(a["boxes"])
                for j, (b, c) in enumerate(zip(a["boxes"], a["colors"])):
                    op.box[j][:] = list(b)
                    op.color[j][:] = list(c)
    return arr


class TrainAugmenter(ImagePreprocessor):
    """The training list on the device: draws plans on the host, then one vdk_augment_batch call per batch."""

    def __init__(self, spec: TrainAugment, device="cuda"):
        super().__init__(spec.size, spec.mean, spec.std, device)
        self.spec = spec

    def plans(self, images: Sequence[np.ndarray] | DecodedBatch, py: _random.Random, nprs: np.random.RandomState,
              g: torch.Generator) -> List[ImagePlan]:
        shapes = images.shapes if isinstance(images, DecodedBatch) else [im.shape for im in images]
        return [sample_plan(self.spec, s[1], s[0], py, nprs, g) for s in shapes]

    def __call__(self, images: Sequence[np.ndarray], py: _random.Random, nprs: np.random.RandomState,
                 g: torch.Generator) -> torch.Tensor:
        return self.apply(images, self.plans(images, py, nprs, g))

    def apply(self, images: Sequence[np.ndarray], plans: Sequence[ImagePlan]) -> torch.Tensor:
        lib = _lib.load()
        n = len(images)
        if n == 0:
            return torch.empty((0, 3, self.size, self.size), dtype=torch.float32, device=self.device)
        recs = pack_plans(plans)
        packed, descs = self._stage(images)
        with torch.cuda.device(self.device):
            need = lib.vdk_augment_workspace_bytes(descs, recs, n, self.size)
            if need == 0:
                raise RuntimeError("vdk_augment_workspace_bytes: " + _lib.last_error())
            ws = self._workspace(need)
            out = torch.empty((n, 3, self.size, self.size), dtype=torch.float32, device=self.device)
            _lib.check(lib.vdk_augment_batch(packed, descs, recs, n, self.size, self.mean, self.std, out.data_ptr(),
                                             ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_augment_batch")
        return out
