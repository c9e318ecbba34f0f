"""GPU tests of the training transform list (csrc/augment.cu via visiondk_b200.augment): every stage on its own against the
installed Pillow / torchvision, the reference Compose's own outputs (tests/golden/train_augment_ref.npz), batching, bounds of
the output writes, and an image-folder training run through CenterProcessor."""
import copy
import os
import random

import numpy as np
import pytest
import torch
import torchvision.transforms as T
import torchvision.transforms.functional as F
import yaml
from PIL import Image, ImageEnhance

from visiondk_b200 import _lib
from visiondk_b200.augment import (ImagePlan, TrainAugmenter, gaussian_kernel1d, pack_plans, parse_train_augment,
                                   rotate_matrix)

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
BIL, NEAR, CROP = _lib.AUG_RESIZE_PAD_BILINEAR, _lib.AUG_RESIZE_PAD_NEAREST, _lib.AUG_CROP_RESIZE


def ref_cfg(name):
    with open(os.path.join(GOLDEN, "reference_configs", f"{name}.yaml")) as f:
        return yaml.safe_load(f)


def augmenter(size):
    spec = parse_train_augment(ref_cfg("cbir")["data"]["train"]["augment"])
    return TrainAugmenter(type(spec)(spec.stages, size, MEAN, STD), "cuda")


def pil_tail(img, resize, crop, size):
    """What the reference does after the source-resolution stages: ResizeAndPadding2Square or the resized crop, then
    ToTensor + Normalize."""
    if resize == CROP:
        j, i, w, h = crop
        img = img.crop((j, i, j + w, i + h)).resize((size, size), Image.BILINEAR)
    else:
        w, h = img.size
        s = size / max(w, h)
        nw, nh = int(w * s), int(h * s)
        img = img.resize((nw, nh), Image.BILINEAR if resize == BIL else Image.NEAREST)
        canvas = Image.new("RGB", (size, size), (0, 0, 0))
        canvas.paste(img, ((size - nw) // 2, (size - nh) // 2))
        img = canvas
    return T.Normalize(MEAN, STD)(T.ToTensor()(img))


def to_bytes(x):
    m = torch.tensor(MEAN, device=x.device)[:, None, None]
    s = torch.tensor(STD, device=x.device)[:, None, None]
    return torch.round((x * s + m) * 255).clamp(0, 255).to(torch.uint8).cpu()


def image(w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx * 7 + yy * 3) % 256], axis=2)
    return np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)


SHAPES = [(64, 64), (37, 29), (3, 5), (97, 41), (150, 200), (1, 1)]


def cases():
    """(name, op record, PIL reference) with the parameters at their extremes."""
    out = []
    for a in (0.0, 0.37, 0.9, 1.0, 1.1, 2.0, 3.5):
        out.append((f"brightness{a}", (_lib.AUG_BRIGHTNESS, {"alpha": a}), lambda im, a=a: ImageEnhance.Brightness(im).enhance(a)))
        out.append((f"contrast{a}", (_lib.AUG_CONTRAST, {"alpha": a}), lambda im, a=a: ImageEnhance.Contrast(im).enhance(a)))
        out.append((f"saturation{a}", (_lib.AUG_SATURATION, {"alpha": a}), lambda im, a=a: ImageEnhance.Color(im).enhance(a)))
        out.append((f"sharpness{a}", (_lib.AUG_SHARPNESS, {"alpha": a}), lambda im, a=a: F.adjust_sharpness(im, a)))
    for f in (-0.5, -0.1, -0.0371, 0.003, 0.1, 0.25, 0.5):
        shift = int(np.int32(f * 255).astype(np.uint8))
        out.append((f"hue{f}", (_lib.AUG_HUE, {"hue_shift": shift}), lambda im, f=f: F.adjust_hue(im, f)))
    out.append(("hflip", (_lib.AUG_HFLIP, {}), F.hflip))
    return out


@pytest.mark.parametrize("resize", [BIL, NEAR])
def test_each_pixel_stage_matches_pil(lib, resize):
    aug = augmenter(64)
    for w, h in SHAPES:
        im = image(w, h, w * 131 + h)
        for name, op, ref in cases():
            got = aug.apply([im], [ImagePlan([op], resize)])[0]
            want = pil_tail(ref(Image.fromarray(im)), resize, None, 64).cuda()
            assert torch.equal(got, want), (name, (w, h), resize)


def test_rotation_and_cutout_match_pil(lib):
    aug = augmenter(64)
    for w, h in SHAPES:
        im = image(w, h, w + 7 * h)
        for angle in (-45.0, -10.0, -3.3, 0.01, 7.25, 10.0, 45.0):
            plan = ImagePlan([(_lib.AUG_ROTATE, {"matrix": rotate_matrix(angle, w, h)})], BIL)
            want = pil_tail(F.rotate(Image.fromarray(im), angle, T.InterpolationMode.BILINEAR), BIL, None, 64).cuda()
            assert torch.equal(aug.apply([im], [plan])[0], want), ("rotate", angle, (w, h))
        boxes = [(max(0, w // 2 - 6), max(0, h // 3 - 6), 11, 12), (0, 0, 13, 12), (max(0, w - 3), max(0, h - 2), 9, 12)]
        colors = [(255, 0, 17), (3, 200, 90), (0, 0, 0)]
        ref = Image.fromarray(im)
        for b, c in zip(boxes, colors):
            ref.paste(Image.new("RGB", (b[2], b[3]), c), (b[0], b[1]))
        plan = ImagePlan([(_lib.AUG_CUTOUT, {"boxes": boxes, "colors": colors})], BIL)
        assert torch.equal(aug.apply([im], [plan])[0], pil_tail(ref, BIL, None, 64).cuda()), ("cutout", (w, h))


def test_blur_within_one_unit_of_torchvision(lib):
    """Square images at their own size: the resample is the identity, so the bytes compared are the blur's."""
    worst, differ, total = 0, 0, 0
    for side in (3, 5, 31, 64, 128):
        aug = augmenter(side)
        im = image(side, side, side)
        for sigma in (0.1, 0.7, 1.3, 2.0):
            for ks in (3, 5):
                if ks // 2 >= side:
                    continue
                plan = ImagePlan([(_lib.AUG_BLUR, {"kernel": gaussian_kernel1d(ks, sigma).tolist()})], BIL)
                got = to_bytes(aug.apply([im], [plan])[0]).int()
                want = torch.from_numpy(np.asarray(F.gaussian_blur(Image.fromarray(im), [ks, ks], [sigma, sigma]))).permute(2, 0, 1).int()
                d = (got - want).abs()
                worst, differ, total = max(worst, int(d.max())), differ + int((d > 0).sum()), total + d.numel()
    assert worst <= 1 and differ <= 1e-4 * total, (worst, differ, total)


def test_resized_crop_matches_pil(lib):
    aug = augmenter(64)
    for (w, h), crop in (((97, 80), (3, 5, 60, 71)), ((64, 64), (0, 0, 64, 64)), ((150, 200), (20, 40, 130, 150)),
                         ((37, 29), (36, 28, 1, 1)), ((500, 375), (10, 0, 400, 375))):
        im = image(w, h, w * h)
        got = aug.apply([im], [ImagePlan([], CROP, crop)])[0]
        assert torch.equal(got, pil_tail(Image.fromarray(im), CROP, crop, 64).cuda()), ((w, h), crop)


def golden():
    z = np.load(os.path.join(GOLDEN, "train_augment_ref.npz"))
    imgs = [z[f"img{n}"] for n in range(len(z["shapes"]))]
    for r in range(int(z["runs"])):
        yield (str(z[f"run{r}_cfg"]), int(z[f"run{r}_size"]), int(z[f"run{r}_seed"]), imgs[:z[f"run{r}_out"].shape[0]],
               z[f"run{r}_out"])


def at_size(augment, size):
    aug = copy.deepcopy(augment)
    for a in aug:
        for t in a.get("random_choice", {}).get("transforms", []):
            for params in t.values():
                if isinstance(params, dict) and "size" in params:
                    params["size"] = size
    return aug


def test_reference_compose_outputs(lib):
    """Seeded like the reference's globals, the batch equals the reference Compose: exactly where no blur was drawn,
    within one unit (and on a small share of the bytes) where one was."""
    blur_stats = []
    for cfg, size, seed, imgs, outs in golden():
        spec = parse_train_augment(at_size(ref_cfg(cfg)["data"]["train"]["augment"], size))
        aug = TrainAugmenter(spec, "cuda")
        py, nprs, g = random.Random(seed), np.random.RandomState(seed), torch.Generator().manual_seed(seed)
        plans = aug.plans(imgs, py, nprs, g)
        got = to_bytes(aug.apply(imgs, plans)).numpy()
        for k, (p, want) in enumerate(zip(plans, outs)):
            d = np.abs(got[k].astype(int) - want.astype(int))
            if any(kind == _lib.AUG_BLUR for kind, _ in p.ops):
                blur_stats.append((int(d.max()), int((d > 0).sum()), d.size))
                assert d.max() <= 1, (cfg, size, seed, k, int(d.max()))
            else:
                assert d.max() == 0, (cfg, size, seed, k, [kind for kind, _ in p.ops], p.resize, int(d.max()), int((d > 0).sum()))
    differ = sum(s[1] for s in blur_stats)
    total = sum(s[2] for s in blur_stats)
    assert blur_stats and differ <= 1e-3 * total, blur_stats


def test_mixed_batch_equals_single_calls_and_writes_only_its_output(lib):
    spec = parse_train_augment(at_size(ref_cfg("cbir")["data"]["train"]["augment"], 96))
    aug = TrainAugmenter(spec, "cuda")
    z = np.load(os.path.join(GOLDEN, "train_augment_ref.npz"))
    imgs = [z[f"img{n}"] for n in range(len(z["shapes"]))]
    plans = aug.plans(imgs, random.Random(9), np.random.RandomState(9), torch.Generator().manual_seed(9))
    batch = aug.apply(imgs, plans)
    for k in range(len(imgs)):
        assert torch.equal(batch[k], aug.apply([imgs[k]], [plans[k]])[0]), k
    n = len(imgs)
    guard = torch.full((n + 2, 3, 96, 96), float("nan"), device="cuda")
    recs = pack_plans(plans)
    descs = aug._upload(imgs)
    lib = _lib.load()
    need = lib.vdk_augment_workspace_bytes(descs, recs, n, 96)
    ws = aug._workspace(need)
    _lib.check(lib.vdk_augment_batch(aug._dev.data_ptr(), descs, recs, n, 96, aug.mean, aug.std, guard[1].data_ptr(),
                                     ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_augment_batch")
    torch.cuda.synchronize()
    assert torch.isnan(guard[0]).all() and torch.isnan(guard[n + 1]).all()
    assert torch.equal(guard[1:n + 1], batch)


def test_bad_plans_are_refused(lib):
    aug = augmenter(64)
    im = image(20, 10, 1)
    with pytest.raises(RuntimeError, match="crop box"):
        aug.apply([im], [ImagePlan([], CROP, (5, 0, 20, 10))])
    with pytest.raises(RuntimeError, match="blur kernel"):
        aug.apply([image(2, 9, 1)], [ImagePlan([(_lib.AUG_BLUR, {"kernel": gaussian_kernel1d(5, 1.0).tolist()})], BIL)])


def test_center_processor_trains_on_an_image_folder(lib, tmp_path, monkeypatch):
    from engine.vision_engine import CenterProcessor
    from visiondk_b200 import train as TR
    rng = np.random.default_rng(3)
    for split, per in (("train", 8), ("gallery", 3), ("query", 1)):
        for c in range(8):
            d = tmp_path / "data" / split / f"id{c}"
            d.mkdir(parents=True)
            for k in range(per):
                w, h = int(rng.integers(40, 90)), int(rng.integers(40, 90))
                Image.fromarray(image(w, h, c * 100 + k)).save(d / f"{k}.{'png' if k % 2 else 'jpg'}")
    cbir = ref_cfg("cbir")
    cfgs = {
        "model": {"task": "cbir", "image_size": 64, "load_from": None,
                  "backbone": {"timm-convnext_pico": {"pretrained": False, "image_size": 64, "feat_dim": 64}},
                  "head": {"circleloss": {"feat_dim": 64, "num_class": 8, "margin": 0.25, "gamma": 64}}},
        "data": {"root": str(tmp_path / "data"), "nw": 2,
                 "train": {"bs": 16, "base_aug": None, "class_aug": None, "aug_epoch": 2,
                           "augment": at_size(cbir["data"]["train"]["augment"], 64)},
                 "val": {"bs": 16, "metrics": {"metrics": ["mrr", "recall"], "cutoffs": [1, 5]},
                         "augment": [{"resize_and_padding": {"size": 64, "training": False}}, {"to_tensor": "no_params"},
                                     {"normalize": {"mean": list(MEAN), "std": list(STD)}}]}},
        "hyp": {"epochs": 3, "lr0": 0.01, "lrf_ratio": None, "momentum": 0.937, "weight_decay": 0.0005, "warmup_momentum": 0.8,
                "warm_ep": 1, "loss": {"ce": True}, "label_smooth": 0.1, "optimizer": ["sgd", True], "scheduler": "cosine_with_warm"},
    }
    losses, fitness = [], []
    step = TR.FaceTrainer.step
    monkeypatch.setattr(TR.FaceTrainer, "step", lambda self, x, y: losses.append(float(step(self, x, y))) or torch.tensor(losses[-1], device=x.device))
    cp = CenterProcessor(cfgs, rank=-1, project=str(tmp_path / "run"))
    assert type(cp.data).__name__ == "FolderTrainData" and len(cp.data) == 4
    save = cp.save_and_eval
    cp.save_and_eval = lambda *a: fitness.append(save(*a)) or fitness[-1]
    cp.run_embedding()
    assert len(losses) == 12 and all(np.isfinite(losses)), losses
    assert [f["checkpoint"] for f in fitness] == ["Epoch_1.pt", "Epoch_2.pt", "Epoch_3.pt"]
    assert all((tmp_path / "run" / f"Epoch_{e}.pt").is_file() for e in (1, 2, 3))
    metrics = fitness[-1]["fitness"]
    assert metrics and all(np.isfinite(v) for v in metrics.values()), metrics
