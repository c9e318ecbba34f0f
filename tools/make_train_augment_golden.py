#!/usr/bin/env python
"""Mints tests/golden/train_augment_ref.npz by executing the REFERENCE's own training input pipeline (authoring container
only; never runs on the GPU).

    python tools/make_train_augment_golden.py

dataset/transforms.py is loaded by path (oracle.make_golden.load, as the eval-pipeline golden is) and its
`create_AugTransforms` builds the `data.train.augment` lists of the reference's own configs/faceX/{cbir,face}.yaml at the
config's image size and at 96 / 64.  Each run seeds the three global generators the Compose draws from (random,
numpy.random, torch) and passes synthetic images of assorted sizes through it: an aspect ratio above 1.5, sides below the
output size, odd sides, a 3-pixel side.  Stored: the uint8 inputs, each output as the uint8 image ToTensor saw (recovered
from the float tensor and checked to map back to it exactly), and one draw of each generator after the run's last image,
which fingerprints the generators' positions.  Smooth ramps (noisy on the small images only) keep the committed file small."""
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402

from oracle.make_golden import OUT, REF, load  # noqa: E402

SHAPES = [(120, 90), (90, 120), (200, 60), (37, 41), (33, 47), (3, 7), (64, 64), (97, 96), (100, 100), (45, 80), (81, 55),
          (4, 3), (60, 33), (110, 86), (31, 97), (70, 70)]
RUNS = ((None, 2, (0,)), (96, 8, (1,)), (64, 16, (3, 4)))   # (size (None = the config's), images, seeds)


def at_size(augment, size):
    return [{k: (dict(v, transforms=[{tk: (dict(tv, size=size) if isinstance(tv, dict) and "size" in tv else tv)
                                      for tk, tv in t.items()} for t in v["transforms"]])
                 if k == "random_choice" else v) for k, v in a.items()} for a in augment]


def main():
    from PIL import Image
    if not os.path.isdir(REF):
        sys.exit("make_train_augment_golden.py needs the reference tree (authoring container only)")
    ref = load("dataset/transforms.py", "ref_transforms_train")
    rng = np.random.default_rng(77)
    out = {"shapes": np.array(SHAPES, np.int32)}
    for n, (w, h) in enumerate(SHAPES):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx * 3 + yy * 5 + 40 * n) % 256], axis=2)
        noise = rng.integers(-12, 13, (h, w, 3)) if w * h <= 2500 else 0  # noise on the small images only: the file stays small
        out[f"img{n}"] = np.clip(base + noise, 0, 255).astype(np.uint8)
    run = 0
    for cfg_name in ("cbir", "face"):
        with open(os.path.join(REF, f"configs/faceX/{cfg_name}.yaml")) as f:
            cfg = yaml.safe_load(f)
        augment = cfg["data"]["train"]["augment"]
        mean = np.array(augment[-1]["normalize"]["mean"], np.float32)
        std = np.array(augment[-1]["normalize"]["std"], np.float32)
        for size, count, seeds in RUNS:
            size = size or int(cfg["model"]["image_size"])
            pipeline = ref.create_AugTransforms(at_size(augment, size))
            for seed in seeds:
                random.seed(seed)
                np.random.seed(seed)
                torch.manual_seed(seed)
                outs = []
                for n in range(count):
                    t = pipeline(Image.fromarray(out[f"img{n}"]))
                    assert tuple(t.shape) == (3, size, size) and t.dtype == torch.float32
                    u8 = np.clip(np.round((t.numpy() * std[:, None, None] + mean[:, None, None]) * 255), 0, 255).astype(np.uint8)
                    back = (torch.from_numpy(u8).float() / 255 - torch.from_numpy(mean)[:, None, None]) / torch.from_numpy(std)[:, None, None]
                    assert torch.equal(back, t), "uint8 recovery of the Compose output is not exact"
                    outs.append(u8)
                out[f"run{run}_cfg"] = np.array(cfg_name)
                out[f"run{run}_size"] = np.int32(size)
                out[f"run{run}_seed"] = np.int32(seed)
                out[f"run{run}_out"] = np.stack(outs)
                out[f"run{run}_fingerprint"] = np.array([random.random(), np.random.random(), torch.rand(1).item()], np.float64)
                run += 1
    out["runs"] = np.int32(run)
    path = os.path.join(OUT, "train_augment_ref.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {run} runs, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
