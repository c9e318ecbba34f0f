"""Times the training input pipeline of configs/faceX/cbir.yaml's `data.train.augment` list (not the bench contract) and
prints one JSON line with the card's name and power limit read in the same run:

    device_ms / device_img_s : vdk_augment_batch (host plan draws + upload + kernels) on 256 decoded ~500x375 images, CUDA events
    decode_img_s             : host JPEG decode alone on `nw` threads (engine.cbir.folder.read_image)
    pil_img_s                : the reference-equivalent PIL / torchvision Compose on every host core (processes), CPU baseline

    python tools/time_augment.py [--n 256] [--nw 64] [--iters 10]
Compare with the ConvNeXt-B train step's rate on the same card (README)."""
import argparse
import json
import multiprocessing as mp
import os
import random
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "tests", "golden", "reference_configs", "cbir.yaml")


def images(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        w, h = (500, 375) if k % 2 == 0 else (375, 500)
        w, h = w + int(rng.integers(-20, 21)), h + int(rng.integers(-20, 21))
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // w, yy * 255 // h, (xx + yy + 17 * k) % 256], axis=2)
        out.append(np.clip(base + rng.integers(-30, 31, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def pil_compose(augment):
    """The reference's train list built from torchvision / PIL pieces (dataset/transforms.py:63-109, 170-179, 325-400)."""
    import torchvision.transforms as T
    from PIL import Image, ImageOps

    class Cutout:
        def __init__(self, n_holes=1, length=200, ratio=0.2, prob=0.5, color=(0, 0)):
            self.n, self.length, self.ratio, self.prob, self.color = n_holes, length, ratio, prob, color

        def __call__(self, img):
            if random.random() > self.prob:
                return img
            img = img.copy()
            mw = int(random.uniform(1 - self.ratio, 1 + self.ratio) * self.length)
            for _ in range(self.n):
                mask = Image.new("RGB", (mw, self.length), tuple(random.randint(*self.color) for _ in range(3)))
                y, x = np.random.randint(0, img.height), np.random.randint(0, img.width)
                img.paste(mask, (max(0, x - self.length // 2), max(0, y - self.length // 2)))
            return img

    class Jitter(T.ColorJitter):
        def __init__(self, prob=0.5, **kw):
            super().__init__(**kw)
            self.prob = prob

        def forward(self, img):
            return super().forward(img) if random.random() < self.prob else img

    class ResizePad:
        def __init__(self, size, training=False):
            self.size, self.training = size, training

        def __call__(self, img):
            resample = (Image.BILINEAR if random.random() < 0.5 else Image.NEAREST) if self.training else Image.BILINEAR
            w, h = img.size
            s = self.size / max(w, h)
            nw, nh = int(w * s), int(h * s)
            img = img.resize((nw, nh), resample)
            pw, ph = (self.size - nw) // 2, (self.size - nh) // 2
            return ImageOps.expand(img, (pw, ph, self.size - nw - pw, self.size - nh - ph), fill=(0, 0, 0))

    class Crop(T.RandomResizedCrop):
        def __init__(self, size, **kw):
            super().__init__(size, **kw)
            self.fallback = ResizePad(size, True)

        def forward(self, img):
            w, h = img.size
            return self.fallback(img) if max(h / w, w / h) > 1.5 else super().forward(img)

    def one(name, p):
        p = {} if p == "no_params" else dict(p)
        return {"random_color_jitter": lambda: Jitter(**p), "random_cutout": lambda: Cutout(**p),
                "random_gaussianblur": lambda: T.RandomApply([T.GaussianBlur(p.get("kernel_size", 3), p.get("sigma", (0.1, 2.0)))],
                                                             p=p.get("prob", 0.5)),
                "random_rotate": lambda: T.RandomRotation(p["degrees"], interpolation=T.InterpolationMode.BILINEAR),
                "random_adjustsharpness": lambda: T.RandomAdjustSharpness(p.get("sharpness_factor", 2), p.get("p", 0.5)),
                "random_horizonflip": lambda: T.RandomHorizontalFlip(p.get("p", 0.5)),
                "resize_and_padding": lambda: ResizePad(**p), "random_crop_and_resize": lambda: Crop(**p),
                "to_tensor": T.ToTensor, "normalize": lambda: T.Normalize(**p)}[name]()

    out = []
    for a in augment:
        (name, p), = a.items()
        out.append(T.RandomChoice([one(*next(iter(t.items()))) for t in p["transforms"]]) if name == "random_choice" else one(name, p))
    return T.Compose(out)


_POOL_STATE = {}


def _pil_init(augment, files):
    from PIL import Image
    _POOL_STATE["compose"] = pil_compose(augment)
    _POOL_STATE["images"] = [Image.open(f).convert("RGB") for f in files]


def _pil_work(k):
    imgs = _POOL_STATE["images"]
    return tuple(_POOL_STATE["compose"](imgs[k % len(imgs)]).shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--nw", type=int, default=None, help="decode threads (default: the config's data.nw)")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_augment.py measures on a CUDA device; none is visible")
    from PIL import Image
    from engine.cbir.folder import decode_batches
    from visiondk_b200.augment import TrainAugmenter, parse_train_augment
    with open(CFG) as f:
        cfg = yaml.safe_load(f)
    augment, nw = cfg["data"]["train"]["augment"], args.nw or int(cfg["data"]["nw"])
    spec = parse_train_augment(augment)
    imgs = images(args.n)
    aug = TrainAugmenter(spec, "cuda")
    py, nprs, g = random.Random(0), np.random.RandomState(0), torch.Generator().manual_seed(0)
    for _ in range(2):
        aug(imgs, py, nprs, g)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        aug(imgs, py, nprs, g)
    e1.record()
    torch.cuda.synchronize()
    device_ms = e0.elapsed_time(e1) / args.iters

    with tempfile.TemporaryDirectory() as tmp:
        files = []
        for k, im in enumerate(imgs):
            files.append(os.path.join(tmp, f"{k}.jpg"))
            Image.fromarray(im).save(files[-1], quality=90)
        t0 = time.perf_counter()
        for _ in decode_batches(files, 80, nw):
            pass
        decode_s = time.perf_counter() - t0
        cores = os.cpu_count() or 1
        with mp.get_context("fork").Pool(cores, _pil_init, (augment, files[:32])) as pool:
            pool.map(_pil_work, range(cores))
            t0 = time.perf_counter()
            pool.map(_pil_work, range(args.n), chunksize=4)
            pil_s = time.perf_counter() - t0
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip() or torch.cuda.get_device_name(), "images": args.n,
                      "device_ms": round(device_ms, 3), "device_img_s": round(args.n / device_ms * 1e3, 1),
                      "decode_threads": nw, "decode_img_s": round(args.n / decode_s, 1),
                      "host_cores": cores, "pil_img_s": round(args.n / pil_s, 1)}))


if __name__ == "__main__":
    main()
