"""Times JPEG decoding of image folders on the host and on the device (not the bench contract) and prints one JSON line with the
card's name and power limit read in the same run.  Two seeded corpora:
    A: the tools/time_augment.py images (256, about 500x375), saved at quality 90, 4:2:0
    B: 32 photo-like 4032x3024 images at quality 90, 4:2:0, without and with a restart interval (one MCU row)
Per corpus:
    host_img_s[nw]  : engine.cbir.folder.read_image on nw host threads (8 and 64)
    device_img_s    : files -> device RGB (visiondk_b200.jpeg.JpegDecoder: read, parse, upload, kernels, status read-back),
                      host clock around a synchronised batch
    kernel_ms       : per-kernel device time of one decode (torch.profiler, in a run of its own)
and for corpus A, alternating host and device decoding on the same folder: folder-fed ConvNeXt-B extraction
(CBIRFolderData -> embed, batch 256) and a folder-fed ConvNeXt-B train step (FolderTrainData val list -> FaceTrainer.step,
batch 128), in images/s.
With --progressive every file of both corpora is saved progressive (Pillow's default scan script, 10 scans), and kernel_ms
also lists the progressive Huffman kernel's time per dependency level (level_ms, one launch each).
    python tools/time_decode.py [--reps 3] [--progressive]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402


def write_corpora(root, progressive=False):
    from time_augment import images
    a_dir = os.path.join(root, "A", "gallery", "id0")
    os.makedirs(a_dir)
    for k, im in enumerate(images(256)):
        Image.fromarray(im).save(os.path.join(a_dir, f"{k:04d}.jpg"), quality=90, subsampling=2, progressive=progressive)
    os.makedirs(os.path.join(root, "A", "query", "id0"))
    Image.fromarray(images(1)[0]).save(os.path.join(root, "A", "query", "id0", "q.jpg"), quality=90, subsampling=2,
                                       progressive=progressive)
    rng = np.random.default_rng(1)
    for name, kw in (("B", {}), ("B_dri", {"restart_marker_rows": 1})):
        os.makedirs(os.path.join(root, name))
    for k in range(32):
        small = rng.integers(0, 256, (48, 63, 3), dtype=np.uint8)
        base = np.asarray(Image.fromarray(small).resize((4032, 3024), Image.BICUBIC), np.int16)
        im = Image.fromarray(np.clip(base + rng.integers(-12, 13, (3024, 4032, 3)), 0, 255).astype(np.uint8))
        im.save(os.path.join(root, "B", f"{k:02d}.jpg"), quality=90, subsampling=2, progressive=progressive)
        im.save(os.path.join(root, "B_dri", f"{k:02d}.jpg"), quality=90, subsampling=2, restart_marker_rows=1,
                progressive=progressive)


def host_rate(files, nw, reps):
    from engine.cbir.folder import read_image
    with ThreadPoolExecutor(nw) as pool:
        list(pool.map(read_image, files[:nw]))
        t = time.perf_counter()
        for _ in range(reps):
            list(pool.map(read_image, files))
        return reps * len(files) / (time.perf_counter() - t)


def device_rate(files, batch, reps):
    from engine.cbir.folder import read_image
    from visiondk_b200.jpeg import JpegDecoder
    dec = JpegDecoder("cuda", read_image, nw=8)
    chunks = [files[a:a + batch] for a in range(0, len(files), batch)]
    for c in chunks:
        b = dec(c)
        assert all(s == 0 for s in b.status), b.status
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        for c in chunks:
            dec(c)
    torch.cuda.synchronize()
    rate = reps * len(files) / (time.perf_counter() - t)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dec(chunks[0])
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        for k in ("entropy", "progressive", "idct", "color"):
            if f"jpeg_{k}_kernel" in ev.key:
                split[k] = split.get(k, 0.0) + ev.device_time_total / 1e3
    split = {k: round(v, 3) for k, v in split.items()}
    levels = [round(e.time_range.elapsed_us() / 1e3, 3) for e in prof.events()
              if "jpeg_progressive_kernel" in e.name and e.device_type.name == "CUDA"]
    if levels:
        split["level_ms"] = levels
    dec.close()
    return rate, split, len(chunks[0])


def folder_fed(root_a, reps):
    """(extraction img/s, train-step img/s) per decoder, host and device runs alternating."""
    import engine.cbir.folder as CF
    import engine.folder_train as FT
    from engine.cbir.folder import CBIRFolderData
    from visiondk_b200.backbone import TimmWrapper
    from visiondk_b200.train import FaceTrainer, FaceTrainingModel
    aug = [{"resize_and_padding": {"size": 224, "training": False}}, {"to_tensor": "no_params"}, {"normalize": "no_params"}]
    data = CBIRFolderData(root_a, aug, batch=256, device="cuda", nw=8)
    m = TimmWrapper("convnext_base", 512, 224, pretrained=False).cuda().eval()
    dev_decode = CF.device_decode_batches

    def host_decode(files, batch, device, nw):
        return CF.decode_batches(files, batch, nw)

    def extract(mode):
        CF.device_decode_batches = dev_decode if mode == "device" else host_decode
        try:
            torch.cuda.synchronize()
            t = time.perf_counter()
            with torch.no_grad():
                for x in data._device_batches(data.gallery_files):
                    m.embed(x, True)
            torch.cuda.synchronize()
            return len(data.gallery_files) / (time.perf_counter() - t)
        finally:
            CF.device_decode_batches = dev_decode

    train_root = os.path.join(os.path.dirname(root_a), "train_root")  # two classes (the head needs more than one): even / odd files
    for c in (0, 1):
        os.makedirs(os.path.join(train_root, "train", f"c{c}"))
    for k, f in enumerate(data.gallery_files):
        os.symlink(f, os.path.join(train_root, "train", f"c{k % 2}", os.path.basename(f)))
    import yaml
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs",
                           "cbir.yaml")) as f:
        data_cfg = yaml.safe_load(f)["data"]
    data_cfg = dict(data_cfg, nw=8, train=dict(data_cfg["train"], bs=128, aug_epoch=0), val=dict(data_cfg["val"], augment=aug))
    cfg = {"backbone": {"timm-convnext_base": {"pretrained": False, "image_size": 224, "feat_dim": 512}},
           "head": {"arcface": {"feat_dim": 512, "num_class": 2, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32}}}
    model = FaceTrainingModel(cfg).cuda()
    trainer = FaceTrainer(model, lr0=0.001, momentum=0.9, weight_decay=5e-4, label_smooth=0.1, layer_wise=True, warm_steps=0,
                          total_steps=100000, use_ema=True)
    tdata = FT.FolderTrainData(train_root, data_cfg, 2, "cuda")

    def train(mode):
        FT.device_decode_batches = dev_decode if mode == "device" else host_decode
        try:
            torch.cuda.synchronize()
            t = time.perf_counter()
            n = 0
            for x, y in tdata.train_batches(0):
                trainer.step(x, y)
                n += x.shape[0]
            torch.cuda.synchronize()
            return n / (time.perf_counter() - t)
        finally:
            FT.device_decode_batches = dev_decode

    out = {"extract": {"host": [], "device": []}, "train": {"host": [], "device": []}}
    for mode in ("host", "device"):  # warm-up
        extract(mode)
        train(mode)
    for _ in range(reps):
        for mode in ("host", "device"):
            out["extract"][mode].append(extract(mode))
            out["train"][mode].append(train(mode))
    return {k: {mode: round(float(np.median(v)), 1) for mode, v in d.items()} for k, d in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--progressive", action="store_true", help="save both corpora as progressive JPEGs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_decode.py measures on a CUDA device; none is visible")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    with tempfile.TemporaryDirectory() as root:  # the corpora (about 210 MB) are removed when the run ends
        write_corpora(root, args.progressive)
        res = {"gpu": q.stdout.strip().splitlines()[0] if q.stdout else "unknown", "host_cores": os.cpu_count(),
               "progressive": args.progressive}
        for name, d, batch in (("A", os.path.join(root, "A", "gallery", "id0"), 256), ("B", os.path.join(root, "B"), 32),
                               ("B_dri", os.path.join(root, "B_dri"), 32)):
            files = sorted(os.path.join(d, f) for f in os.listdir(d))
            reps = args.reps if name == "A" else 1
            r = {f"host_img_s_nw{nw}": round(host_rate(files, nw, reps), 1) for nw in (8, 64)}
            rate, split, nb = device_rate(files, batch, reps)
            r.update(device_img_s=round(rate, 1), kernel_ms=split, kernel_batch=nb,
                     mean_file_kb=round(sum(os.path.getsize(f) for f in files) / len(files) / 1024, 1))
            res[name] = r
        res["A"]["folder_fed_convnext_b"] = folder_fed(os.path.join(root, "A"), args.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
