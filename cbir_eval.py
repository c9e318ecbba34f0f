#!/usr/bin/env python
"""cbir_eval.py — stand-alone CBIR evaluation on H100 (entry point kept from the reference; new code).

    python cbir_eval.py [--cfgs configs/faceX/cbir_convnext_b200.yaml] [--weight Epoch_N.pt] [--ema]
                        [--gallery 100000] [--queries 1000] [--k 10] [--index_factory IVF1024,PQ64 --nprobe 32]

The reference script (cbir_eval.py) hard-codes its paths, builds a random-init model, extracts gallery and query
embeddings, builds a faiss Flat/IP index and searches k=10.  This one does the same through visiondk_b200:
ConvNeXt embeddings on the sm_90a kernels, FlatIPIndex (or an IVF index, --index_factory / --nprobe) for index/search, everything resident in HBM.  Without a
dataset on disk it evaluates on synthetic images (random tensors: timing / plumbing) — real datasets plug in through
any iterable of [B,3,S,S] float tensors (the reference's CBIRDatasets + DataLoader yield exactly that).
"""
from __future__ import annotations

import argparse
import os
import time

import torch
import yaml

from engine.cbir.evaluation import compute_metrics
from engine.synthetic import SyntheticFaceData, is_synthetic
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.cbir import FeatureExtractor, index, search


class SyntheticImages:
    """Iterable of `n` random normalised images in batches of `bs`, generated on the device."""

    def __init__(self, n, bs, size, device, seed):
        self.n, self.bs, self.size, self.device, self.seed = n, bs, size, device, seed

    def __iter__(self):
        gen = torch.Generator(device=self.device).manual_seed(self.seed)
        for a in range(0, self.n, self.bs):
            b = min(self.bs, self.n - a)
            yield torch.randn(b, 3, self.size, self.size, device=self.device, generator=gen)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfgs", default="configs/faceX/cbir_convnext_b200.yaml")
    ap.add_argument("--weight", default=None, help="Epoch_N.pt written by the trainer (keys 'state_dict' / 'ema')")
    ap.add_argument("--ema", action="store_true")
    ap.add_argument("--gallery", type=int, default=20000)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--index_factory", default="Flat", help="'Flat', 'IVF<nlist>,Flat' or 'IVF<nlist>,PQ<M>[x8]'")
    ap.add_argument("--nprobe", type=int, default=1, help="lists probed per query by an IVF index")
    opt = ap.parse_args(argv)

    with open(opt.cfgs, errors="ignore") as f:
        cfgs = yaml.safe_load(f)
    model_cfg, data_cfg = cfgs["model"], cfgs["data"]
    device = torch.device(opt.device)
    model = BackboneFactory(model_cfg["backbone"]).get_backbone()
    if opt.weight:  # models/faceX/face_model.py:73-86
        ckpt = torch.load(opt.weight, map_location="cpu", weights_only=False)
        model.load_state_dict(ckpt["ema"] if opt.ema else ckpt["state_dict"], strict=True)
    extractor = FeatureExtractor(model)
    size, bs = model_cfg["image_size"], data_cfg["val"]["bs"]

    root = str(data_cfg["root"])
    if is_synthetic(root):  # identity-structured synthetic images: the metrics below mean something
        data = SyntheticFaceData(root, size, bs, device)
        gallery, queries = data.gallery_batches(opt.gallery), data.query_batches(opt.queries)
        g_label, q_label = data.gallery_labels(opt.gallery), data.query_labels(opt.queries)
    elif os.path.isdir(root):  # the reference's CBIRDatasets folder layout: decoded on host threads, transformed on the device
        from engine.cbir.folder import CBIRFolderData
        data = CBIRFolderData(root, data_cfg["val"]["augment"], bs, device, nw=data_cfg.get("nw", 8))
        gallery, queries = data.gallery_batches(opt.gallery), data.query_batches(opt.queries)
        g_label, q_label = data.gallery_labels(opt.gallery), data.query_labels(opt.queries)
    else:
        gallery, queries = SyntheticImages(opt.gallery, bs, size, device, 1), SyntheticImages(opt.queries, bs, size, device, 2)
        g_label = q_label = None
    t0 = time.perf_counter()
    faiss_index = index(extractor, gallery, device, index_factory=opt.index_factory)
    if opt.index_factory != "Flat":
        faiss_index.nprobe = opt.nprobe
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    scores, indices = search(extractor, queries, faiss_index, device, k=opt.k)
    t2 = time.perf_counter()
    n_q = scores.shape[0]
    print(f"indexed {faiss_index.ntotal} gallery images in {t1 - t0:.2f} s "
          f"({faiss_index.ntotal / (t1 - t0):.0f} embeddings/s incl. synthetic image generation)")
    print(f"searched {n_q} queries (k={opt.k}) in {t2 - t1:.3f} s; top-1 scores mean {scores[:, 0].mean():.4f}")
    if opt.index_factory == "Flat":
        print("status", faiss_index.check_status())
    else:
        print(f"{opt.index_factory} nprobe {faiss_index.nprobe}: {faiss_index.nbytes / max(faiss_index.ntotal, 1):.1f} bytes per row")
    if g_label is not None:  # cbir_eval.py:124-199 `evaluate`: metrics at the config's cutoffs (capped at k)
        cutoffs = [c for c in data_cfg["val"]["metrics"]["cutoffs"] if c <= opt.k] or [opt.k]
        m = compute_metrics(torch.from_numpy(indices).to(device), torch.from_numpy(scores).to(device), q_label, g_label,
                            metrics=data_cfg["val"]["metrics"]["metrics"], cutoffs=cutoffs)
        print({k_: round(float(v), 6) for k_, v in m.items()})
        return m


if __name__ == "__main__":
    main()
