"""Cluster extracted embeddings with DBSCAN (cosine) on the GPU and optionally copy each cluster's images into its own folder:
the reference's tools/clustering.py without its hard-coded paths and its 1000-file cap.

    python tools/cluster_embeddings.py --features DIR [--images DIR --out DIR] [--eps 0.4] [--min_samples 5]
    python tools/cluster_embeddings.py --memmap PATH --feat_dim 512 [--dtype float16] [--eps 0.4] [--min_samples 5]

--features: one <name>.npy vector per image (the reference's layout), read in sorted order; with --images, only features
whose <name>.jpg exists are used, and cluster c's images are copied to <out>/<c>/.  --memmap: the raw embedding store
cbir.index(..., memmap_save_path=...) writes, read chunk by chunk.  Prints the reference's two lines.
"""
import argparse
import glob
import os
import shutil
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser()
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--features", help="directory of <name>.npy embedding files")
    src.add_argument("--memmap", help="raw embedding store (np.memmap, rows of --feat_dim)")
    ap.add_argument("--feat_dim", type=int, default=None)
    ap.add_argument("--dtype", choices=("float16", "float32"), default="float16")
    ap.add_argument("--images", default=None, help="directory of <name>.jpg images (with --features)")
    ap.add_argument("--out", default=None, help="copy each cluster's images to OUT/<label>/")
    ap.add_argument("--eps", type=float, default=0.4)
    ap.add_argument("--min_samples", type=int, default=5)
    opt = ap.parse_args(argv)
    if (opt.images is None) != (opt.out is None):
        ap.error("--images and --out go together")
    if opt.images is not None and opt.features is None:
        ap.error("--images needs --features (the image names come from the feature files)")
    from visiondk_b200.cluster import DBSCAN

    names = None
    if opt.features is not None:
        names, rows = [], []
        for npy in sorted(glob.glob(os.path.join(opt.features, "*.npy"))):
            name = os.path.basename(npy)[:-len(".npy")]
            if opt.images is not None and not os.path.isfile(os.path.join(opt.images, f"{name}.jpg")):
                continue
            rows.append(np.load(npy).reshape(-1))
            names.append(name)
        if not rows:
            ap.error(f"no usable .npy files under {opt.features}")
        X = np.stack(rows)
    else:
        if opt.feat_dim is None:
            ap.error("--memmap needs --feat_dim")
        X = np.memmap(opt.memmap, mode="r", dtype=opt.dtype).reshape(-1, opt.feat_dim)

    db = DBSCAN(eps=opt.eps, min_samples=opt.min_samples, metric="cosine").fit(X)
    labels = db.labels_
    n_clusters_ = len(set(labels.tolist())) - (1 if -1 in labels else 0)
    n_noise_ = int((labels == -1).sum())
    print("Estimated number of clusters: %d" % n_clusters_)
    print("Estimated number of noise points: %d" % n_noise_)

    if opt.out is not None:
        os.makedirs(opt.out, exist_ok=True)
        names = np.array(names)
        for label in range(n_clusters_):
            target = os.path.join(opt.out, str(label))
            os.makedirs(target, exist_ok=True)
            for name in names[labels == label]:
                shutil.copy(os.path.join(opt.images, f"{name}.jpg"), target)
    return labels


if __name__ == "__main__":
    main()
