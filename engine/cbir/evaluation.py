"""CBIR evaluation of the reference (engine/cbir/evaluation.py:106-291) on the H100 kernels — same function names and
argument meaning: `index`, `search`, `compute_metrics`, `valuate`.

`valuate` (:226-291) = build query / gallery loaders (shuffle=False) -> FeatureExtractor -> index(gallery) -> search(queries,
k = cutoffs[-1]) -> map returned ids to gallery entries, dropping -1 (:269-272) -> compute_metrics against every query's
positives (:274-291) -> {name: float}.  Embeddings, ids and scores stay on the device; relevance is an integer comparison of
identity labels (visiondk_b200.metrics) instead of the reference's per-query Python loops over path strings."""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from engine.synthetic import SyntheticFaceData, is_synthetic
from visiondk_b200 import metrics as M
from visiondk_b200.cbir import FeatureExtractor, index, search  # noqa: F401  (reference exports the same names)


def compute_metrics(ids: torch.Tensor, scores: torch.Tensor, query_label: torch.Tensor, gallery_label: torch.Tensor,
                    metrics: Sequence[str] = ("mrr", "precision", "recall", "auc", "ndcg"),
                    cutoffs: Sequence[int] = (1, 3, 10)) -> Dict[str, float]:
    """engine/cbir/evaluation.py:202-224 with the retrieval result as tensors: `ids`/`scores` [Nq,k] as `search` returns them
    (-1 padded), identity labels of queries and gallery items.  Keys and values as the reference's metrics dict."""
    rel, n_pos = M.relevance_from_labels(ids, query_label, gallery_label)
    out: Dict[str, float] = {}
    for m in metrics:
        try:
            out.update(M.cbir_metrics(ids, scores, rel, n_pos, cutoffs, [m]))
        except ValueError as e:
            # sklearn's roc_auc_score raises when the retrieved pairs are all relevant (or all irrelevant), which would abort the
            # reference's in-training eval on an easy dataset; report the metric as undefined instead of losing the checkpoint
            if m != "auc" or "one class" not in str(e):
                raise
            out[f"AUC@{list(cutoffs)[-1]}"] = float("nan")
    return out


def valuate(model, data_cfg: dict, device, logger=None, vis: bool = False, image_size: Optional[int] = None,
            gallery_limit: Optional[int] = None, query_limit: Optional[int] = None):
    """engine/cbir/evaluation.py:226-291.  `data_cfg['root']`: a synthetic:// URL (engine/synthetic.py) or a local directory in
    the reference's CBIRDatasets layout (<root>/query/<identity>/*, <root>/gallery/<identity>/*: engine/cbir/folder.py — images
    decoded on host threads, the val transform list on the device).  HuggingFace dataset names (basedataset.py:516-573) need the
    network and are not built.  `gallery_limit` / `query_limit` bound the in-training eval."""
    import os
    device = torch.device(device)
    root = str(data_cfg["root"])
    size = image_size if image_size is not None else getattr(model, "image_size")
    if is_synthetic(root):
        data = SyntheticFaceData(root, size, data_cfg["val"]["bs"], device)
    elif os.path.isdir(root):
        from engine.cbir.folder import CBIRFolderData
        data = CBIRFolderData(root, data_cfg["val"]["augment"], data_cfg["val"]["bs"], device, nw=data_cfg.get("nw", 8))
        if data.size != size:
            raise ValueError(f"val.augment resizes to {data.size} but the model takes {size} x {size} images")
    else:
        raise ValueError(f"Dataset loading error: {root} is neither a synthetic:// URL nor a local directory (HuggingFace "
                         "dataset names need the network and are not built)")
    extractor = FeatureExtractor(model)
    faiss_index = index(extractor, data.gallery_batches(gallery_limit), device, logger=logger)
    cutoffs = list(data_cfg["val"]["metrics"]["cutoffs"])
    q = extractor.extract_cbir_device(data.query_batches(query_limit), device)
    if logger is not None:
        logger.console("Searching ...")
    scores, ids = faiss_index.search_device(q, cutoffs[-1], resolve_overflow=True)
    q_label, g_label = data.query_labels(query_limit), data.gallery_labels(gallery_limit)
    if vis:  # (retrieval results, scores, ground truths, queries) like :279 — file lists for a folder root, label tensors otherwise
        if hasattr(data, "gallery_files"):
            files = data.gallery_files[:gallery_limit]
            results = [[files[j] for j in row if j != -1] for row in ids.cpu().tolist()]
            return results, scores.cpu().numpy(), data.positives(query_limit), data.query_files[:query_limit]
        return ids, scores, g_label, q_label
    out = compute_metrics(ids, scores, q_label, g_label, metrics=data_cfg["val"]["metrics"]["metrics"], cutoffs=cutoffs)
    return {k: float(v) for k, v in out.items()}
