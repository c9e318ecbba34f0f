"""Face pair verification of the reference (engine/faceX/evaluation.py:8-140) on the H100 kernels — same names and argument
meaning: `process_pairtxt`, `Evaluator.test / test_one_model`, `valuate(model, data_cfg, device) -> (mean, std)`.

`valuate` = parse `data.val.pair_txt` (rows "<img a> <img b> <0|1>", images under <root>/val/) -> embed every distinct image once
(FeatureExtractor.extract_face: host decode, device val transforms, H100 backbone, L2-normalised) -> cosine score per pair ->
10-fold LFW protocol (threshold chosen on nine folds, accuracy on the tenth): visiondk_b200.metrics.face_verification_accuracy,
pinned to the reference's Evaluator by tests/golden/face_verification.npz.  Pair scores are one gather + row-wise dot on the
device instead of the reference's per-pair Python loop over a dict.  With a synthetic:// root the pairs are drawn from the
identity-structured synthetic images (half genuine, half impostor per fold), so the face task's in-training eval has a value."""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from engine.synthetic import SyntheticFaceData, is_synthetic
from visiondk_b200.cbir import FeatureExtractor
from visiondk_b200.metrics import face_verification_accuracy


def process_pairtxt(pair_txt: str, imgdir: str) -> Tuple[List[str], List[List[str]]]:
    """evaluation.py:8-19: -> (real paths of the distinct images, under <imgdir>/val/; pair rows [a, b, label])."""
    assert os.path.isfile(pair_txt), f"please check the path of {pair_txt}"
    pair_array = np.loadtxt(pair_txt, dtype=str, ndmin=2)
    unique_face_images = np.unique(pair_array[:, :2].flatten()).tolist()
    return [os.path.join(imgdir, "val", p) for p in unique_face_images], pair_array.tolist()


class Evaluator:
    def __init__(self, feature_extractor: FeatureExtractor):
        self.feature_extractor = feature_extractor

    @staticmethod
    def check_nps(pair_list: Sequence) -> None:
        assert len(pair_list) % 10 == 0, "make sure the number of rows is a multiple of 10 in pair.txt"  # evaluation.py:110-113

    def test(self, pair_list, feature_dataloader, device):
        Evaluator.check_nps(pair_list)
        image_name2feature = self.feature_extractor.extract_face(feature_dataloader, device)
        return self.test_one_model(pair_list, image_name2feature, device=device)

    def test_one_model(self, test_pair_list, image_name2feature: Dict[str, np.ndarray], is_normalize: bool = True, device="cuda"):
        """evaluation.py:34-82 -> (mean accuracy, standard error).  Names are looked up like the reference (os.path.normpath)."""
        names = list(image_name2feature)
        row = {n: i for i, n in enumerate(names)}
        feats = torch.from_numpy(np.stack([np.asarray(image_name2feature[n], np.float32) for n in names])).to(device)
        if not is_normalize:
            feats = feats / feats.norm(dim=1, keepdim=True)
        ia = torch.tensor([row[os.path.normpath(p[0])] for p in test_pair_list], device=feats.device)
        ib = torch.tensor([row[os.path.normpath(p[1])] for p in test_pair_list], device=feats.device)
        labels = torch.tensor([int(p[2]) for p in test_pair_list], device=feats.device)
        scores = (feats[ia] * feats[ib]).sum(dim=1)
        return face_verification_accuracy(scores, labels)


def image_batches(paths: Sequence[str], augment, batch: int, device, nw: int = 8):
    """(None, device tensors [b, 3, S, S], file paths) per batch — what PredictImageDatasets.collate_fn yields
    (dataset/basedataset.py:455-458) — with the baseline JPEGs decoded on the device (every other file on host threads)
    and the val transform list on the device."""
    from engine.cbir.folder import decode_batches, device_decode_batches, parse_val_augment
    from visiondk_b200.preprocess import ImagePreprocessor
    size, mean, std = parse_val_augment(augment)
    pre = ImagePreprocessor(size, mean, std, device)
    a = 0
    device = torch.device(device)
    batches = (device_decode_batches(list(paths), int(batch), device, nw) if device.type == "cuda"
               else decode_batches(list(paths), int(batch), nw))
    for images in batches:
        yield None, pre(images), list(paths[a:a + len(images)])
        a += len(images)


def synthetic_pair_scores(model, root: str, image_size: int, batch: int, device, n_pairs: int = 6000):
    """Pairs drawn from engine/synthetic.py's identities: per fold of n_pairs / 10, the first half genuine (two renderings of one
    identity), the second half impostors -> (scores [n_pairs] on the device, labels)."""
    data = SyntheticFaceData(root, image_size, batch, device)
    per = n_pairs // 10
    labels = (torch.arange(n_pairs, device=device) % per < per // 2).to(torch.int64)
    gen = torch.Generator(device=device).manual_seed(31)
    id_a = torch.randint(0, data.ids, (n_pairs,), device=device, generator=gen)
    shift = torch.randint(1, max(data.ids, 2), (n_pairs,), device=device, generator=gen)
    id_b = torch.where(labels == 1, id_a, (id_a + shift) % data.ids)
    model.eval()
    scores = []
    with torch.no_grad():
        for s in range(0, n_pairs, batch):
            fa = model.embed(data.render(id_a[s:s + batch], gen), l2_normalize=True)
            fb = model.embed(data.render(id_b[s:s + batch], gen), l2_normalize=True)
            scores.append((fa * fb).sum(dim=1))
    return torch.cat(scores), labels


def valuate(model, data_cfg: dict, device, image_size=None, n_pairs: int = 6000):
    """evaluation.py:115-140 -> (mean, std)."""
    device = torch.device(device)
    root = str(data_cfg["root"])
    if is_synthetic(root):
        size = image_size if image_size is not None else getattr(model, "image_size")
        scores, labels = synthetic_pair_scores(model.to(device), root, size, data_cfg["val"]["bs"], device, n_pairs)
        return face_verification_accuracy(scores, labels)
    test_images_path, pair_list = process_pairtxt(data_cfg["val"]["pair_txt"], root)
    loader = image_batches(test_images_path, data_cfg["val"]["augment"], data_cfg["val"]["bs"], device, nw=data_cfg.get("nw", 8))
    return Evaluator(FeatureExtractor(model)).test(pair_list, loader, device)
