"""Image-folder source of the training split: the reference's local layout (dataset/basedataset.py:65-93)

    <root>/train/<class>/*.jpg|png        (class index = position of the directory name in sorted order)

with the reference's sampling (DistributedSampler over seed + epoch, padded to a multiple of the world size, rank-strided;
a drop_last loader) and its epoch schedule of transform lists (engine/vision_engine.py:539-550 of the reference): epochs
before `warm_ep` and from `aug_epoch` on take the val list (visiondk_b200.preprocess), the epochs between take the train list
(visiondk_b200.augment).  On a CUDA device the baseline JPEGs are decoded there (visiondk_b200.jpeg, bit-exact with
`read_image`), every other file on `nw` host threads, one batch ahead of the device."""
from __future__ import annotations

import math
import os
import random
from typing import Iterable, List, Optional, Sequence

import numpy as np
import torch

from engine.cbir.folder import decode_batches, device_decode_batches, parse_val_augment

SUFFIXES = (".jpg", ".png")


def list_classes(train_dir: str) -> List[str]:
    return sorted(d for d in os.listdir(train_dir)
                  if not (d.startswith(".") or d.startswith("_")) and os.path.isdir(os.path.join(train_dir, d)))


class FolderTrainData:
    """Train batches of a local root (same train surface as SyntheticFaceData: num_classes, __len__, train_batches)."""

    def __init__(self, root: str, data_cfg: dict, num_class: int, device, rank: int = 0, world: int = 1,
                 warm_ep: int = 0, seed: int = 0):
        from visiondk_b200.augment import parse_train_augment
        train_dir = os.path.join(root, "train")
        if not os.path.isdir(train_dir):
            raise ValueError(f"Training data error: {train_dir} not found")
        self.classes = list_classes(train_dir)
        if len(self.classes) != num_class:
            raise ValueError(f"Model configuration error: Number of classes mismatch. Expected {len(self.classes)} from "
                             f"dataset, but got {num_class} in model configuration")
        self.files: List[str] = []
        labels: List[int] = []
        for c, name in enumerate(self.classes):
            d = os.path.join(train_dir, name)
            fs = sorted(f for f in os.listdir(d) if os.path.splitext(f)[1].lower() in SUFFIXES)
            self.files += [os.path.join(d, f) for f in fs]
            labels += [c] * len(fs)
        self.labels = np.asarray(labels, np.int64)
        train = data_cfg["train"]
        self.train_spec = parse_train_augment(train["augment"], train.get("base_aug"), train.get("class_aug"),
                                              train.get("common_aug"))
        self.val_size, self.val_mean, self.val_std = parse_val_augment(data_cfg["val"]["augment"])
        self.batch, self.nw = int(train["bs"]), max(1, int(data_cfg.get("nw", 8)))
        self.aug_epoch = int(train.get("aug_epoch", 0))
        self.device, self.rank, self.world = torch.device(device), max(rank, 0), max(world, 1)
        self.warm_ep, self.seed = int(warm_ep), int(seed)
        self._val = self._train = None

    @property
    def num_classes(self) -> int:
        return len(self.classes)

    def __len__(self):  # DistributedSampler's per-rank count, drop_last batches
        return math.ceil(len(self.files) / self.world) // self.batch

    def uses_train_list(self, epoch: int) -> bool:
        return self.warm_ep <= epoch < self.aug_epoch

    def epoch_indices(self, epoch: int) -> List[int]:
        """torch.utils.data.DistributedSampler(shuffle=True, seed) after set_epoch(epoch), for this rank."""
        n = len(self.files)
        g = torch.Generator()
        g.manual_seed(self.seed + epoch)
        idx = torch.randperm(n, generator=g).tolist()
        total = math.ceil(n / self.world) * self.world
        pad = total - n
        if pad <= len(idx):
            idx += idx[:pad]
        else:
            idx += (idx * math.ceil(pad / len(idx)))[:pad]
        return idx[self.rank:total:self.world]

    def _transform(self, epoch: int):
        if self.uses_train_list(epoch):
            from visiondk_b200.augment import TrainAugmenter
            if self._train is None:
                self._train = TrainAugmenter(self.train_spec, self.device)
            s = 1000 * epoch + self.rank  # the augmentation streams of one (epoch, rank): a run is reproducible
            py, nprs, g = random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s)
            return lambda images: self._train(images, py, nprs, g)
        from visiondk_b200.preprocess import ImagePreprocessor
        if self._val is None:
            self._val = ImagePreprocessor(self.val_size, self.val_mean, self.val_std, self.device)
        return self._val

    def train_batches(self, epoch: int) -> Iterable:
        idx = self.epoch_indices(epoch)[:len(self) * self.batch]
        transform = self._transform(epoch)
        files = [self.files[i] for i in idx]
        labels = torch.from_numpy(self.labels[idx])
        batches = (device_decode_batches(files, self.batch, self.device, self.nw) if self.device.type == "cuda"
                   else decode_batches(files, self.batch, self.nw))
        for b, images in enumerate(batches):
            yield transform(images), labels[b * self.batch:(b + 1) * self.batch].to(self.device, non_blocking=True)
