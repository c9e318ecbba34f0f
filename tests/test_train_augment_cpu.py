"""The training transform list on the host: parsing the reference configs' `data.train.augment`, the plan sampler's draws
against the reference Compose (tests/golden/train_augment_ref.npz, minted by tools/make_train_augment_golden.py), and the
image-folder train source's host logic with a test double standing in for the device transforms."""
import copy
import os
import random

import numpy as np
import pytest
import torch
import yaml

from visiondk_b200 import _lib
from visiondk_b200.augment import Choice, parse_train_augment, sample_plan

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def ref_cfg(name):
    with open(os.path.join(GOLDEN, "reference_configs", f"{name}.yaml")) as f:
        return yaml.safe_load(f)


def at_size(augment, size):
    aug = copy.deepcopy(augment)
    for a in aug:
        for t in a.get("random_choice", {}).get("transforms", []):
            for params in t.values():
                if isinstance(params, dict) and "size" in params:
                    params["size"] = size
    return aug


@pytest.mark.parametrize("name", ["cbir", "face"])
def test_reference_train_lists_parse(name):
    cfg = ref_cfg(name)
    spec = parse_train_augment(cfg["data"]["train"]["augment"])
    assert spec.size == cfg["model"]["image_size"]
    assert spec.mean == (0.485, 0.456, 0.406) and spec.std == (0.229, 0.224, 0.225)
    assert isinstance(spec.stages[0], Choice) and isinstance(spec.stages[-1], Choice)
    assert [t.name for t in spec.stages[-1].options] == ["resize_and_padding", "random_crop_and_resize"]
    jitter = spec.stages[0].options[0]
    assert jitter.params["brightness"] == (0.9, 1.1) and jitter.params["hue"] == (-0.1, 0.1)


@pytest.mark.parametrize("bad", ["random_augment", "random_equalize", "random_affine", "random_grayscale", "center_crop"])
def test_unsupported_transforms_are_refused_by_name(bad):
    aug = ref_cfg("cbir")["data"]["train"]["augment"]
    with pytest.raises(NotImplementedError, match=bad):
        parse_train_augment([{bad: "no_params"}] + aug)
    inner = copy.deepcopy(aug)
    inner[0]["random_choice"]["transforms"].append({bad: "no_params"})
    with pytest.raises(NotImplementedError, match=bad):
        parse_train_augment(inner)


@pytest.mark.parametrize("key", ["base_aug", "class_aug", "common_aug"])
def test_class_wise_augmentation_is_refused(key):
    with pytest.raises(NotImplementedError, match=key):
        parse_train_augment(ref_cfg("cbir")["data"]["train"]["augment"], **{key: {"0": "0"}})


def test_a_list_without_a_final_resize_stage_is_refused():
    aug = ref_cfg("cbir")["data"]["train"]["augment"]
    with pytest.raises(NotImplementedError, match="resize stage"):
        parse_train_augment(aug[:2] + aug[-2:])
    with pytest.raises(NotImplementedError, match="resize stage"):
        parse_train_augment([aug[2], aug[1]] + aug[-2:])


def golden_runs():
    z = np.load(os.path.join(GOLDEN, "train_augment_ref.npz"))
    imgs = [z[f"img{n}"] for n in range(len(z["shapes"]))]
    for r in range(int(z["runs"])):
        yield (str(z[f"run{r}_cfg"]), int(z[f"run{r}_size"]), int(z[f"run{r}_seed"]), imgs[:z[f"run{r}_out"].shape[0]],
               z[f"run{r}_out"], z[f"run{r}_fingerprint"])


def test_sampler_draws_what_the_reference_compose_draws():
    """Same seeds -> every generator ends where the reference's left it, and each plan's resize stage matches the output:
    the pad band of a resize_and_padding image is black, a resized crop fills the square."""
    for cfg, size, seed, imgs, outs, fingerprint in golden_runs():
        spec = parse_train_augment(at_size(ref_cfg(cfg)["data"]["train"]["augment"], size))
        py, nprs, g = random.Random(seed), np.random.RandomState(seed), torch.Generator().manual_seed(seed)
        plans = [sample_plan(spec, im.shape[1], im.shape[0], py, nprs, g) for im in imgs]
        assert [py.random(), nprs.random_sample(), torch.rand(1, generator=g).item()] == fingerprint.tolist(), (cfg, size, seed)
        for im, p, out in zip(imgs, plans, outs):
            h, w = im.shape[:2]
            if p.resize == _lib.AUG_CROP_RESIZE:
                assert max(h / w, w / h) <= 1.5 and p.crop[2] <= w and p.crop[3] <= h
                continue
            nw, nh = int(w * (size / max(w, h))), int(h * (size / max(w, h)))
            left, top = (size - nw) // 2, (size - nh) // 2
            band = np.ones((size, size), bool)
            band[top:top + nh, left:left + nw] = False
            assert not out[:, band].any(), (cfg, size, seed, (w, h))


# ---- FolderTrainData host logic ----------------------------------------------------------------------------------------

PIL = pytest.importorskip("PIL")
from PIL import Image  # noqa: E402


class Recorder:
    """Stands in for the device transforms: records which list ran and returns one scalar per image."""
    calls = []

    def __init__(self, *args, **kwargs):
        self.kind = "train" if args and hasattr(args[0], "stages") else "val"

    def __call__(self, images, *streams):
        Recorder.calls.append((self.kind, len(images)))
        return torch.tensor([float(im[0, 0, 0]) for im in images])


def make_train_tree(root, counts):
    for c, n in counts.items():
        d = root / "train" / c
        d.mkdir(parents=True)
        for k in range(n):
            Image.fromarray(np.full((5 + k % 3, 6, 3), 10 * k % 256, np.uint8)).save(d / f"{k:03d}.{'PNG' if k % 2 else 'jpg'}")
        (d / "notes.txt").write_text("not an image")
    (root / "train" / ".hidden").mkdir()


def data_cfg(bs=4, aug_epoch=3):
    cfg = ref_cfg("cbir")["data"]
    cfg = copy.deepcopy(cfg)
    cfg["train"]["bs"], cfg["train"]["aug_epoch"], cfg["nw"] = bs, aug_epoch, 2
    return cfg


@pytest.fixture
def doubles(monkeypatch):
    import visiondk_b200.augment as A
    import visiondk_b200.preprocess as P
    monkeypatch.setattr(A, "TrainAugmenter", Recorder)
    monkeypatch.setattr(P, "ImagePreprocessor", Recorder)
    Recorder.calls = []
    return Recorder


def test_folder_train_data_classes_files_and_lengths(tmp_path, doubles):
    from engine.folder_train import FolderTrainData
    make_train_tree(tmp_path, {"b_cls": 5, "a_cls": 4, "c_cls": 2})
    d = FolderTrainData(str(tmp_path), data_cfg(), 3, "cpu")
    assert d.classes == ["a_cls", "b_cls", "c_cls"] and d.num_classes == 3
    assert len(d.files) == 11 and all(os.path.splitext(f)[1].lower() in (".jpg", ".png") for f in d.files)
    assert d.labels.tolist() == [0] * 4 + [1] * 5 + [2] * 2
    with pytest.raises(ValueError, match="Number of classes mismatch"):
        FolderTrainData(str(tmp_path), data_cfg(), 4, "cpu")
    for world in (1, 2, 3):
        parts = [FolderTrainData(str(tmp_path), data_cfg(bs=2), 3, "cpu", rank=r, world=world) for r in range(world)]
        idx = [p.epoch_indices(5) for p in parts]
        per = -(-11 // world)
        assert all(len(i) == per for i in idx) and len(parts[0]) == per // 2
        sampler = torch.utils.data.DistributedSampler(range(11), num_replicas=world, rank=0, shuffle=True, seed=0)
        sampler.set_epoch(5)
        assert idx[0] == list(sampler)
        assert sorted(set(sum(idx, []))) == list(range(11))


def test_folder_train_data_switches_lists_by_epoch(tmp_path, doubles):
    from engine.folder_train import FolderTrainData
    make_train_tree(tmp_path, {"x": 6, "y": 6})
    d = FolderTrainData(str(tmp_path), data_cfg(bs=4, aug_epoch=3), 2, "cpu", warm_ep=1)
    kinds = []
    for epoch in range(4):
        Recorder.calls = []
        batches = list(d.train_batches(epoch))
        assert len(batches) == len(d) == 3
        for (x, y), (kind, n) in zip(batches, Recorder.calls):
            assert n == 4 and x.shape == (4,) and y.shape == (4,)
        kinds.append({k for k, _ in Recorder.calls})
        labels = torch.cat([y for _, y in batches])
        expect = torch.from_numpy(d.labels[d.epoch_indices(epoch)[:12]])
        assert torch.equal(labels, expect)
    assert kinds == [{"val"}, {"train"}, {"train"}, {"val"}]
