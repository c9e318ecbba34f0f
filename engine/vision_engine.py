"""Orchestrator of the faceX / CBIR embedding path on H100 — the surface of the reference's
engine/vision_engine.py (yaml_load :35-38, increment_path :41-57, CenterProcessor.__init__ :67-167,
run_embedding :438-560) over the visiondk_b200 kernels.  Written from scratch: model / step / eval come from
visiondk_b200.{train,cbir} and engine.cbir.evaluation; `data.root` is a synthetic:// URL (engine/synthetic.py) or a local
image folder (engine/folder_train.py: decoded on host threads, the config's train / val transform lists on the device).
"""
from __future__ import annotations

import glob
import os
import re
import time
from pathlib import Path
from typing import Optional

import torch
import torch.distributed as dist
import yaml

from engine.cbir.evaluation import valuate as valuate_cbir
from engine.faceX.evaluation import valuate as valuate_face
from engine.folder_train import FolderTrainData
from engine.synthetic import SyntheticFaceData, is_synthetic
from visiondk_b200.train import FaceTrainer, FaceTrainingModel


def yaml_load(file="data.yaml", error_ok=False):
    with open(file, errors="ignore") as f:
        return yaml.safe_load(f)


def increment_path(path, exist_ok=False, sep="", mkdir=False):
    """run/exp -> run/exp2, run/exp3 ... (first free), like the reference's run-directory naming."""
    path = Path(path)
    if path.exists() and not exist_ok:
        base, suffix = (path.with_suffix(""), path.suffix) if path.is_file() else (path, "")
        taken = [int(m.group(1)) for d in glob.glob(f"{base}{sep}*")
                 if (m := re.search(rf"{re.escape(base.name)}{re.escape(sep)}(\d+)", d))]
        path = Path(f"{base}{sep}{max(taken) + 1 if taken else 2}{suffix}")
    if mkdir:
        path.mkdir(parents=True, exist_ok=True)
    return path


def check(task: str, cfgs: dict) -> None:
    """utils/checks.py:225-229 for the two embedding tasks: the schema the reference's configs/faceX/{face,cbir}.yaml follow
    (model{task,image_size,load_from,backbone{timm-<name>:{...}},head{<kind>:{feat_dim,num_class,...}}}, data{root,nw,train,val},
    hyp{...}) and its asserts (:111-143: the head's num_class equals the number of training identities; one backbone, one
    head; CE loss).  Raises ValueError / AssertionError with the reference's wording."""
    if task not in ("face", "cbir"):
        raise ValueError(f"{task} is not supported")
    for sec in ("model", "data", "hyp"):
        if sec not in cfgs:
            raise ValueError(f"Configuration error: missing top-level section '{sec}'")
    model_cfg, data_cfg, hyp_cfg = cfgs["model"], cfgs["data"], cfgs["hyp"]
    if model_cfg.get("task") != task:
        raise ValueError(f"Configuration error: model.task is {model_cfg.get('task')!r}, expected {task!r}")
    for sec, keys in ((model_cfg, ("image_size", "backbone", "head")), (data_cfg, ("root", "train", "val")),
                      (hyp_cfg, ("epochs", "lr0", "momentum", "weight_decay", "warmup_momentum", "warm_ep", "optimizer", "scheduler"))):
        for k in keys:
            if k not in sec:
                raise ValueError(f"Configuration error: missing key '{k}'")
    if len(model_cfg["backbone"]) != 1 or len(model_cfg["head"]) != 1:
        raise ValueError("Model configuration error: exactly one backbone and one head must be configured")
    backbone_key = next(iter(model_cfg["backbone"]))
    if backbone_key.split("-")[0] != "timm":
        raise ValueError("Model name error: Format should be [timm-ModelName] for timm models")
    bb = model_cfg["backbone"][backbone_key]
    head_key = next(iter(model_cfg["head"]))
    head = model_cfg["head"][head_key]
    if bb["feat_dim"] != head["feat_dim"]:
        raise ValueError("Model configuration error: backbone feat_dim and head feat_dim differ")
    if bb.get("image_size", model_cfg["image_size"]) != model_cfg["image_size"]:
        raise ValueError("Model configuration error: backbone image_size differs from model.image_size")
    loss = hyp_cfg.get("loss", {"ce": True})
    if not loss.get("ce", False):
        raise ValueError("Loss configuration error: the face / cbir tasks train with CE (hyp.loss.ce: true)")
    root = str(data_cfg["root"])
    if is_synthetic(root):
        num_classes = SyntheticFaceData(root, model_cfg["image_size"], 1, "cpu").num_classes
    elif os.path.isdir(root):
        train_dir = Path(root) / "train"
        if not train_dir.is_dir():
            raise ValueError(f"Training data error: {train_dir} not found")
        num_classes = len([x for x in os.listdir(train_dir) if not (x.startswith(".") or x.startswith("_"))])
    else:
        raise ValueError(f"Dataset loading error: {root} is neither a synthetic:// URL nor a local directory "
                         "(HuggingFace hub datasets need a network, which the GPU hosts may not have)")
    model_classes = head["num_class"]
    assert model_classes == num_classes, \
        f"Model configuration error: Number of classes mismatch. Expected {num_classes} from dataset, but got {model_classes} in model configuration"


class CenterProcessor:
    def __init__(self, cfgs: dict, rank: int, project: Optional[str] = None, train: bool = True, opt=None):
        self.cfgs, self.rank, self.project, self.opt = cfgs, rank, project, opt
        self.model_cfg, self.data_cfg, self.hyp_cfg = cfgs["model"], cfgs["data"], cfgs["hyp"]
        self.task = self.model_cfg["task"]
        if self.task not in ("face", "cbir"):
            raise ValueError("only the faceX / cbir embedding tasks are built for H100")
        if not torch.cuda.is_available():
            raise RuntimeError("visiondk_b200 needs a CUDA (sm_90a) device; there is no CPU path")
        self.device = torch.device("cuda", max(rank, 0))
        torch.cuda.set_device(self.device)
        self.world = int(os.environ.get("WORLD_SIZE", "1")) if rank != -1 else 1
        if getattr(opt, "sync_bn", False) and self.world > 1:
            # main.py:57-60 -> vision_engine.py:224-225 converts the neck's two BatchNorms to SyncBatchNorm.  The H100 neck
            # kernels normalise with the LOCAL batch statistics; silently ignoring the flag would train a different model.
            raise NotImplementedError("--sync_bn with WORLD_SIZE > 1: cross-rank BatchNorm statistics are not built for the "
                                      "H100 neck kernels (they use per-rank batch statistics); drop the flag")
        self.model = FaceTrainingModel(self.model_cfg).to(self.device)
        root = str(self.data_cfg["root"])
        if is_synthetic(root):
            self.data = SyntheticFaceData(root, self.model_cfg["image_size"], self.data_cfg["train"]["bs"], self.device,
                                          max(rank, 0), self.world)
        elif os.path.isdir(root):
            head = next(iter(self.model_cfg["head"].values()))
            self.data = FolderTrainData(root, self.data_cfg, head["num_class"], self.device, max(rank, 0), self.world,
                                        warm_ep=self.hyp_cfg.get("warm_ep", 0))
        else:
            raise NotImplementedError(f"{root}: dataset roots are a synthetic:// URL or a local directory (HuggingFace hub "
                                      "datasets need a network, which the GPU hosts may not have)")

    def log(self, msg: str):
        if self.rank in (-1, 0):
            print(msg, flush=True)

    # ---- fine-tune / resume (vision_engine.py:444-454, :494-507) -------------------------------------------------------
    def _load_from(self, path: str):
        state = torch.load(path, map_location="cpu", weights_only=False)
        state = state["ema"] if "ema" in state else state["model_state_dict"]
        missing, unexpected = self.model.trainingwrapper["backbone"].load_state_dict(state, strict=False)
        self.log(f"load_from: {path}")
        self.log(f"Missing keys: {missing}")
        self.log(f"Unexpected keys: {unexpected}")

    def _resume(self, trainer: FaceTrainer, path: str) -> int:
        """Restores everything the reference's checkpoint carries (:494-507: model, EMA + `updates`, optimizer, scheduler) and
        what it forgets (the head's class weights are not in its `state_dict` entry): backbone + head weights, EMA copies,
        momentum buffers, step counters, the position in the LR schedule and the post-warm-up momentum."""
        ckpt = torch.load(path, map_location="cpu", weights_only=False)
        wrap = self.model.trainingwrapper
        wrap["backbone"].load_state_dict(ckpt["state_dict"], strict=True)  # in place: the parameters live in the flat buffers
        if "head" in ckpt:
            wrap["head"].load_state_dict(ckpt["head"], strict=True)
        if trainer.ema is not None:
            trainer.ema.trainingwrapper["backbone"].load_state_dict(ckpt["ema"], strict=True)
            if "ema_head" in ckpt:
                trainer.ema.trainingwrapper["head"].load_state_dict(ckpt["ema_head"], strict=True)
        trainer.load_state_dict({"optimizer": ckpt["optimizer"], "scheduler": ckpt["scheduler"], "updates": ckpt["updates"]})
        start_epoch = ckpt["epoch"] + 1
        if start_epoch > self.hyp_cfg["warm_ep"]:  # the `epoch == warm_ep` switch below has already happened
            trainer.set_momentum(self.hyp_cfg["momentum"])
        self.log(f"resume: {path}")
        return start_epoch

    def run_embedding(self, resume: Optional[str] = None):
        hyp = self.hyp_cfg
        steps_per_epoch = len(self.data)
        name, layer_wise = hyp["optimizer"][0], bool(hyp["optimizer"][1])
        if name != "sgd" or hyp["scheduler"] != "cosine_with_warm":
            raise NotImplementedError("the H100 step implements sgd + cosine_with_warm (the faceX / cbir configs)")
        if self.model_cfg.get("load_from"):
            self._load_from(self.model_cfg["load_from"])
        trainer = FaceTrainer(self.model, lr0=hyp["lr0"], momentum=hyp["warmup_momentum"], weight_decay=hyp["weight_decay"],
                              label_smooth=hyp.get("label_smooth", 0.0), layer_wise=layer_wise,
                              warm_steps=hyp["warm_ep"] * steps_per_epoch, total_steps=hyp["epochs"] * steps_per_epoch,
                              lrf_ratio=hyp.get("lrf_ratio"), use_ema=self.rank in (-1, 0))
        start_epoch = self._resume(trainer, resume) if resume else 0
        t0 = time.time()
        save_freq = getattr(self.opt, "save_freq", 1) if self.opt else 1
        print_freq = getattr(self.opt, "print_freq", 50) if self.opt else 50
        for epoch in range(start_epoch, hyp["epochs"]):
            if epoch == hyp["warm_ep"]:
                trainer.set_momentum(hyp["momentum"])
            running, n = torch.zeros((), device=self.device), 0
            for it, (images, labels) in enumerate(self.data.train_batches(epoch)):
                running += trainer.step(images, labels)
                n += 1
                if (it + 1) % print_freq == 0:  # one device->host read per print, not per step
                    self.log(f"Epoch {epoch + 1}, iter {it + 1}/{steps_per_epoch}, lr {trainer.opt.param_groups[0]['lr']:.6f}, "
                             f"loss {running.item() / n:.4f}")
                    running.zero_()
                    n = 0
            if self.rank in (-1, 0) and (epoch + 1) % save_freq == 0:
                self.save_and_eval(trainer, epoch, steps_per_epoch)
        self.log(f"Training complete ({(time.time() - t0) / 3600:.3f} hours)")
        return trainer

    def save_and_eval(self, trainer: FaceTrainer, epoch: int, steps_per_epoch: int):
        """engine/procedure/train.py:244-278: evaluate the EMA backbone (face: pair verification -> Val_mean / Val_std; cbir:
        valuate_cbir -> {metric: float}), write Epoch_N.pt with
        the reference's key set, plus the entries a faithful resume needs ('head', 'ema_head', momentum buffers)."""
        src = trainer.ema if trainer.ema is not None else self.model
        ema_backbone = src.trainingwrapper["backbone"]
        if self.task == "face":  # train.py:246-253: 10-fold pair verification of the EMA backbone
            mean, std = valuate_face(ema_backbone, self.data_cfg, self.device, image_size=self.model_cfg["image_size"],
                                     n_pairs=getattr(self.opt, "eval_pairs", None) or 6000)
            metrics = {"Val_mean": float(mean), "Val_std": float(std)}
        else:  # train.py:254-260
            metrics = valuate_cbir(ema_backbone, self.data_cfg, self.device, None, image_size=self.model_cfg["image_size"],
                                   gallery_limit=getattr(self.opt, "eval_gallery", None) or 4096,
                                   query_limit=getattr(self.opt, "eval_queries", None) or 256)
        fitness = {"fitness": metrics, "checkpoint": f"Epoch_{epoch + 1}.pt"}
        out_dir = Path(self.project or "run/exp")
        out_dir.mkdir(parents=True, exist_ok=True)
        wrap = self.model.trainingwrapper
        state = trainer.state_dict()

        def host(sd):  # parameters are views into the optimizer's flat buffers: save compact per-tensor copies
            return {k: v.detach().cpu().clone() for k, v in sd.items()}

        ckpt = {"epoch": epoch, "batch_id": steps_per_epoch - 1, "fitness": fitness,
                "state_dict": host(wrap["backbone"].state_dict()), "ema": host(ema_backbone.state_dict()),
                "head": host(wrap["head"].state_dict()), "ema_head": host(src.trainingwrapper["head"].state_dict()),
                "updates": state["updates"], "optimizer": state["optimizer"], "scheduler": state["scheduler"]}
        torch.save(ckpt, out_dir / f"Epoch_{epoch + 1}.pt")
        self.log(str(fitness))
        return fitness
