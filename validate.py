#!/usr/bin/env python
"""validate.py — eval entry point (reference flags --cfgs --weight --ema --eval_topk): loads a checkpoint written by the
trainer (keys 'state_dict' / 'ema', models/faceX/face_model.py:73-86) into the H100 backbone and runs the CBIR evaluation
(engine/cbir/evaluation.py::valuate: extract -> index -> search -> MRR / Recall / Precision / AUC / nDCG at the config's
cutoffs), printing the metrics dict like the reference's validate.py:69-75; the face task runs the 10-fold pair verification
(engine/faceX/evaluation.py::valuate -> mean accuracy, standard error: validate.py:61-66).  New code over visiondk_b200."""
import argparse
import os

import torch

from engine.cbir.evaluation import valuate
from engine.faceX.evaluation import valuate as valuate_face
from engine.vision_engine import check, yaml_load
from visiondk_b200.backbone import BackboneFactory


def parse_opt():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfgs", default="configs/faceX/cbir_convnext_b200.yaml")
    ap.add_argument("--weight", default=None)
    ap.add_argument("--ema", action="store_true")
    ap.add_argument("--eval_topk", type=int, default=5)
    ap.add_argument("--gallery_limit", type=int, default=None, help="evaluate on the first N gallery items only")
    ap.add_argument("--query_limit", type=int, default=None)
    return ap.parse_args()


def main(opt):
    cfgs = yaml_load(opt.cfgs)
    task = cfgs["model"]["task"]
    if task not in ("face", "cbir"):
        raise ValueError(f"Unknown task {task}")  # validate.py:77 (the classification task is not an H100 path)
    check(task, cfgs)
    device = torch.device("cuda", int(os.getenv("LOCAL_RANK", 0)))
    model = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    if opt.weight:
        ckpt = torch.load(opt.weight, map_location="cpu", weights_only=False)
        model.load_state_dict(ckpt["ema"] if opt.ema else ckpt["state_dict"], strict=True)
    if task == "face":  # validate.py:61-66: pair verification, (mean accuracy, standard error)
        mean, std = valuate_face(model, cfgs["data"], device, image_size=cfgs["model"]["image_size"])
        name = os.path.basename(opt.weight) if opt.weight else "random-init"
        print(f"| model_name | mean accuracy | standard error |\n| {name} | {mean} | {std} |")
        return {"Val_mean": mean, "Val_std": std}
    metrics = valuate(model, cfgs["data"], device, None, image_size=cfgs["model"]["image_size"],
                      gallery_limit=opt.gallery_limit, query_limit=opt.query_limit)
    print(metrics)
    return metrics


if __name__ == "__main__":
    main(parse_opt())
