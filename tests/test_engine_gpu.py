"""GPU tests of the kept entry surface: engine.vision_engine.CenterProcessor.run_embedding (train -> EMA eval with the CBIR
metrics -> checkpoint with the reference's Epoch_N.pt key set), resume, the packed-weight cache of the EMA copy, and the
entry scripts themselves (main.py, validate.py, cbir_eval.py run as programs)."""
import os
import subprocess
import sys
import types

import pytest
import torch

from engine.vision_engine import CenterProcessor, check, increment_path, yaml_load
from visiondk_b200.backbone import BackboneFactory

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CFG = """
model:
  task: cbir
  image_size: &imgsz 64
  load_from: null
  backbone:
    timm-convnext_pico:
      pretrained: False
      image_size: *imgsz
      feat_dim: &featd 64
  head:
    circleloss:
      feat_dim: *featd
      num_class: 8
      margin: 0.25
      gamma: 64
data:
  root: synthetic://cbir?ids=8&per_id=16&queries=8
  nw: 0
  train: {bs: 16, base_aug: null, class_aug: null, augment: [], aug_epoch: 0}
  val: {bs: 16, metrics: {metrics: [mrr, recall, precision, auc, ndcg], cutoffs: [1, 5]}, augment: []}
hyp:
  epochs: EPOCHS
  lr0: 0.01
  lrf_ratio: null
  momentum: 0.937
  weight_decay: 0.0005
  warmup_momentum: 0.8
  warm_ep: 1
  loss: {ce: True}
  label_smooth: 0.1
  optimizer: [sgd, True]
  scheduler: cosine_with_warm
"""


def write_cfg(tmp_path, epochs=2, name="cbir.yaml"):
    f = tmp_path / name
    f.write_text(CFG.replace("EPOCHS", str(epochs)))
    return f


def test_run_embedding_trains_evaluates_and_checkpoints(lib, tmp_path):
    cfgs = yaml_load(str(write_cfg(tmp_path)))
    check("cbir", cfgs)
    out = increment_path(tmp_path / "run" / "exp")
    cp = CenterProcessor(cfgs, rank=-1, project=str(out))
    cp.run_embedding(None)
    ckpt = torch.load(out / "Epoch_2.pt", map_location="cpu", weights_only=False)
    assert {"epoch", "batch_id", "fitness", "state_dict", "ema", "updates", "optimizer", "scheduler"} <= set(ckpt)
    assert ckpt["epoch"] == 1 and ckpt["updates"] == 16
    # the in-training eval reports the reference's metric names (engine/cbir/evaluation.py:282-291), not a stub
    fit = ckpt["fitness"]["fitness"]
    assert {"MRR@1", "MRR@5", "Recall@1", "Recall@5", "Precision@1", "Precision@5", "AUC@5", "nDCG@1", "nDCG@5"} == set(fit)
    assert all(0.0 <= v <= 1.0 for k_, v in fit.items() if not (k_.startswith("AUC") and v != v)), fit  # AUC: nan if all hits
    model = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    model.load_state_dict(ckpt["ema"], strict=True)  # validate.py --ema path (face_model.py:73-86)
    emb = model.cuda().eval().embed(torch.randn(4, 3, 64, 64, device="cuda"), l2_normalize=True)
    assert torch.isfinite(emb).all() and emb.shape == (4, 64)
    # the EMA differs from the raw weights and both differ from initialisation (training happened)
    assert any((ckpt["ema"][k].float() - ckpt["state_dict"][k].float()).abs().max() > 0 for k in ckpt["ema"] if "weight" in k)


def test_ema_eval_sees_the_current_ema_weights(lib, tmp_path):
    """The optimizer kernels write EMA parameters through raw pointers (no `_version` bump): the packed inference weights of
    the EMA backbone must be re-packed after every step, so an eval after more training differs from the earlier one and
    equals a fresh model loaded from the same EMA state."""
    cfgs = yaml_load(str(write_cfg(tmp_path)))
    cp = CenterProcessor(cfgs, rank=-1, project=str(tmp_path / "run"))
    trainer = cp.run_embedding(None)
    ema_bb = trainer.ema.trainingwrapper["backbone"]
    x = torch.randn(8, 3, 64, 64, device="cuda")
    e1 = ema_bb.eval().embed(x, l2_normalize=True).clone()
    for it, (images, labels) in enumerate(cp.data.train_batches(7)):
        trainer.step(images, labels)
        if it == 5:
            break
    e2 = ema_bb.eval().embed(x, l2_normalize=True).clone()
    assert (e1 - e2).abs().max().item() > 1e-5, "EMA eval re-used packed weights from before the training steps"
    fresh = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    fresh.load_state_dict({k: v.detach().cpu().clone() for k, v in ema_bb.state_dict().items()}, strict=True)
    e3 = fresh.cuda().eval().embed(x, l2_normalize=True)
    assert torch.equal(e2, e3), (e2 - e3).abs().max().item()


def test_resume_restores_optimizer_scheduler_ema_and_head(lib, tmp_path):
    """vision_engine.py:494-507: 1 epoch + resume for the 2nd == 2 epochs in one go (same seeded batches): step counters,
    schedule position, momentum switch after warm-up, momentum buffers, EMA and head weights all carried over."""
    cfg2 = yaml_load(str(write_cfg(tmp_path, 2)))
    torch.manual_seed(3)
    full = CenterProcessor(cfg2, rank=-1, project=str(tmp_path / "full"))
    init = {k: v.detach().clone() for k, v in full.model.state_dict().items()}
    t_full = full.run_embedding(None)

    first = CenterProcessor(cfg2, rank=-1, project=str(tmp_path / "first"), opt=types.SimpleNamespace(save_freq=1, print_freq=50))
    first.model.load_state_dict(init)
    first.hyp_cfg = dict(first.hyp_cfg)
    # stop after epoch 1 by running a 2-epoch schedule for one epoch only
    import engine.vision_engine as ve
    orig = ve.CenterProcessor.save_and_eval
    calls = []

    def stop_after_first(self, trainer, epoch, spe):
        r = orig(self, trainer, epoch, spe)
        calls.append(epoch)
        if epoch == 0:
            raise StopIteration
        return r

    ve.CenterProcessor.save_and_eval = stop_after_first
    try:
        with pytest.raises(StopIteration):
            first.run_embedding(None)
    finally:
        ve.CenterProcessor.save_and_eval = orig
    second = CenterProcessor(cfg2, rank=-1, project=str(tmp_path / "second"))
    t_res = second.run_embedding(str(tmp_path / "first" / "Epoch_1.pt"))
    assert t_res.sched_step == t_full.sched_step == 16 and t_res.opt.updates == t_full.opt.updates == 16
    assert t_res.opt.steps == t_full.opt.steps
    assert [pg["momentum"] for pg in t_res.opt.param_groups] == [pg["momentum"] for pg in t_full.opt.param_groups] == [0.937, 0.937]
    assert [pg["lr"] for pg in t_res.opt.param_groups] == [pg["lr"] for pg in t_full.opt.param_groups]

    # the restore itself is exact: a fresh trainer resumed from the checkpoint holds the checkpoint's momentum buffers, EMA and
    # head weights bit for bit (a resume that forgot any of them would show up here, not in a tolerance)
    from visiondk_b200.train import FaceTrainer
    ck = torch.load(tmp_path / "first" / "Epoch_1.pt", map_location="cpu", weights_only=False)
    probe = CenterProcessor(cfg2, rank=-1, project=str(tmp_path / "probe"))
    hyp = probe.hyp_cfg
    t_probe = FaceTrainer(probe.model, lr0=hyp["lr0"], momentum=hyp["warmup_momentum"], weight_decay=hyp["weight_decay"],
                          label_smooth=hyp["label_smooth"], layer_wise=True, warm_steps=8, total_steps=16, use_ema=True)
    assert probe._resume(t_probe, str(tmp_path / "first" / "Epoch_1.pt")) == 1
    for g, m in zip(t_probe.opt.groups, ck["optimizer"]["momentum_buffers"]):
        assert torch.equal(g.mom.cpu(), m) and float(m.abs().max()) > 0
    assert t_probe.sched_step == 8 and t_probe.opt.updates == 8 and t_probe.opt.steps == 8
    for k_, v in probe.model.trainingwrapper["head"].state_dict().items():
        assert torch.equal(v.cpu(), ck["head"][k_])
    for k_, v in t_probe.ema.trainingwrapper["backbone"].state_dict().items():
        assert torch.equal(v.cpu(), ck["ema"][k_]), k_

    def close(a, b, what):
        err = (a.float() - b.float()).norm().item() / (b.float().norm().item() + 1e-12)
        # same kernels, same batches: run-to-run differences come from the summation order of atomics (largest on the
        # small bias vectors after 8 steps).  Parameters whose exact gradient is 0 (head.norm.* in front of a
        # batch-statistics BatchNorm) only ever move by rounding noise: for them the absolute difference is what is bounded.
        assert err <= 1e-2 or (a.float() - b.float()).abs().max().item() <= 5e-4, (what, err)

    for (n, a), (_, b) in zip(second.model.state_dict().items(), full.model.state_dict().items()):
        if a.dtype.is_floating_point:
            close(a, b, n)
    for (n, a), (_, b) in zip(t_res.ema.state_dict().items(), t_full.ema.state_dict().items()):
        if a.dtype.is_floating_point:
            close(a, b, "ema." + n)
    for ga, gb in zip(t_res.opt.groups, t_full.opt.groups):
        close(ga.mom, gb.mom, "momentum")


def test_sync_bn_is_refused_on_several_ranks_not_ignored(lib, tmp_path, monkeypatch):
    cfgs = yaml_load(str(write_cfg(tmp_path)))
    CenterProcessor(cfgs, rank=-1, opt=types.SimpleNamespace(sync_bn=True))  # one process: SyncBN == BN
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(NotImplementedError):
        CenterProcessor(cfgs, rank=0, opt=types.SimpleNamespace(sync_bn=True))


def test_entry_scripts_run_as_programs(lib, tmp_path):
    """main.py -> Epoch_1.pt; validate.py --weight --ema -> metrics dict; cbir_eval.py -> metrics dict (the reference's three
    entry points for this path, executed as the user would)."""
    cfg = write_cfg(tmp_path, 1)
    env = dict(os.environ, PYTHONPATH=ROOT)

    def run(args):
        r = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
        assert r.returncode == 0, f"{args}\nstdout:\n{r.stdout[-2000:]}\nstderr:\n{r.stderr[-3000:]}"
        return r.stdout

    out = run(["main.py", "--cfgs", str(cfg), "--project", str(tmp_path / "run"), "--name", "exp", "--save_freq", "1"])
    assert "MRR@1" in out and "Training complete" in out
    weight = tmp_path / "run" / "exp" / "Epoch_1.pt"
    assert weight.exists()
    out = run(["validate.py", "--cfgs", str(cfg), "--weight", str(weight), "--ema"])
    assert "MRR@1" in out and "nDCG@5" in out
    out = run(["cbir_eval.py", "--cfgs", str(cfg), "--weight", str(weight), "--ema", "--gallery", "128", "--queries", "8", "--k", "5"])
    assert "Recall@5" in out and "status" in out
