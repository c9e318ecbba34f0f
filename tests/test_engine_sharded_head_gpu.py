"""GPU test of `run_embedding` with the class-sharded head (`main.py --shard_head`) on one rank: the sharded run gathers its
head before the rank-0 save, so Epoch_N.pt has the unsharded run's keys and shapes, and each mode resumes from the other's
checkpoint with the head, EMA head and momentum bit for bit."""
import types

import pytest
import torch

from engine.vision_engine import CenterProcessor, yaml_load
from test_engine_gpu import write_cfg

pytestmark = pytest.mark.gpu


def _layout(tree):
    if isinstance(tree, dict):
        return {k: _layout(v) for k, v in tree.items() if k != "fitness"}
    if isinstance(tree, (list, tuple)):
        return [_layout(v) for v in tree]
    return (tuple(tree.shape), tree.dtype) if torch.is_tensor(tree) else type(tree).__name__


def _head_state(proc, trainer):
    if trainer.shard_head:
        return CenterProcessor.gathered_head_state(trainer)
    host = lambda sd: {k: v.detach().cpu().clone() for k, v in sd.items()}
    return {"head": host(proc.model.trainingwrapper["head"].state_dict()),
            "ema_head": host(trainer.ema.trainingwrapper["head"].state_dict()), "trainer": trainer.state_dict()}


def test_sharded_head_run_checkpoints_in_the_unsharded_layout_and_cross_resumes(lib, tmp_path):
    cfg = yaml_load(str(write_cfg(tmp_path, 1)))
    torch.manual_seed(3)
    plain = CenterProcessor(cfg, rank=-1, project=str(tmp_path / "plain"))
    init = {k: v.detach().clone() for k, v in plain.model.state_dict().items()}
    plain.run_embedding(None)
    sharded_opt = types.SimpleNamespace(shard_head=True, save_freq=1, print_freq=50)
    sharded = CenterProcessor(cfg, rank=-1, project=str(tmp_path / "sharded"), opt=sharded_opt)
    sharded.model.load_state_dict(init)
    t_s = sharded.run_embedding(None)
    assert t_s.shard_head
    cu = torch.load(tmp_path / "plain" / "Epoch_1.pt", map_location="cpu", weights_only=False)
    cs = torch.load(tmp_path / "sharded" / "Epoch_1.pt", map_location="cpu", weights_only=False)
    assert _layout(cs) == _layout(cu)
    for ck in (cu, cs):
        assert all(bool(torch.isfinite(m).all()) for m in ck["optimizer"]["momentum_buffers"])
    # both runs trained the same model on the same batches (run-to-run differences: the backbone backward's atomics)
    err = (cs["head"]["weight"] - cu["head"]["weight"]).norm() / cu["head"]["weight"].norm()
    assert float(err) < 1e-4, float(err)

    # the one-epoch schedule is over, so each resume only restores: sharded from the unsharded checkpoint and vice versa
    for opt, ck_dir, ck in ((sharded_opt, "plain", cu), (None, "sharded", cs)):
        proc = CenterProcessor(cfg, rank=-1, project=str(tmp_path / f"resume_from_{ck_dir}"), opt=opt)
        t = proc.run_embedding(str(tmp_path / ck_dir / "Epoch_1.pt"))
        got = _head_state(proc, t)
        assert torch.equal(got["head"]["weight"], ck["head"]["weight"])
        assert torch.equal(got["ema_head"]["weight"], ck["ema_head"]["weight"])
        for a, b in zip(got["trainer"]["optimizer"]["momentum_buffers"], ck["optimizer"]["momentum_buffers"]):
            assert torch.equal(a, b)
