"""Two ranks skip the same optimizer step when one rank's gradient is not finite (tools/check_nonfinite_skip.py under torchrun):
a NaN in rank 1's head shard with the class-sharded head, and a NaN in rank 1's backbone gradient with the plain DDP mean.

With >= 2 GPUs the ranks use NCCL, one GPU each; on a one-GPU box both ranks share cuda:0 and the collectives run over gloo."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_ranks_skip_a_step_with_one_rank_nonfinite(lib):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "check_nonfinite_skip.py")]
    env = dict(os.environ, OMP_NUM_THREADS="4")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert r.returncode == 0 and lines, f"rc={r.returncode}\nstdout:\n{r.stdout[-3000:]}\nstderr:\n{r.stderr[-3000:]}"
    out = json.loads(lines[-1])
    assert out["ok"], out
    assert out["backend"] == ("nccl" if torch.cuda.device_count() >= 2 else "gloo")
    checks = [k for k, v in out.items() if isinstance(v, bool) and k != "ok"]
    assert len(checks) == 2 * 9, checks
