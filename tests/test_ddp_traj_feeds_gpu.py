# coding=utf-8
"""Two-rank data-parallel training step on trajectory feeds (tests/ddp_check_traj_feeds.py), each rank micro-batching its
shard with soft labels + masked regression, equals the one-rank step on the whole batch fed dense tensors: NCCL on
two GPUs, and both ranks on one GPU over gloo."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(port, env):
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
         "--master-addr", "127.0.0.1", "--master-port", str(port),
         os.path.join(ROOT, "tests", "ddp_check_traj_feeds.py")]
  r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=dict(os.environ, **env))
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  assert "DDP_CHECK" in r.stdout
  print(r.stdout[r.stdout.index("DDP_CHECK"):].splitlines()[0])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_trajectory_feeds_equal_full_batch_nccl():
  run(29551, {})


@pytest.mark.skipif(torch.cuda.device_count() < 1, reason="needs a GPU")
def test_two_ranks_trajectory_feeds_equal_full_batch_one_device():
  run(29552, {"MVB_DDP_ONE_DEVICE": "1"})
