# coding=utf-8
"""Data-parallel equivalence of the masked regression loss on soft labels (run under torchrun, see
tests/test_ddp_train_options_gpu.py): with --use_soft_grid_class --soft_grid 7 --mask_grid_regression the foreground
count K differs between the shards (labels on the border of rank 0's rows lose cells), so "every loss is a mean over
equal shards" does not hold.  TrainEngine.train_step all-reduces K and divides each rank's Huber by K_all / G; the
all-reduced, 1/G-scaled gradients, the losses and the updated weights of G ranks must equal one rank's step on the
whole batch.

Backend nccl with one GPU per rank; MVB_DDP_ONE_DEVICE=1 runs every rank on cuda:0 over gloo (the collectives copy
through the host), for a machine with one GPU."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiverse_b200 import synthetic
from multiverse_b200.pred_models import _soft_labels
from multiverse_b200.train_engine import TrainEngine

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
one_device = os.environ.get("MVB_DDP_ONE_DEVICE") == "1"
dev = torch.device("cuda", 0 if one_device else local)
torch.cuda.set_device(dev)
if one_device:
  dist.init_process_group("gloo")
else:
  dist.init_process_group("nccl", device_id=dev)
N = 4 * world
kw = dict(use_grids=[True, True], is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
          clip_gradient_norm=10.0)


def config(n):
  cfg = synthetic.make_config(batch_size=n, **kw)
  cfg.mask_grid_regression = True
  return cfg


cfg_full = config(N)
w = synthetic.make_weights(cfg_full, 3)
f = synthetic.make_feeds(cfg_full, N, 3, with_pred=True)
soft, counts = [], []
for a, (h, ww) in zip(f["grid_pred_labels"], cfg_full.scene_grids):
  cls = np.array(a)
  cls[0, :4] = [0, ww - 1, (h - 1) * ww, h * ww - 1]         # corners: 4 of the 25 cells of a soft_grid 7 map remain
  m = _soft_labels(cls, h, ww, 7)
  soft.append(m)
  counts.append([int((m[r * (N // world):(r + 1) * (N // world)] > 0).sum()) for r in range(world)])
f["grid_pred_labels"] = soft
assert all(len(set(c)) > 1 for c in counts), counts                # the shards' foreground counts differ
g = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def feeds_of(r, wsize):
  sh = synthetic.shard_feeds(f, r, wsize)
  return {k: ([g(a) for a in v] if isinstance(v, list) else g(v)) for k, v in sh.items() if k != "traj"}


eng = TrainEngine(config(N // world), {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
losses, _ = eng.train_step(feeds_of(rank, world), 0.2, dist)
ok = True
if rank == 0:
  full = TrainEngine(cfg_full, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  l_full, _ = full.train_step(feeds_of(0, 1), 0.2, None)
  e_loss = float((losses - l_full).abs().max() / l_full.abs().max())
  e_grad = float((eng.flat_grad / world - full.flat_grad).abs().max() / full.flat_grad.abs().max())
  e_w = max(float((eng.params[k] - full.params[k]).abs().max()) for k in eng.names)
  moved = max(float((full.params[k].cpu() - torch.from_numpy(w[k])).abs().max()) for k in eng.names)
  print("DDP_CHECK soft_grid 7 + mask, K per shard %s: loss_rel=%.3e grad_rel=%.3e weight_abs=%.3e (update magnitude "
        "%.3e)" % (counts, e_loss, e_grad, e_w, moved), flush=True)
  ok = e_loss < 1e-4 and e_grad < 5e-4 and e_w < 1e-3 * moved + 1e-7
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
