# coding=utf-8
"""Data-parallel training step on trajectory feeds (run under torchrun, see tests/test_ddp_traj_feeds_gpu.py): two ranks
fed their shard's trajectories, grid centres and label cells - the offsets, targets and soft label maps computed by the
kernels - with --use_soft_grid_class --soft_grid 7 --mask_grid_regression.  The foreground count K is counted once per
rank's batch from the label cells and all-reduced; every rank micro-batches its shard.  The all-reduced gradients, the
losses and the updated weights must equal one rank's step on the whole batch fed the dense tensors the host builds.

MVB_DDP_ONE_DEVICE=1 runs every rank on cuda:0 over gloo (the collectives copy through the host)."""
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
MB, MODE = 4, 7
N = 2 * MB * world
kw = dict(use_grids=[True, True], is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
          clip_gradient_norm=10.0)


def config(n):
  cfg = synthetic.make_config(batch_size=n, **kw)
  cfg.mask_grid_regression, cfg.train_w_onehot = True, False
  return cfg


cfg_full = config(N)
w = synthetic.make_weights(cfg_full, 3)
f = synthetic.make_feeds(cfg_full, N, 3, with_pred=True)
counts = []
for a, (h, ww) in zip(f["grid_pred_labels"], cfg_full.scene_grids):
  a[0, :4] = [0, ww - 1, (h - 1) * ww, h * ww - 1]          # corners: 4 of the 25 cells of a soft_grid 7 map remain
  m = _soft_labels(a, h, ww, MODE)
  counts.append([int((m[r * (N // world):(r + 1) * (N // world)] > 0).sum()) for r in range(world)])
assert all(len(set(c)) > 1 for c in counts), counts                # the shards' foreground counts differ
g = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
T = cfg_full.obs_len
centers = [g(c) for c in synthetic.grid_centers(cfg_full)]


def traj_feeds(r, wsize):
  sh = synthetic.shard_feeds(f, r, wsize)
  return dict(scene_feat=g(sh["scene_feat"]), obs_scene=g(sh["obs_scene"]),
              grid_obs_labels=[g(a) for a in sh["grid_obs_labels"]], grid_obs_regress=[None, None],
              grid_pred_regress=[None, None], grid_pred_labels=[g(a) for a in sh["grid_pred_labels"]],
              traj=dict(obs=g(sh["traj64"][:, :T]), pred=g(sh["traj64"][:, T:]), centers=centers, soft_grid=MODE))


def dense_feeds():
  return dict(scene_feat=g(f["scene_feat"]), obs_scene=g(f["obs_scene"]),
              grid_obs_labels=[g(a) for a in f["grid_obs_labels"]], grid_obs_regress=[g(a) for a in f["grid_obs_regress"]],
              grid_pred_regress=[g(a) for a in f["grid_pred_regress"]],
              grid_pred_labels=[g(_soft_labels(a, h, ww, MODE)) for a, (h, ww) in zip(f["grid_pred_labels"],
                                                                                      cfg_full.scene_grids)])


eng = TrainEngine(config(MB), {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
losses, _ = eng.train_step(traj_feeds(rank, world), 0.2, dist, micro_batch=MB)
ok = True
if rank == 0:
  full = TrainEngine(cfg_full, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  l_full, _ = full.train_step(dense_feeds(), 0.2, None)
  e_loss = float((losses - l_full).abs().max() / l_full.abs().max())
  e_grad = float((eng.flat_grad / world - full.flat_grad).abs().max() / full.flat_grad.abs().max())
  e_w = max(float((eng.params[k] - full.params[k]).abs().max()) for k in eng.names)
  moved = max(float((full.params[k].cpu() - torch.from_numpy(w[k])).abs().max()) for k in eng.names)
  print("DDP_CHECK trajectory feeds, soft_grid 7 + mask, micro-batch %d, K per shard %s: loss_rel=%.3e grad_rel=%.3e "
        "weight_abs=%.3e (update magnitude %.3e)" % (MB, counts, e_loss, e_grad, e_w, moved), flush=True)
  ok = e_loss < 1e-4 and e_grad < 5e-4 and e_w < 1e-3 * moved + 1e-7
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
