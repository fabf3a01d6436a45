# coding=utf-8
"""Data-parallel equivalence of a model built without --use_scene_enc (run under torchrun, see
tests/test_no_scene_enc_gpu.py): its class encoder's embedding person_pred/grid_emb is one variable shared by both
scales, a gradient that every rank accumulates over its scales and steps before the one all-reduce.  The all-reduced,
1/G-scaled gradients, the losses and the updated weights of G ranks must equal one rank's step on the whole batch.
Every rank runs on cuda:0 over gloo (the collectives copy through the host), for a machine with one GPU."""
import os, sys
import torch
import torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiverse_b200 import synthetic
from multiverse_b200.engine import ENC_EMB
from multiverse_b200.train_engine import TrainEngine

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
dist.init_process_group("gloo")
N = 4 * world
kw = dict(use_grids=[True, True], is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.2, wd=0.001,
          clip_gradient_norm=10.0, use_scene_enc=False)
cfg_full = synthetic.make_config(batch_size=N, **kw)
w = synthetic.make_weights(cfg_full, 4)
f = synthetic.make_feeds(cfg_full, N, 4, with_pred=True)
g = lambda x: torch.from_numpy(x).to(dev)


def feeds_of(r, wsize):
  sh = synthetic.shard_feeds(f, r, wsize)
  return {k: ([g(a) for a in v] if isinstance(v, list) else g(v)) for k, v in sh.items() if k not in ("traj", "traj64")}


eng = TrainEngine(synthetic.make_config(batch_size=N // world, **kw), {k: torch.from_numpy(v) for k, v in w.items()},
                  dev, 2)
losses, _ = eng.train_step(feeds_of(rank, world), 0.3, dist)
ok = True
if rank == 0:
  full = TrainEngine(cfg_full, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  l_full, _ = full.train_step(feeds_of(0, 1), 0.3, None)
  e_loss = float((losses - l_full).abs().max() / l_full.abs().max())
  e_grad = float((eng.flat_grad / world - full.flat_grad).abs().max() / full.flat_grad.abs().max())
  e_emb = float((eng.grads[ENC_EMB[0]] / world - full.grads[ENC_EMB[0]]).abs().max()
                / full.grads[ENC_EMB[0]].abs().max())
  e_w = max(float((eng.params[k] - full.params[k]).abs().max()) for k in eng.names)
  moved = max(float((full.params[k].cpu() - torch.from_numpy(w[k])).abs().max()) for k in eng.names)
  print("DDP_CHECK without scene encoding: loss_rel=%.3e grad_rel=%.3e grid_emb_rel=%.3e weight_abs=%.3e (update "
        "magnitude %.3e)" % (e_loss, e_grad, e_emb, e_w, moved), flush=True)
  ok = e_loss < 1e-4 and e_grad < 5e-4 and e_emb < 5e-4 and e_w < 1e-3 * moved + 1e-7
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
