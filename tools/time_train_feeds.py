# coding=utf-8
"""Time the drop-in training step end to end - Model.get_feed_dict + Trainer's sess.run (feeds to the device, step,
losses fetched) + a device synchronise - on dense feeds (the reference's feed dict: offsets, targets and soft label
maps built on the host) and on trajectory feeds (row f-1: the kernels compute them), alternating the two paths.

  python tools/time_train_feeds.py [--rounds R] [--iters K] [--bytes-only]

Two sizes: batch 1 024 in micro-batches of 128 on the published 36x64 scene (grids 18x32 + 9x16) with soft labels
(--soft_grid 1) and the masked regression - the shape of bench.py's c5 step - and TRAINING.md's batch of 20 (same
grids, --train_w_onehot, sparse labels).  Each number is the median over R rounds of the mean of K steps.  Prints one
JSON line with the GPU's name and power limit, and the host-to-device bytes per step of each path, computed from the
shapes of the fed arrays (--bytes-only prints those alone, without a GPU)."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {   # name: (batch, micro-batch, drop-in flags)
    "c5_1024_mb128_soft_mask": (1024, 128, dict(use_soft_grid_class=True, soft_grid=1, mask_grid_regression=True,
                                                train_w_onehot=False, grid_reg_loss_weight=0.1, init_lr=0.2)),
    "training_md_20": (20, 0, dict(use_soft_grid_class=False, soft_grid=1, mask_grid_regression=False,
                                   train_w_onehot=True, grid_reg_loss_weight=0.2, init_lr=0.3)),
}


def h2d_bytes(model, fd):
  """Bytes Trainer.step copies to the device for feed dict fd (Model._device_feeds and _train_step), from shapes."""
  cfg = model.config
  nb = lambda a, dt: int(np.asarray(a).size) * np.dtype(dt).itemsize
  traj = model.pred_traj in fd
  soft = bool(getattr(cfg, "use_soft_grid_class", False))
  b = nb(fd[model.scene_feat], np.float32) + nb(fd[model.obs_scene], np.int32)
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      continue
    b += nb(fd[model.grid_obs_labels[i]], np.int32)
    if traj:
      b += nb(fd[model.grid_centers[i]], np.float64) + nb(fd[model.grid_pred_labels_T[i]], np.int32)
    else:
      b += nb(fd[model.grid_obs_regress[i]], np.float32) + nb(fd[model.grid_pred_regress[i]], np.float32)
      b += nb(fd[model.grid_pred_labels_T[i]], np.float32 if soft else np.int32)
  if traj:
    b += nb(fd[model.obs_traj], np.float64) + nb(fd[model.pred_traj], np.float64)
  return b


def dropin(n, flags):
  """(tf shim, pred_models, model, args, batch) of a drop-in training model on the 36x64 scene, strides 2,4."""
  sys.path.insert(0, os.path.join(ROOT, "multiverse_b200", "dropin"))
  import tensorflow as tf
  import pred_models
  from multiverse_b200 import synthetic
  tf.reset_default_graph()
  cfg = synthetic.make_config(batch_size=n, is_train=True, grid_loss_weight=1.0, wd=0.001, clip_gradient_norm=10.0,
                              scene_h=36, scene_w=64, scene_grid_strides=[2, 4], use_grids=[True, True])
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname = "m"; args.use_gt_grid = False; args.use_teacher_forcing = False; args.optimizer = "adadelta"
  args.emb_lr = 1.0; args.learning_rate_decay = 0.95; args.num_epoch_per_decay = 2.0; args.train_num_examples = 10 ** 6
  args.use_cosine_lr = False
  for k, v in flags.items():
    setattr(args, k, v)
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  w = synthetic.make_weights(cfg, 7)
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  f = synthetic.make_feeds(cfg, n, 7, with_pred=True)
  ns, t = len(cfg.scene_grids), cfg.obs_len
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(n)],
              pred_grid_class=[np.stack([f["grid_pred_labels"][j][i] for j in range(ns)]) for i in range(n)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None],
              obs_traj=list(f["traj64"][:, :t]), pred_traj=list(f["traj64"][:, t:]))
  for j in range(ns):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  shared = {"grid_center_%d" % j: c for j, c in enumerate(synthetic.grid_centers(cfg))}
  return tf, pred_models, model, args, types.SimpleNamespace(data=data, shared=shared)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=5)
  ap.add_argument("--bytes-only", action="store_true")
  args = ap.parse_args()
  out = dict(h2d_bytes_per_step={}, ms_per_step={}, spread_ms={})
  for name, (n, mb, flags) in SIZES.items():
    tf, pred_models, model, margs, batch = dropin(n, flags)
    fds = dict(dense=lambda: model.get_feed_dict(batch, is_train=True),
               traj=lambda: model.get_feed_dict(batch, is_train=True, train_traj=True))
    out["h2d_bytes_per_step"][name] = {k: h2d_bytes(model, fd()) for k, fd in fds.items()}
    if args.bytes_only:
      continue
    import torch
    from multiverse_b200.train_engine import TrainEngine
    assert torch.cuda.is_available(), "timing needs a CUDA device"
    eng = model._ensure_engine()
    if mb:          # the drop-in step on the whole batch in micro-batches (TrainEngine.loss_and_grads_chunked)
      eng.train_step = lambda feeds, lr, dist=None, eng=eng: TrainEngine.train_step(eng, feeds, lr, dist, micro_batch=mb)
    trainer = pred_models.Trainer(model, margs)
    times = {k: [] for k in fds}
    with tf.Session() as sess:
      fetches = [model.loss, trainer.train_op, model.wd_loss, model.pred_grid_loss]
      for k in fds:                                 # warm-up: every buffer and kernel of both paths
        for _ in range(2):
          sess.run(fetches, feed_dict=fds[k]())
      torch.cuda.synchronize()
      for _ in range(args.rounds):
        for k in fds:
          t0 = time.perf_counter()
          for _ in range(args.iters):
            sess.run(fetches, feed_dict=fds[k]())   # get_feed_dict + Trainer.step's run, losses fetched
          torch.cuda.synchronize()
          times[k].append((time.perf_counter() - t0) * 1e3 / args.iters)
    out["ms_per_step"][name] = {k: float(np.median(v)) for k, v in times.items()}
    out["spread_ms"][name] = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
    model._engine = None
    del eng, trainer
    torch.cuda.empty_cache()
  if not args.bytes_only:
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
  print(json.dumps(out))


if __name__ == "__main__":
  main()
