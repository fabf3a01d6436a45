# coding=utf-8
"""Seconds for the single-future evaluation of a synthetic ActEV-shaped test set, end to end from get_batches to the
returned dict, three ways per configuration:
  host:     Tester.step (one sess.run per batch, dense logits and offsets fetched) + the NumPy restatement of
            pred_utils.evaluate (tests/single_future_eval_ref.py: the reference's own loop);
  dev_g1:   single_future_eval.evaluate, one batch per forward;
  dev_full: single_future_eval.evaluate at its default rows per forward (largest multiple of the batch <= 256).

Configurations: TESTING.md's test model (batch 16, use_grids 1,0) and TRAINING.md's validation (the training model,
batch 20, use_grids 1,1); scene 36x64 -> grids 18x32 and 9x16, emb 32, scene encoding, graph attention, synthetic
weights.  The test-set size is an ASSUMPTION (--n, default 2000 trajectories, 64 scene frames shared round-robin).
Median of `rounds` alternating rounds after one warm-up of each path; the card and its power limit are read in the
same run.

  python tools/time_single_future_eval.py [--n 2000] [--rounds 3] [--out results/time_sf_eval.json]
"""
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
sys.path.insert(0, os.path.join(ROOT, "multiverse_b200", "dropin"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = {
    "test_b16_grids10": (dict(batch_size=16, use_grids=[True, False]), False),
    "val_b20_grids11": (dict(batch_size=20, use_grids=[True, True]), True),
}
TRAIN_FLAGS = dict(grid_loss_weight=1.0, wd=0.001, clip_gradient_norm=10.0, optimizer="adadelta", emb_lr=1.0,
                   learning_rate_decay=0.95, num_epoch_per_decay=2.0, train_num_examples=100, use_cosine_lr=False,
                   use_soft_grid_class=False, soft_grid=1, mask_grid_regression=False, train_w_onehot=True,
                   init_lr=0.3, use_teacher_forcing=False)


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
  except OSError:
    return "unknown"


def setup(over, train, n):
  import tensorflow as tf
  import pred_models
  import single_future_eval_ref as ref
  from multiverse_b200 import synthetic
  sys.modules["pred_utils"] = ref
  tf.reset_default_graph()
  cfg = synthetic.make_config(scene_h=36, scene_w=64, scene_grid_strides=[2, 4], emb_size=32, use_scene_enc=True,
                              use_gnn=True, is_train=train, **over)
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname, args.use_gt_grid, args.per_scene_eval, args.save_output = "model", False, False, None
  args.use_soft_grid_class = False
  if train:
    for k, v in TRAIN_FLAGS.items():
      setattr(args, k, v)
  w = synthetic.make_weights(cfg, 3)
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  return tf, pred_models, model, args, ref.synthetic_dataset(args, n, 3, frames=64)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=2000)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  import torch
  import single_future_eval_ref as ref
  from multiverse_b200 import single_future_eval as sfe
  res = dict(card=card(), device=torch.cuda.get_device_name(0), n=a.n, rounds=a.rounds, configs={})
  for name, (over, train) in CONFIGS.items():
    tf, pred_models, model, args, ds = setup(over, train, a.n)
    with tf.Session() as sess:
      tester = pred_models.Tester(model, args, sess)
      paths = {"host": lambda: ref.evaluate(ds, args, ref.tester_step(model, sess))[0],
               "dev_g1": lambda: sfe.evaluate(ds, args, sess, tester, rows_per_forward=args.batch_size),
               "dev_full": lambda: sfe.evaluate(ds, args, sess, tester)}
      times, results = {k: [] for k in paths}, {}
      for k, f in paths.items():         # warm-up: engine buffers and graph captures of every batch size
        results[k] = f()
      same = all(results[k] == results["host"] for k in paths)
      for _ in range(a.rounds):
        for k, f in paths.items():
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          f()
          torch.cuda.synchronize()
          times[k].append(time.perf_counter() - t0)
    med = {k: float(np.median(v)) for k, v in times.items()}
    res["configs"][name] = dict(batch_size=args.batch_size, rows_per_forward=sfe.default_rows_per_forward(
        args.batch_size), train_model=train, seconds=med, all=times, equal_dicts=bool(same),
        speedup_full_vs_host=med["host"] / med["dev_full"], speedup_g1_vs_host=med["host"] / med["dev_g1"])
    print(name, json.dumps(res["configs"][name]), flush=True)
  print(json.dumps(res))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
