# coding=utf-8
"""Time one c5 micro-batch training step (forward + loss + BPTT over 128 trajectories, both scales; bench.py's c5
configuration) with each training option of code/train.py:85-92 against the default path.

  python tools/time_train_options.py [--rounds R] [--iters K]

Options run in alternating rounds so that clock drift and other tenants of the GPU spread over all of them; each
number is the median over rounds of the mean step time of K steps between CUDA events.  Prints one JSON line with
the GPU's name and power limit beside the times."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPTIONS = {               # soft grid mode (0: sparse labels), mask_grid_regression, train_w_onehot
    "default": (0, False, True),
    "soft7": (7, False, True),
    "mask": (0, True, True),
    "soft7_mask": (7, True, True),
    "logits_fed": (0, False, False),
}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--iters", type=int, default=10)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "timing needs a CUDA device"
  from bench import WORKLOADS
  from multiverse_b200 import build, synthetic
  from multiverse_b200.pred_models import _soft_labels
  from multiverse_b200.train_engine import TrainEngine
  build.build()
  dev = torch.device("cuda:0")
  wl = WORKLOADS["c5"]
  n = wl["micro_batch"]
  cfg = synthetic.make_config(batch_size=n, **wl["cfg"])
  w = {k: torch.from_numpy(v) for k, v in synthetic.make_weights(cfg).items()}
  f = synthetic.make_feeds(cfg, n, with_pred=True)
  up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  base = dict(scene_feat=up(f["scene_feat"]), obs_scene=up(f["obs_scene"]))
  for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_regress"):
    base[k] = [up(a) for a in f[k]]
  eng = TrainEngine(cfg, w, dev, 2)      # one engine (one activation store); the options are read per call
  feeds = {}

  def select(name):
    _, mask, onehot = OPTIONS[name]
    eng.cfg.mask_grid_regression, eng.cfg.train_w_onehot = mask, onehot
    return feeds[name]

  for name, (mode, _, _) in OPTIONS.items():
    feeds[name] = dict(base, grid_pred_labels=[up(_soft_labels(a, h, ww, mode)) if mode else up(a)
                                               for a, (h, ww) in zip(f["grid_pred_labels"], cfg.scene_grids)])
    for _ in range(2):
      eng.loss_and_grads(select(name))
  torch.cuda.synchronize()
  times = {name: [] for name in OPTIONS}
  for _ in range(args.rounds):
    for name in OPTIONS:
      fd = select(name)
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(args.iters):
        eng.loss_and_grads(fd)
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / args.iters)
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  med = {k: float(np.median(v)) for k, v in times.items()}
  print(json.dumps(dict(gpu=gpu, micro_batch=n, ms_per_step=med,
                        spread_ms={k: float(np.max(v) - np.min(v)) for k, v in times.items()},
                        vs_default={k: med[k] / med["default"] for k in med})))


if __name__ == "__main__":
  main()
