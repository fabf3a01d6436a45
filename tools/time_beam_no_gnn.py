# coding=utf-8
"""Time the K=20 diverse-beam decode of 512 trajectories (bench.py's c4 configuration: 36x18 grid, obs 8 -> pred 12,
plus the greedy offset decoder) with the graph attention (c4 as published) and without it (use_gnn off, the models
code/multifuture_inference.py builds without --use_gnn).

  python tools/time_beam_no_gnn.py [--rounds R] [--iters K]

The configurations run in alternating rounds so that clock drift and other tenants of the GPU spread over both; each
number is the median over rounds of the mean forward time of K forwards between CUDA events (device-resident feeds,
eager launches; each configuration on an engine of its own, built per round).  Prints one JSON line with the GPU's
name and power limit beside the times."""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"c4": True, "no_gnn": False}     # use_gnn


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--iters", type=int, default=5)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "timing needs a CUDA device"
  from bench import WORKLOADS
  from multiverse_b200 import build, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  build.build()
  dev = torch.device("cuda:0")
  wl = WORKLOADS["c4"]
  n = wl["global_batch"]
  up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  # one engine at a time (two sets of beam buffers do not fit beside each other at this size), built per configuration
  # and round and warmed up by one forward before the timed ones
  cfgs = {name: synthetic.make_config(batch_size=n, **dict(wl["cfg"], use_gnn=use_gnn)) for name, use_gnn in CONFIGS.items()}
  w = {k: torch.from_numpy(v) for k, v in synthetic.make_weights(cfgs["c4"]).items()}   # the attention has no weights
  f = synthetic.make_feeds(cfgs["c4"], n)
  feeds = dict(scene_feat=up(f["scene_feat"]), obs_scene=up(f["obs_scene"]),
               grid_obs_labels=[up(a) for a in f["grid_obs_labels"]],
               grid_obs_regress=[up(a) for a in f["grid_obs_regress"]])
  times = {name: [] for name in CONFIGS}
  for _ in range(args.rounds):
    for name in CONFIGS:
      eng = ConvRNNEngine(cfgs[name], w, dev, 2)
      eng.forward(feeds)
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(args.iters):
        eng.forward(feeds)
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / args.iters)
      del eng
      gc.collect()
      torch.cuda.empty_cache()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  med = {k: float(np.median(v)) for k, v in times.items()}
  print(json.dumps(dict(gpu=gpu, trajectories=n, beam=wl["cfg"]["beam_size"], ms_per_forward=med,
                        spread_ms={k: float(np.max(v) - np.min(v)) for k, v in times.items()},
                        trajectories_per_s={k: n * 1e3 / v for k, v in med.items()})))


if __name__ == "__main__":
  main()
