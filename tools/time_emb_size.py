# coding=utf-8
"""Time --emb_size 128 against the published 32 (bench.py's configurations):
  decode  the c3 forward (256 trajectories, greedy two-scale with graph attention): the regression decoder's x block
          grows from one 32-channel chunk to two 64-channel chunks (cell FLOPs x 384 / 288 = 1.33); the class decoder
          folds its input into the epilogue, so its GEMM does not change;
  train   one c5-shaped micro-batch training step (forward + loss + BPTT over 128 trajectories, both scales): both
          decoders' x blocks, their dgrad / wgrad GEMMs and emb_bwd grow.

  python tools/time_emb_size.py [--rounds R] [--iters K]

The two sizes run in alternating rounds so that clock drift and other tenants of the GPU spread over both; each
number is the median over rounds of the mean time of K calls between CUDA events (device-resident feeds, eager
launches; each model on an engine of its own, built per round and warmed up by one call).  Prints one JSON line with
the GPU's name and power limit beside the times."""
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

SIZES = (32, 128)


def timed(run, iters):
  run()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    run()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--iters", type=int, default=5)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "timing needs a CUDA device"
  from bench import WORKLOADS
  from multiverse_b200 import build, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  from multiverse_b200.train_engine import TrainEngine
  build.build()
  dev = torch.device("cuda:0")
  up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  legs = {}
  for leg, wl, n, engine, pred in (("decode", WORKLOADS["c3"], WORKLOADS["c3"]["global_batch"], ConvRNNEngine, False),
                                   ("train", WORKLOADS["c5"], WORKLOADS["c5"]["micro_batch"], TrainEngine, True)):
    for emb in SIZES:
      cfg = synthetic.make_config(batch_size=n, **dict(wl["cfg"], emb_size=emb))
      f = synthetic.make_feeds(cfg, n, with_pred=pred)
      feeds = {k: ([up(a) for a in v] if isinstance(v, list) else up(v)) for k, v in f.items()
               if k not in ("traj", "traj64") and (pred or k not in ("grid_pred_labels", "grid_pred_regress"))}
      w = {k: torch.from_numpy(v) for k, v in synthetic.make_weights(cfg).items()}
      legs[(leg, emb)] = (engine, cfg, w, feeds)
  times = {"%s/emb%d" % k: [] for k in legs}
  for _ in range(args.rounds):
    for (leg, emb), (engine, cfg, w, feeds) in legs.items():
      eng = engine(cfg, w, dev, 2)
      run = (lambda: eng.forward(feeds)) if leg == "decode" else (lambda: eng.loss_and_grads(feeds))
      times["%s/emb%d" % (leg, emb)].append(timed(run, args.iters))
      del eng, run
      gc.collect()
      torch.cuda.empty_cache()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  med = {k: float(np.median(v)) for k, v in times.items()}
  print(json.dumps(dict(gpu=gpu, decode_trajectories=WORKLOADS["c3"]["global_batch"],
                        train_micro_batch=WORKLOADS["c5"]["micro_batch"], ms=med,
                        spread_ms={k: float(np.max(v) - np.min(v)) for k, v in times.items()},
                        emb128_vs_emb32={leg: med[leg + "/emb128"] / med[leg + "/emb32"]
                                         for leg in ("decode", "train")})))


if __name__ == "__main__":
  main()
