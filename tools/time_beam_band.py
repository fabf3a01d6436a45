# coding=utf-8
"""Time bench.py's c4 forward (512 trajectories, K=20 diverse beam on the 36x18 grid, obs 8 -> pred 12, plus the
greedy offset decoder) with the beam decoder's image-row bands on (default) and off (MVB_BEAM_BAND=0).

  python tools/time_beam_band.py [--rounds R] [--iters K]

The two settings alternate on one engine, R rounds each.  Per setting it prints the median over rounds of
  - the forward time: mean of K forwards between CUDA events (device-resident feeds, eager launches);
  - the K=20 beam cell launch: mean over the forward's ten launches (engine.cell_events, tag "beam").  With the bands
    on this is the launch on the work list; the base rollout's launches (tag "beam_base") and the copies are not in it.
It also prints the share of the full launch's M tiles that the tracker's work list holds at every beam step (times
2 .. 11), next to an estimate from a CPU replay of the reference decoder on the same synthetic inputs: the share of
the launch's own 128-row tiles that touch a band.  One JSON line, with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CPU_ESTIMATE = [0.36, 0.36, 0.53, 0.63, 0.67, 0.77, 0.81, 0.89, 0.94, 0.98]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=3)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "timing needs a CUDA device"
  from bench import WORKLOADS
  from multiverse_b200 import build, ops, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  build.build()
  dev = torch.device("cuda:0")
  wl = WORKLOADS["c4"]
  n = wl["global_batch"]
  cfg = synthetic.make_config(batch_size=n, **wl["cfg"])
  h, w = cfg.scene_grids[0]
  ns = n * cfg.beam_size
  up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  f = synthetic.make_feeds(cfg, n)
  feeds = dict(scene_feat=up(f["scene_feat"]), obs_scene=up(f["obs_scene"]),
               grid_obs_labels=[up(a) for a in f["grid_obs_labels"]],
               grid_obs_regress=[up(a) for a in f["grid_obs_regress"]])
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in synthetic.make_weights(cfg).items()}, dev, 2)
  settings = {"band": "1", "full": "0"}
  step_ms = {k: [] for k in settings}
  beam_ms = {k: [] for k in settings}
  counts = []
  real_band = ops.beam_band

  def track(ids, parents, band_in, band_out, tiles, tile_count, *a):
    real_band(ids, parents, band_in, band_out, tiles, tile_count, *a)
    counts.append(tile_count)
  for r in range(args.rounds):
    for name, env in settings.items():
      os.environ["MVB_BEAM_BAND"] = env
      eng.forward(feeds)                       # warm-up
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(args.iters):
        eng.forward(feeds)
      e1.record()
      torch.cuda.synchronize()
      step_ms[name].append(e0.elapsed_time(e1) / args.iters)
      eng.cell_events = []
      if r == 0 and name == "band":
        ops.beam_band = track
      eng.forward(feeds)
      ops.beam_band = real_band
      torch.cuda.synchronize()
      launches = [a.elapsed_time(b) for tag, _, a, b in eng.cell_events if tag == "beam"]
      eng.cell_events = None
      beam_ms[name].append(float(np.mean(launches)))
  full_tiles = -(-ns * (h + 1) * (w + 1) // 128)
  frac = [round(int(c[0].item()) / full_tiles, 3) for c in counts[1:]]     # the fan-out step (time 1) has no list
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  med = {k: float(np.median(v)) for k, v in step_ms.items()}
  print(json.dumps(dict(gpu=gpu, trajectories=n, beam=cfg.beam_size, grid=[h, w], rounds=args.rounds,
                        ms_per_forward=med, spread_ms={k: float(np.ptp(v)) for k, v in step_ms.items()},
                        trajectories_per_s={k: n * 1e3 / v for k, v in med.items()},
                        beam_launch_ms={k: float(np.median(v)) for k, v in beam_ms.items()},
                        tile_fraction=frac, tile_fraction_mean=round(float(np.mean(frac)), 3),
                        cpu_estimate_touching_tiles=CPU_ESTIMATE)))


if __name__ == "__main__":
  main()
