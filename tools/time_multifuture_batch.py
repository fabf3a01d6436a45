# coding=utf-8
"""Trajectories per second of multi-future inference: code/multifuture_inference.py's per-trajectory loop (one
drop-in `sess.run` per trajectory, N=1, CUDA-graph replay as that loop runs today) against
multiverse_b200.multifuture.infer at batch 64, 256 and 512.

The set is synthetic and shaped like Forking Paths' test split as TESTING.md runs it: scene 36x64 (grid 18x32), K=20
diverse beam (gamma 0.01, fix_num_timestep 1), graph attention, scene encoding, two frames per trajectory.  The
lengths are an ASSUMPTION, not measured from the dataset: uniform over 10..26 steps (the longest ground-truth future
of a trajectory, multifuture_inference.py:229-231).  Both sides build the script's output_data without the beam
probabilities; the loop fetches the beam logits anyway (its sess.run asks for beam_outputs), infer does not.

  python tools/time_multifuture_batch.py [--n 512] [--loop_n 128] [--rounds 3] [--out results/time_multifuture.json]

Median of `rounds` alternating rounds (loop, then each batch size) of one process; the card and its power limit are
read in the same run.
"""
import argparse
import gc
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


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
  except OSError:
    return "unknown"


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--loop_n", type=int, default=128)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--batches", default="64,256,512")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  import torch
  from test_multifuture_gpu import K20, script_feeds
  import tensorflow as tf
  import pred_models
  from multiverse_b200 import multifuture, synthetic
  if not torch.cuda.is_available():
    raise SystemExit("no GPU: nothing to time")
  cfg = synthetic.make_config(batch_size=1, **K20)
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname, args.use_soft_grid_class, args.use_gt_grid = "model", False, False
  w = synthetic.make_weights(cfg, 5)

  def new_model():
    """A drop-in Model with its own engine: every batch size gets one, freed after its run (one K=20 engine at batch
    512 on 18x32 holds about 37 GB of decoder buffers)."""
    m = pred_models.get_model(args, gpuid=0)
    tf.global_variables_initializer().run()
    for v in tf.global_variables():
      if v.name.split(":")[0] in w:
        v.assign(w[v.name.split(":")[0]])
    return m

  def batched(b):
    """infer over the whole set at batch b on a fresh engine (warmed on one batch first); returns its seconds."""
    m = new_model()
    multifuture.infer(m, feeds_of(m)[:b], b, iargs, traj_ids)
    fd = feeds_of(m)
    sec = timed(lambda: multifuture.infer(m, fd, b, iargs, traj_ids))
    del m, fd
    gc.collect()
    torch.cuda.empty_cache()
    return sec

  model = new_model()
  base_feeds = script_feeds(model, cfg, a.n, 5)
  # the feed dicts are keyed by the handles of one model: re-keyed for another by name and index
  feeds_of = lambda m: [{getattr(m, h.name) if h.index is None else getattr(m, h.name)[h.index]: v
                         for h, v in fd.items()} for fd in base_feeds]
  feeds = base_feeds
  traj_ids = ["t%d" % r for r in range(a.n)]
  gi = cfg.use_grids.index(True)
  centers = synthetic.grid_centers(cfg)[gi].reshape([-1, 2])
  iargs = types.SimpleNamespace(scene_grid_centers=synthetic.grid_centers(cfg), num_out=20, center_only=False)
  sess = tf.Session()

  def loop(n):
    out = {}
    for tid, fd in zip(traj_ids[:n], feeds[:n]):
      cls, reg, (lg, ids, lp) = sess.run([model.grid_pred_decoded[gi], model.grid_pred_reg_decoded[gi],
                                          model.beam_outputs], feed_dict=fd)
      length = int(fd[model.pred_length][0])
      reg = reg.reshape([1, length, -1, 2])
      out[tid] = [[centers[ids[0, j, t]] + reg[0, t, ids[0, j, t], :] for t in range(length)] for j in range(20)]
    return out

  def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0

  batches = [int(b) for b in a.batches.split(",")]
  loop(min(8, a.loop_n))                                       # warm-up: graph capture of the lengths seen first
  loop(a.loop_n)
  rates = {"loop": []}
  rates.update({"batch%d" % b: [] for b in batches})
  for _ in range(a.rounds):
    rates["loop"].append(a.loop_n / timed(lambda: loop(a.loop_n)))
    for b in batches:
      rates["batch%d" % b].append(a.n / batched(b))
  lens = [int(fd[model.pred_length][0]) for fd in feeds]
  res = dict(card=card(), trajectories=a.n, loop_trajectories=a.loop_n, rounds=a.rounds,
             lengths="uniform 10..26 (assumed), mean %.2f" % np.mean(lens),
             median_traj_per_s={k: float(np.median(v)) for k, v in rates.items()},
             all_traj_per_s={k: [round(x, 2) for x in v] for k, v in rates.items()})
  print(json.dumps(res))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
