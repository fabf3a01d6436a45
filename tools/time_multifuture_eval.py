# coding=utf-8
"""Seconds to decode and score a synthetic Forking-Paths-shaped set, two ways:
  pickles: multifuture.infer with the beam probabilities, output_data and beam_prob pickled to a temporary directory,
           then read back and scored by the NumPy restatements of code/multifuture_eval_trajs.py and
           code/multifuture_eval_trajs_prob.py (tests/multifuture_eval_ref.py: the scripts' own numpy operations, in
           one process instead of two interpreters);
  --eval:  multifuture.infer with a multifuture_eval.Evaluation: scored on the device, logits never leave it.

The set: scene 36x64 (grid 18x32), K=20 diverse beam (gamma 0.01), graph attention, prediction lengths ASSUMED
uniform over 10..26, 1-15 ground-truth futures per trajectory.  Median of `rounds` alternating rounds; the card and its
power limit are read in the same run.

  python tools/time_multifuture_eval.py [--n 512] [--batch 256] [--rounds 3] [--out results/time_mf_eval.json]
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
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
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit("no GPU: nothing to time")
  from test_multifuture_gpu import K20, script_feeds
  from test_multifuture_eval_gpu import synthetic_gt
  import multifuture_eval_ref as ref
  import tensorflow as tf
  import pred_models
  from multiverse_b200 import multifuture, synthetic
  cfg = synthetic.make_config(batch_size=1, **K20)
  margs = types.SimpleNamespace(**vars(cfg))
  margs.modelname, margs.use_soft_grid_class, margs.use_gt_grid = "model", False, False
  w = synthetic.make_weights(cfg, 5)
  model = pred_models.get_model(margs, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  feeds = script_feeds(model, cfg, a.n, 5)
  traj_ids = ["%04d_%d_%d_cam%d" % (r, r + 3, r + 7, 1 + r % 4) for r in range(a.n)]
  gts = dict(zip(traj_ids, synthetic_gt([int(fd[model.pred_length][0]) for fd in feeds], 6)))
  args = types.SimpleNamespace(scene_grid_centers=synthetic.grid_centers(cfg), num_out=20, center_only=False,
                               video_h=1080, video_w=1920)
  gi = cfg.use_grids.index(True)
  h, w_ = cfg.scene_grids[gi]

  def pickles():
    out, prob = multifuture.infer(model, feeds, a.batch, args, traj_ids, with_prob=True)
    with tempfile.TemporaryDirectory() as tmp:
      for name, obj in (("out.p", out), ("prob.p", prob)):
        with open(os.path.join(tmp, name), "wb") as f:
          pickle.dump(obj, f)
      with open(os.path.join(tmp, "out.p"), "rb") as f:
        out = pickle.load(f)
      with open(os.path.join(tmp, "prob.p"), "rb") as f:
        prob = pickle.load(f)
    return ref.trajs_stdout(out, gts) + ref.prob_stdout(prob, gts, h, w_)

  def device():
    ev = multifuture.make_evaluation(model, args, gts)
    multifuture.infer(model, feeds, a.batch, args, traj_ids, evaluation=ev)
    return "\n".join(ev.lines()) + "\n"

  def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r

  _, text_p = timed(pickles)                    # warm-up of both, and their printed lines
  _, text_d = timed(device)
  secs = {"pickles": [], "eval": []}
  for _ in range(a.rounds):
    secs["pickles"].append(timed(pickles)[0])
    secs["eval"].append(timed(device)[0])
  res = dict(card=card(), trajectories=a.n, batch=a.batch, rounds=a.rounds,
             lengths="uniform 10..26 (assumed)", median_s={k: float(np.median(v)) for k, v in secs.items()},
             all_s={k: [round(x, 3) for x in v] for k, v in secs.items()},
             ade_fde_lines_equal=text_p.splitlines()[:3] == text_d.splitlines()[:3],
             pickle_path=text_p.splitlines(), eval_path=text_d.splitlines())
  print(json.dumps(res))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
