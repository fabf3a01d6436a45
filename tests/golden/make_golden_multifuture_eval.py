# coding=utf-8
"""Golden output of the two multi-future evaluation scripts on a synthetic set shaped like Forking Paths' test split:
code/multifuture_eval_trajs.py (minADE / minFDE) and code/multifuture_eval_trajs_prob.py (NLL), both UNMODIFIED, run
as subprocesses on pickles written here; their stdout is stored with the inputs.  The per-trajectory NLL of the prob
script's own functions (imported; they need no TensorFlow) is stored too.

The set: 48 trajectories over cameras cam1..cam4 (cam4 is the top-down split), 1-15 futures each with lengths 1..T
(T, 5..14, the trajectory's prediction length, is the longest future's), K = 20 predictions formed like
multifuture_inference.py's (fp64 centre + fp32 offset), duplicated predictions (ties), and ground-truth points on
exact cell boundaries, at 0 and slightly negative (wrapped by numpy's indexing).  The beam logits [1,20,T,576] are
stored compactly as scale * pattern (one fp32 product per element; multifuture_eval_golden_inputs rebuilds them).

  python tests/golden/make_golden_multifuture_eval.py        (needs the reference tree)"""
import importlib.util
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

REF = os.path.join(os.environ.get("MVB_REFERENCE_ROOT", "/root/reference"), "code")
OUT = os.path.dirname(os.path.abspath(__file__))
N, K, H, W, VH, VW, R = 48, 20, 18, 32, 1080, 1920, 32


def make_set(seed=11):
  rng = np.random.default_rng(seed)
  gap = np.array([VW / W, VH / H])
  centers = np.stack(np.meshgrid((np.arange(W) + 0.5) * gap[0], (np.arange(H) + 0.5) * gap[1]), -1).reshape(-1, 2)
  lengths = rng.integers(5, 15, N).astype(np.int32)
  tmax = int(lengths.max())
  ids = rng.integers(0, H * W, (N, K, tmax)).astype(np.int32)
  offs = rng.normal(0, 20, (N, K, tmax, 2)).astype(np.float32)
  dup = np.arange(0, N, 3)
  ids[dup, 9], offs[dup, 9] = ids[dup, 2], offs[dup, 2]                # prediction 9 repeats 2: the first must win
  pts = centers[ids] + offs                                           # fp64 centre + fp32 offset, one fp64 add
  for n in range(N):
    pts[n, :, lengths[n]:] = 0.0
  g_count = rng.integers(1, 16, N).astype(np.int32)
  g_count[:3] = [1, 15, 15]
  gmax = int(g_count.max())
  gt_len = np.zeros((N, gmax), np.int32)
  gt = np.zeros((N, gmax, tmax, 2))
  for n in range(N):
    gl = rng.integers(1, lengths[n] + 1, g_count[n])
    gl[rng.integers(0, g_count[n])] = lengths[n]
    gt_len[n, :g_count[n]] = gl
    near = rng.integers(0, K, g_count[n])
    gt[n, :g_count[n]] = pts[n, near] + rng.normal(0, 25, (g_count[n], tmax, 2))
  gt[dup, 0, :] = pts[dup, 2] + rng.normal(0, 0.5, (len(dup), tmax, 2))   # future 0 nearest the duplicated prediction
  # cell boundaries, 0 and slightly negative points in the NLL's steps 0..4
  special = [(0.0, 0.0), (60.0, 60.0), (1920.0, 1080.0), (-0.25, 3.0), (-1e-9, -1e-9), (-61.0, 120.0),
             (420.0, -59.5), (1859.9999999999998, 540.0), (600.0, 1020.0)]
  for i, xy in enumerate(special):
    gt[i % N, i % g_count[i % N], i % 5] = xy
  gt = np.clip(gt, -100.0, [VW, VH])
  for n in range(N):
    for g in range(gmax):
      gt[n, g, gt_len[n, g]:] = 0.0
  scale = rng.uniform(0.5, 4.0, (N, K, tmax)).astype(np.float32)
  pick = rng.integers(0, R, (N, K, tmax)).astype(np.int16)
  patterns = rng.standard_normal((R, H * W)).astype(np.float32)
  logprobs = (-np.abs(rng.standard_normal((N, K))) * 4).astype(np.float32)
  cams = np.array([1 + (n * 7) % 4 for n in range(N)], np.int32)
  traj_ids = np.array(["%04d_%d_%d_cam%d" % (n, 10 + n, 3 + n, cams[n]) for n in range(N)])
  return dict(traj_ids=traj_ids, lengths=lengths, points=pts, ids=ids, offs=offs, centers=centers, gt=gt,
              gt_len=gt_len, g_count=g_count, logit_scale=scale, logit_pick=pick, logit_patterns=patterns,
              logprobs=logprobs)


def run(script, *args):
  r = subprocess.run([sys.executable, os.path.join(REF, script)] + list(args), capture_output=True, text=True,
                     check=True)
  return r.stdout


def load(name):
  spec = importlib.util.spec_from_file_location("_ref_" + name, os.path.join(REF, name + ".py"))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


def main():
  sys.path.insert(0, os.path.dirname(OUT))
  from multifuture_eval_ref import golden_pickles
  d = make_set()
  with tempfile.TemporaryDirectory() as tmp:
    gt_dir, pred_file, prob_file = golden_pickles(d, tmp)
    out_trajs = run("multifuture_eval_trajs.py", gt_dir, pred_file)
    out_prob = run("multifuture_eval_trajs_prob.py", gt_dir, prob_file)
    with open(prob_file, "rb") as f:
      prob = pickle.load(f)
    gts = {}
    for t in prob:
      with open(os.path.join(gt_dir, "%s.p" % t), "rb") as f:
        gts[t] = pickle.load(f)
  # per-trajectory NLL of the script's own functions (its loop body, :82-109)
  evp = load("multifuture_eval_trajs_prob")
  a = type("A", (), dict(scene_h=H, scene_w=W, video_h=VH, video_w=VW, w_gap=VW * 1.0 / W, h_gap=VH * 1.0 / H))
  nll = np.zeros((N, 5))
  cnt = np.zeros((N, 5), np.int32)
  for n, t in enumerate(d["traj_ids"]):
    beams, lp = prob[t]
    lp = evp.softmax(np.squeeze(lp))
    beams = evp.softmax(np.squeeze(beams), axis=-1)
    for j in range(5):
      xys = [gts[t][f]["x_agent_traj"][j][2:] for f in gts[t] if len(gts[t][f]["x_agent_traj"]) > j]
      if xys:
        nll[n, j] = evp.compute_nll(evp.get_hw_prob(beams, lp, j), evp.xys_to_indexes(np.asarray(xys), a))
        cnt[n, j] = len(xys)
  np.savez_compressed(os.path.join(OUT, "multifuture_eval.npz"), stdout_trajs=np.array(out_trajs),
                      stdout_prob=np.array(out_prob), nll=nll, count=cnt, **d)
  print(out_trajs + out_prob)


if __name__ == "__main__":
  main()
