# coding=utf-8
"""NumPy restatements of the two multi-future evaluation scripts, from their pickles to the lines they print:
code/multifuture_eval_trajs.py (minADE / minFDE over the 45-degree and top-down cameras) and
code/multifuture_eval_trajs_prob.py (NLL of the ground-truth cells under the beam mixture at T=1..5), plus the
synthetic set of tests/golden/multifuture_eval.npz as those pickles.  tests/test_multifuture_eval_cpu.py checks both
restatements against the scripts' own stdout stored there."""
import os
import pickle

import numpy as np

KEYS = ["45-degree", "top-down", "all"]


def golden_logits(d):
  """Beam logits fp32 [N,K,Tmax,V] of the golden set: scale * pattern, one fp32 product per element."""
  return d["logit_scale"][..., None] * d["logit_patterns"][d["logit_pick"].astype(np.int64)]


def gt_dict(points, length, seed):
  """One trajectory's ground truth as the Forking Paths pickles hold it: future id -> {"x_agent_traj": [[frame,
  person, x, y], ...]}, ids in a non-sorted order, integral coordinates as Python ints, the rest as floats."""
  out = {}
  for g, ln in enumerate(length):
    if ln == 0:
      continue
    rows = []
    for t in range(int(ln)):
      x, y = (float(v) for v in points[g, t])
      rows.append([100 + 12 * t, seed, int(x) if x.is_integer() and g % 2 else x, int(y) if y.is_integer() else y])
    out["%d_%d" % (seed, (7 * g + 3) % 31)] = {"x_agent_traj": rows}
  return out


def golden_pickles(d, root):
  """Writes the golden set as the scripts read it: <root>/gt/<traj id>.p, the prediction pickle (output_data of
  multifuture_inference.py: traj id -> K lists of fp64 points) and the probability pickle (--save_prob_file: traj id
  -> (logits [1,K,T,V], log-probabilities [1,K])).  Returns (gt dir, prediction file, probability file)."""
  gt_dir = os.path.join(root, "gt")
  os.makedirs(gt_dir, exist_ok=True)
  logits = golden_logits(d)
  pred, prob = {}, {}
  for n, tid in enumerate(d["traj_ids"]):
    tid, ln = str(tid), int(d["lengths"][n])
    with open(os.path.join(gt_dir, tid + ".p"), "wb") as f:
      pickle.dump(gt_dict(d["gt"][n], d["gt_len"][n], n), f)
    pred[tid] = [[d["points"][n, k, t] for t in range(ln)] for k in range(d["points"].shape[1])]
    prob[tid] = (np.ascontiguousarray(logits[n:n + 1, :, :ln]), d["logprobs"][n:n + 1].copy())
  files = os.path.join(root, "pred.p"), os.path.join(root, "prob.p")
  for path, obj in zip(files, (pred, prob)):
    with open(path, "wb") as f:
      pickle.dump(obj, f)
  return (gt_dir,) + files


def load_gts(gt_dir, traj_ids):
  out = {}
  for t in traj_ids:
    with open(os.path.join(gt_dir, "%s.p" % t), "rb") as f:
      out[t] = pickle.load(f)
  return out


def trajs_stdout(prediction, gts):
  """What multifuture_eval_trajs.py prints for its prediction dict and the ground-truth dicts."""
  ade = {k: [] for k in KEYS}
  fde = {k: [] for k in KEYS}
  for tid, preds in prediction.items():
    view = "top-down" if tid.split("_")[-1] == "cam4" else "45-degree"
    p = np.asarray(preds, dtype=np.float64)                          # [K, T, 2]
    for fut in gts[tid].values():
      g = np.asarray([row[2:] for row in fut["x_agent_traj"]], dtype=np.float64)
      sq = (g[None] - p[:, :len(g)]) ** 2
      err = np.sqrt(sq[..., 0] + sq[..., 1])                           # [K, L]
      sums = [sum(row) for row in err.tolist()]                        # Python's sum, as get_min
      last = err[:, -1].tolist()
      best = err[sums.index(min(sums))].tolist()
      for k in (view, "all"):
        ade[k] += best
        fde[k].append(last[last.index(min(last))])
  return "ADE/FDE:\n%s\n%s\n" % (" ".join(KEYS + KEYS), " ".join(
      ["%s" % np.mean(ade[k]) for k in KEYS] + ["%s" % np.mean(fde[k]) for k in KEYS]))


def cell_of(xy, scene_h, scene_w, video_h, video_w):
  """xys_to_indexes for one point: ceil(c / gap) per axis, 0 counted as 1, minus one, numpy's negative wrap."""
  out = []
  for c, gap, size in ((xy[1], video_h * 1.0 / scene_h, scene_h), (xy[0], video_w * 1.0 / scene_w, scene_w)):
    i = int(np.ceil(np.float64(c) / gap))
    i = (1 if i == 0 else i) - 1
    if not -size <= i < size:
      raise IndexError("index %d is out of bounds for axis with size %d" % (i, size))
    out.append(i % size)
  return out[0] * scene_w + out[1]


def nll_rows(prob, gts, scene_h=18, scene_w=32, video_h=1080, video_w=1920, steps=(0, 1, 2, 3, 4)):
  """{"T=t": [per-trajectory NLL]} of multifuture_eval_trajs_prob.py, trajectories in the pickle's order."""
  eps = np.finfo(float).eps
  out = {"T=%d" % (t + 1): [] for t in steps}
  for tid, (beams, logprobs) in prob.items():
    lp = np.squeeze(logprobs)
    w = np.exp(lp - lp.max())
    w = w / w.sum()
    b = np.squeeze(beams)
    e = np.exp(b - b.max(axis=-1, keepdims=True))
    b = e / e.sum(axis=-1, keepdims=True)
    for t in steps:
      grid = (b[:, t, :] * w[:, None]).sum(axis=0)                     # float32, like get_hw_prob
      cells = [cell_of(f["x_agent_traj"][t][2:], scene_h, scene_w, video_h, video_w)
               for f in gts[tid].values() if len(f["x_agent_traj"]) > t]
      if not cells:
        continue
      acc = 0.0
      for c in cells:
        acc += -np.log(grid[c] + eps)
      out["T=%d" % (t + 1)].append(acc / len(cells))
  return out


def prob_stdout(prob, gts, scene_h=18, scene_w=32, video_h=1080, video_w=1920):
  """What multifuture_eval_trajs_prob.py prints."""
  rows = nll_rows(prob, gts, scene_h, scene_w, video_h, video_w)
  keys = sorted(rows)
  return "%s\nNLL:\n%s\n%s\n" % ([len(rows[k]) for k in rows], " ".join(keys),
                                 " ".join(["%s" % np.mean(rows[k]) for k in keys]))
