# coding=utf-8
"""Multi-future evaluation on the device: what code/multifuture_eval_trajs.py (minADE / minFDE, :41-85) and
code/multifuture_eval_trajs_prob.py (NLL at T=1..5, :67-116) print, from the tensors the batched decode holds or from
the pickles those scripts read.

The per-future work runs in sm_90a kernels: ops.min_ade_fde_cells scores the selected cells (centre + offset in fp64,
as multifuture_inference.py forms the points) against every ground-truth future; ops.points_to_cells is the prob
script's xys_to_indexes; ops.beam_nll_ragged weighs the beam mixture at steps 0..4 of every row.  Only [N,G]-sized
results come back to the host, where the final np.mean runs over them concatenated in the scripts' order (the
predictions' order, then `for future_id in gt`), so that the printed numbers are the scripts' own.

Command lines (the scripts' arguments):

  python -m multiverse_b200.multifuture_eval trajs <gt_path> <prediction_file>
  python -m multiverse_b200.multifuture_eval prob <gt_path> <prediction_file> [--scene_h --scene_w --video_h --video_w]
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys

import numpy as np

TIME_LIST = (0, 1, 2, 3, 4)       # the prob script's evaluated steps
KEYS = ["45-degree", "top-down", "all"]
CHUNK = 256                       # trajectories per device pass from a pickle


def is_top_down(traj_id):
  """The trajs script's camera split: cam4 is the top-down view."""
  return traj_id.split("_")[-1] == "cam4"


def pack_gt(gts):
  """(gt fp64 [N,G,Tg,2], gt_len int32 [N,G]) of N ground-truth dicts (future id -> {"x_agent_traj": [[frame, person,
  x, y], ...]}), the futures of each in the dict's order, zero-padded."""
  g = max([1] + [len(d) for d in gts])
  tg = max([1] + [len(f["x_agent_traj"]) for d in gts for f in d.values()])
  gt = np.zeros((len(gts), g, tg, 2))
  gt_len = np.zeros((len(gts), g), np.int32)
  for n, d in enumerate(gts):
    for j, fid in enumerate(d):
      traj = d[fid]["x_agent_traj"]
      gt_len[n, j] = len(traj)
      if len(traj):
        gt[n, j, :len(traj)] = np.array([one[2:] for one in traj], dtype=np.float64)
  return gt, gt_len


def score_trajectories(ids, offs, centers, lengths, gt, gt_len, center_only=False):
  """minADE / minFDE of every (trajectory, ground-truth future) on the device.  ids int32 [N,K,T] (beam_outputs[1],
  or the greedy arg-max as K = 1), offs fp32 [N,K,T,2] (ops.gather_offsets), centers fp64 [V,2], lengths int32 [N]
  (the rows' prediction lengths), gt fp64 [N,G,Tg,2], gt_len int32 [N,G]: all CUDA tensors.  Returns (ade_err fp64
  [N,G,Tg] of the min-ADE prediction, ade_idx, fde fp64 [N,G], fde_idx) on the device.  Raises AssertionError, as the
  script does, for a future longer than its trajectory's predictions."""
  from . import ops
  ade_err, ade_idx, fde, fde_idx, err = ops.min_ade_fde_cells(ids, offs, centers, lengths, gt, gt_len, center_only)
  e = int(err.item())
  if e & 1:
    raise AssertionError("a ground-truth future is longer than its trajectory's predictions")
  if e & 2:
    raise ValueError("a selected cell id is outside the %d grid centres" % centers.shape[0])
  return ade_err, ade_idx, fde, fde_idx


def score_nll(logits, logprobs, lengths, gt, gt_len, scene_h, scene_w, video_h=1080, video_w=1920):
  """The prob script's per-trajectory NLL at T=1..5 on the device.  logits fp32 [N,K,Tmax,V], logprobs fp32 [N,K]
  (beam_outputs[0], [2] of a ragged decode), lengths int32 [N], gt / gt_len as score_trajectories; the grid is
  scene_h x scene_w cells over a video_h x video_w frame.  Returns (nll fp64 [N,5], count int32 [N,5]) on the device;
  count 0 where no future reaches the step (the script skips it).  Raises AssertionError if V is not the grid's size
  and IndexError for a row shorter than 5 steps or a point off the grid, as the script does."""
  import torch
  from . import ops
  n, _, _, v = logits.shape
  if v != scene_h * scene_w:
    raise AssertionError("beam logits have %d classes, the %dx%d grid has %d" % (v, scene_h, scene_w,
                                                                                 scene_h * scene_w))
  j = len(TIME_LIST)
  if int(lengths.min()) < j:
    raise IndexError("a trajectory is decoded to %d steps; the NLL reads steps 0..%d" % (int(lengths.min()), j - 1))
  if gt.shape[2] < j:
    gt = torch.nn.functional.pad(gt, (0, 0, 0, j - gt.shape[2]))
  steps = torch.tensor(TIME_LIST, dtype=torch.int32, device=logits.device)
  present = steps[None, :, None] < gt_len[:, None, :]                     # [N,J,G]
  pts = torch.where(present[..., None], gt[:, :, :j].transpose(1, 2), 0.0).contiguous()
  cells, err = ops.points_to_cells(pts, scene_h, scene_w, video_h, video_w)
  gt_idx = torch.where(present, cells, -1).to(torch.int32).contiguous()
  nll, cnt = ops.beam_nll_ragged(logits, logprobs, lengths, gt_idx, steps)
  if int(err.item()):
    raise IndexError("a ground-truth point lies off the %dx%d grid" % (scene_h, scene_w))
  return nll, cnt


class Scores(object):
  """Per-future device results gathered on the host in the scripts' order, and the lines the scripts print."""

  def __init__(self):
    self.ade = {k: [] for k in KEYS}
    self.fde = {k: [] for k in KEYS}
    self.nll = {"T=%d" % (t + 1): [] for t in TIME_LIST}

  def add_trajectories(self, traj_ids, ade_err, fde, gt_len):
    """ade_err [N,G,Tg], fde [N,G] (host or device), gt_len int32 [N,G] numpy of the trajectories traj_ids."""
    ade_err, fde = _host(ade_err), _host(fde)
    top = np.array([is_top_down(t) for t in traj_ids], bool)
    step = np.arange(ade_err.shape[2]) < gt_len[..., None]
    present = gt_len > 0
    for k, rows in (("45-degree", ~top), ("top-down", top), ("all", np.ones_like(top))):
      self.ade[k].append(ade_err[rows][step[rows]])
      self.fde[k].append(fde[rows][present[rows]])

  def add_nll(self, nll, count):
    nll, count = _host(nll), _host(count)
    for j, t in enumerate(TIME_LIST):
      self.nll["T=%d" % (t + 1)].append(nll[count[:, j] > 0, j])

  def trajectory_lines(self):
    mean = lambda parts: "%s" % np.mean(np.concatenate(parts) if parts else np.zeros(0))
    return ["ADE/FDE:", " ".join(KEYS + KEYS),
            " ".join([mean(self.ade[k]) for k in KEYS] + [mean(self.fde[k]) for k in KEYS])]

  def nll_lines(self):
    vals = {k: np.concatenate(p) if p else np.zeros(0) for k, p in self.nll.items()}
    keys = sorted(vals)
    return ["%s" % [len(vals[k]) for k in vals], "NLL:", " ".join(keys), " ".join(["%s" % np.mean(vals[k])
                                                                                 for k in keys])]


def _host(t):
  return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


class Evaluation(object):
  """Scores batches of the decode as multifuture.infer produces them (evaluation=...), against the ground truth the
  inference script loaded (gt_trajs: traj id -> future dict).  `grid` (h, w) and `video` (h, w) are the NLL's grid
  and frame; with_nll needs the beam's logits (not the greedy decode)."""

  def __init__(self, gt_trajs, centers, center_only, grid, video, with_nll):
    self.gt_trajs, self.center_only, self.grid, self.video, self.with_nll = gt_trajs, center_only, grid, video, with_nll
    self.centers = np.ascontiguousarray(centers, dtype=np.float64).reshape(-1, 2)
    self._centers_dev = None
    self.scores = Scores()

  def add(self, traj_ids, ids, offs, lengths, logits=None, logprobs=None):
    """One batch of rows traj_ids: ids int32 [N,K,T], offs fp32 [N,K,T,2], lengths int32 [N] (device), and with
    with_nll the beam logits [N,K,T,V] and log-probabilities [N,K] - all on the device, none copied to the host."""
    import torch
    dev = ids.device
    if self._centers_dev is None:
      self._centers_dev = torch.from_numpy(self.centers).to(dev)
    gt_h, gt_len_h = pack_gt([self.gt_trajs[t] for t in traj_ids])
    gt, gt_len = torch.from_numpy(gt_h).to(dev), torch.from_numpy(gt_len_h).to(dev)
    _refuse_empty_futures(traj_ids, gt_len_h, self.gt_trajs)
    ade_err, _, fde, _ = score_trajectories(ids, offs, self._centers_dev, lengths, gt, gt_len, self.center_only)
    self.scores.add_trajectories(traj_ids, ade_err, fde, gt_len_h)
    if self.with_nll:
      nll, cnt = score_nll(logits, logprobs, lengths, gt, gt_len, self.grid[0], self.grid[1], self.video[0],
                           self.video[1])
      self.scores.add_nll(nll, cnt)

  def lines(self):
    return self.scores.trajectory_lines() + (self.scores.nll_lines() if self.with_nll else [])


def _refuse_empty_futures(traj_ids, gt_len, gt_dicts):
  """The trajs script cannot score a future without points (numpy fails on its empty difference)."""
  for n, tid in enumerate(traj_ids):
    if (gt_len[n, :len(gt_dicts[tid])] == 0).any():
      raise ValueError("trajectory %s has a ground-truth future without points" % tid)


def load_gt(gt_path, traj_ids):
  out = {}
  for tid in traj_ids:
    with open(os.path.join(gt_path, "%s.p" % tid), "rb") as f:
      out[tid] = pickle.load(f)
  return out


def eval_trajs(gt_path, prediction, device=None):
  """The trajs script's printed lines for its prediction dict (traj id -> K trajectories of points)."""
  import torch
  dev = torch.device(device or "cuda")
  traj_ids = list(prediction)
  gts = load_gt(gt_path, traj_ids)
  scores = Scores()
  for c0 in range(0, len(traj_ids), CHUNK):
    rows = traj_ids[c0:c0 + CHUNK]
    k = len(prediction[rows[0]])
    if any(len(prediction[t]) != k for t in rows):
      raise ValueError("every trajectory needs the same number of predictions")
    lengths = np.array([min(len(p) for p in prediction[t]) for t in rows], np.int32)
    # the pickled points themselves are the centres, each selected once, offset-free (center_only)
    table = np.zeros((len(rows), k, int(lengths.max()), 2))
    for n, t in enumerate(rows):
      for j, p in enumerate(prediction[t]):
        table[n, j, :lengths[n]] = np.asarray(p[:lengths[n]], dtype=np.float64).reshape(-1, 2)
    ids = torch.arange(table.size // 2, dtype=torch.int32, device=dev).reshape(table.shape[:3])
    gt_h, gt_len_h = pack_gt([gts[t] for t in rows])
    _refuse_empty_futures(rows, gt_len_h, gts)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ade_err, _, fde, _ = score_trajectories(ids, torch.zeros(table.shape, dtype=torch.float32, device=dev),
                                            up(table.reshape(-1, 2)), up(lengths), up(gt_h), up(gt_len_h),
                                            center_only=True)
    scores.add_trajectories(rows, ade_err, fde, gt_len_h)
  return scores.trajectory_lines()


def eval_prob(gt_path, predictions, scene_h=18, scene_w=32, video_h=1080, video_w=1920, device=None):
  """The prob script's printed lines for its dict (traj id -> (beam logits [1,K,T,V], log-probabilities [1,K]))."""
  import torch
  dev = torch.device(device or "cuda")
  traj_ids = list(predictions)
  gts = load_gt(gt_path, traj_ids)
  scores = Scores()
  for c0 in range(0, len(traj_ids), CHUNK):
    rows = traj_ids[c0:c0 + CHUNK]
    beams = [np.asarray(predictions[t][0], dtype=np.float32) for t in rows]
    k, v = beams[0].shape[1], beams[0].shape[3]
    if any(b.shape[1] != k or b.shape[3] != v for b in beams):
      raise ValueError("every trajectory needs the same beam size and grid")
    lengths = np.array([b.shape[2] for b in beams], np.int32)
    logits = np.zeros((len(rows), k, int(lengths.max()), v), np.float32)
    for n, b in enumerate(beams):
      logits[n, :, :lengths[n]] = b[0]
    logprobs = np.stack([np.asarray(predictions[t][1], dtype=np.float32).reshape(k) for t in rows])
    gt_h, gt_len_h = pack_gt([gts[t] for t in rows])
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    nll, cnt = score_nll(up(logits), up(logprobs), up(lengths), up(gt_h), up(gt_len_h), scene_h, scene_w, video_h,
                         video_w)
    scores.add_nll(nll, cnt)
  return scores.nll_lines()


def main(argv=None):
  p = argparse.ArgumentParser(prog="python -m multiverse_b200.multifuture_eval")
  sub = p.add_subparsers(dest="cmd", required=True)
  t = sub.add_parser("trajs", help="minADE / minFDE (code/multifuture_eval_trajs.py)")
  t.add_argument("gt_path")
  t.add_argument("prediction_file")
  q = sub.add_parser("prob", help="NLL at T=1..5 (code/multifuture_eval_trajs_prob.py)")
  q.add_argument("gt_path")
  q.add_argument("prediction_file")
  q.add_argument("--scene_h", type=int, default=18)
  q.add_argument("--scene_w", type=int, default=32)
  q.add_argument("--video_h", type=int, default=1080)
  q.add_argument("--video_w", type=int, default=1920)
  args = p.parse_args(sys.argv[1:] if argv is None else argv)
  with open(args.prediction_file, "rb") as f:
    prediction = pickle.load(f)
  if args.cmd == "trajs":
    lines = eval_trajs(args.gt_path, prediction)
  else:
    lines = eval_prob(args.gt_path, prediction, args.scene_h, args.scene_w, args.video_h, args.video_w)
  for line in lines:
    print(line)


if __name__ == "__main__":
  main()
