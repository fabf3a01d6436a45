# coding=utf-8
"""Single-future evaluation on the device: what code/pred_utils.py's `evaluate` (:354-586) and SimAug's (its :403-640)
return, from many of the scripts' batches per forward.

code/test.py (TESTING.md's first table, every number of SimAug's TESTING.md) and the validation code/train.py runs every
--save_period steps call pred_utils.evaluate: one `sess.run` per --batch_size rows (12-20 in the published commands),
the dense class logits [N,T,h,w,1] and offsets [N,T,h,w,2] of every used scale fetched to the host, and the points and
distances formed in a Python loop over rows x steps x scales.  `evaluate` here iterates the user's own
`dataset.get_batches(config.batch_size, full=True, shuffle=False)` and `model.get_feed_dict(batch)`, concatenates G
consecutive batches' feeds into one forward (multifuture.batch_feeds) and, per used scale, on the device:
  - selects the first arg-max over h*w of grid_pred_decoded (the best beam's logits under beam search, :799-803;
    torch.argmax returns the first maximum, as np.argmax does), or the ground-truth class with --use_gt_grid;
  - gathers the selected cells' fp32 offsets (ops.gather_offsets) and measures every step against the ground truth,
    point = fp64 centre + fp32 offset and error sqrt((g - p)^2) in fp64 with numpy's operation order
    (multifuture_eval.score_trajectories, K = 1), and the centre-only error.
Only the selections and the two [rows, T] error arrays come back to the host (with --save_output also the selected
offsets, the class logits and the beam outputs, which the pickle holds), where the reference's lists are rebuilt in its
order and the same np.mean runs over them: every returned value is the reference's np.float64, bit for bit.

Command line (the script's own arguments; only `evaluate` of the script's pred_utils is replaced):

  python -m multiverse_b200.single_future_eval <code/test.py | code/train.py | SimAug/code/test.py |
      SimAug/code/train.py> <its arguments> [--eval_batch_size N]

--eval_batch_size: rows per forward (default: the largest multiple of the script's --batch_size not above 256).
"""
from __future__ import annotations

import pickle
import sys

import numpy as np

from . import multifuture

DEFAULT_ROWS = 256
SCENES = ["0000", "0002", "0400", "0401", "0500"]      # the ActEV scenes of --per_scene_eval (:376)


def default_rows_per_forward(batch_size):
  """The largest multiple of the script's batch size not above DEFAULT_ROWS, and at least one batch."""
  return max(1, DEFAULT_ROWS // int(batch_size)) * int(batch_size)


def _to_host(t):
  """Every device -> host copy of this module goes through here."""
  return t.cpu().numpy()


def _user_pred_utils():
  """The script's own pred_utils (get_scene): the one the script imported."""
  mod = sys.modules.get("pred_utils")
  if mod is None:
    import pred_utils as mod       # noqa: F811  (the script's directory is on sys.path)
  return mod


def check_data(dataset, config):
  """Refuse data numpy would compute something else for: centres that are not float64 (the fp64 centre + fp32 offset
  of :491) and ground-truth trajectories that are not float32 / float64 (widened exactly to fp64 here)."""
  for j in range(len(config.scene_grids)):
    if not config.use_grids[j]:
      continue
    c = dataset.shared.get("grid_center_%d" % j)
    if c is None or np.asarray(c).dtype != np.float64:
      raise TypeError("grid_center_%d must be float64 (is %s)" % (j, None if c is None else np.asarray(c).dtype))
  pt = dataset.data["pred_traj"]
  dtypes = {np.asarray(pt).dtype} if isinstance(pt, np.ndarray) else {np.asarray(a).dtype for a in pt}
  if not dtypes <= {np.dtype(np.float32), np.dtype(np.float64)}:
    raise TypeError("pred_traj must be float32 or float64 (is %s)" % sorted(str(d) for d in dtypes))


class _Results(object):
  """The reference's accumulators (:369-404), filled one forward at a time in its order, and its reduction
  (:536-586)."""

  def __init__(self, dataset, config):
    self.config = config
    ns = len(config.scene_grids)
    self.hits = [[] for _ in range(ns)]            # bool [rows, T] per forward: grid_class_pred / _at_T
    self.err = [[] for _ in range(ns)]             # fp64 [rows, T]: l2dis_grid
    self.err_c = [[] for _ in range(ns)]           # l2dis_grid_centerOnly
    self.scene_err = [[] for _ in SCENES]
    self.out_data = None
    if config.save_output is not None:
      self.out_data = {"obs_list": [], "pred_gt_list": [], "seq_ids": []}
      for i in range(ns):
        self.out_data.update({("grid%s_class" % i): []})
        self.out_data.update({("grid%s_gt_class" % i): []})
        self.out_data.update({("grid%s_pred_traj" % i): []})
        self.out_data.update({("grid_center_%d" % i): dataset.shared["grid_center_%d" % i]})
      if config.use_beam_search:
        self.out_data.update({"beam_grid_ids": [], "beam_logprobs": []})

  def result(self):
    cfg, p = self.config, {}
    for j in range(len(cfg.scene_grids)):
      if not cfg.use_grids[j]:
        continue
      hits = np.concatenate(self.hits[j]) if self.hits[j] else np.zeros((0, cfg.pred_len), bool)
      p.update({("grid%d_acc" % j): np.mean(hits.ravel())})
      for t in range(cfg.pred_len):
        p.update({("grid%d_acc_@T=%d" % (j, t)): np.mean(np.ascontiguousarray(hits[:, t]))})
      for err, tag in ((self.err[j], "traj"), (self.err_c[j], "traj_centerOnly")):
        e = np.concatenate(err) if err else np.zeros((0, cfg.pred_len))
        p.update({("grid%d_%s_ade" % (j, tag)): np.mean(e.ravel()),
                  ("grid%d_%s_fde" % (j, tag)): np.mean(np.ascontiguousarray(e[:, -1]))})
    if cfg.per_scene_eval:
      for s, scene in enumerate(SCENES):
        rows = self.scene_err[s]
        e = np.concatenate(rows) if rows else None
        p.update({("%s_ade" % scene): np.mean(e.ravel()) if e is not None and e.size else 0.0,
                  ("%s_fde" % scene): np.mean(np.ascontiguousarray(e[:, -1])) if e is not None and len(e) else 0.0})
    if self.out_data is not None:
      with open(cfg.save_output, "wb") as f:
        pickle.dump(self.out_data, f)
      print("saved output at %s." % cfg.save_output)
    return p


def _forward(model, feed):
  """One engine forward of a concatenated feed, eager or graph-replayed by the model's own rule (_launch_bound)."""
  eng = model._ensure_engine()
  feeds = model._device_feeds(feed)
  if model._launch_bound(feeds):
    return eng.forward_graph(feeds, pred_len=model.config.pred_len)
  return eng.forward(feeds, pred_len=model.config.pred_len)


def _score_group(model, config, group, res, centers_dev, get_scene):
  """Decodes the batches `group` ([(batch, feed dict)]) in one forward and adds their rows to `res`."""
  import torch
  from . import multifuture_eval, ops
  cfg, tp = config, config.pred_len
  eng = model._ensure_engine()
  dev = eng.device
  feed, _ = multifuture.batch_feeds(model, [fd for _, fd in group])
  # the rows each batch contributes: the first original_batch_size (the padding repeats the last row), and with
  # SimAug's --only_scene those of that scene (its :502-506)
  only = getattr(cfg, "only_scene", None)
  keep, base = [], 0
  for batch, fd in group:
    n_fed = np.asarray(fd[model.obs_scene]).shape[0]
    if "traj_key" not in batch.data and "seq_key" in batch.data:
      batch.data["traj_key"] = batch.data["seq_key"]       # SimAug's :474-475
    rows = [i for i in range(batch.data["original_batch_size"])
            if only is None or get_scene(batch.data["traj_key"][i]) == only]
    keep.append((batch, base, rows))
    base += n_fed
  n = base
  gt = np.zeros((n, tp, 2))
  for batch, b0, _ in keep:
    for i, a in enumerate(batch.data["pred_traj"]):
      gt[b0 + i] = np.asarray(a)[:tp]
  with torch.cuda.device(dev):
    out = _forward(model, feed)
    lengths = torch.full((n,), tp, dtype=torch.int32, device=dev)
    gt_d = torch.from_numpy(gt).to(dev).reshape(n, 1, tp, 2)
    gt_len = torch.full((n, 1), tp, dtype=torch.int32, device=dev)
    beam = None
    if cfg.use_beam_search and res.out_data is not None:
      beam = (_to_host(out["beam_outputs"][1]), _to_host(out["beam_outputs"][2]))
    for j, (h, w) in enumerate(cfg.scene_grids):
      if not cfg.use_grids[j]:
        continue
      v = h * w
      logits = out["grid_pred_decoded"][j].reshape(n, tp, v)
      if cfg.use_gt_grid:
        sel = np.zeros((n, tp), np.int64)
        for batch, b0, _ in keep:
          for i, a in enumerate(batch.data["pred_grid_class"]):
            sel[b0 + i] = np.asarray(a)[j, :]
        if ((sel < -v) | (sel >= v)).any():
          raise IndexError("a ground-truth grid class is outside the %d cells of scale %d" % (v, j))
        ids = torch.from_numpy(np.where(sel < 0, sel + v, sel).astype(np.int32)).to(dev)
      else:
        ids = logits.argmax(-1).to(torch.int32)
      ids = ids.unsqueeze(1).contiguous()
      offs = ops.gather_offsets(ids, out["_offs"][j].contiguous(), lengths)
      err = multifuture_eval.score_trajectories(ids, offs, centers_dev[j], lengths, gt_d, gt_len, False)[0]
      err_c = multifuture_eval.score_trajectories(ids, offs, centers_dev[j], lengths, gt_d, gt_len, True)[0]
      err, err_c = _to_host(err[:, 0]), _to_host(err_c[:, 0])
      if not cfg.use_gt_grid:
        sel = _to_host(ids[:, 0])
      if res.out_data is not None:
        offs_h, logits_h = _to_host(offs[:, 0]), _to_host(logits)
        centers_h = res.out_data["grid_center_%d" % j].reshape([-1, 2])
      for batch, b0, rows in keep:
        r = [b0 + i for i in rows]
        gt_cls = [batch.data["pred_grid_class"][i][j, :] for i in rows]
        res.hits[j].append(np.array([g == sel[b0 + i] for g, i in zip(gt_cls, rows)], bool).reshape(-1, tp))
        res.err[j].append(err[r])
        res.err_c[j].append(err_c[r])
        if cfg.per_scene_eval:
          for i in rows:
            res.scene_err[SCENES.index(get_scene(batch.data["traj_key"][i]))].append(err[b0 + i][None])
        if res.out_data is None:
          continue
        od = res.out_data
        for i, g in zip(rows, gt_cls):
          if j == 0:                          # :521-524: a model of scale 1 alone writes none of these
            od["seq_ids"].append(batch.data["traj_key"][i])
            od["obs_list"].append(batch.data["obs_traj"][i])
            od["pred_gt_list"].append(batch.data["pred_traj"][i])
          c = sel[b0 + i]
          od["grid%s_pred_traj" % j].append(centers_h[c] + offs_h[b0 + i])
          od["grid%s_gt_class" % j].append(g)
          od["grid%s_class" % j].append(logits_h[b0 + i])
          if cfg.use_beam_search:
            od["beam_grid_ids"].append(beam[0][b0 + i])
            od["beam_logprobs"].append(beam[1][b0 + i])


def evaluate(dataset, config, sess, tester, rows_per_forward=None):
  """pred_utils.evaluate(dataset, config, sess, tester) on the device: the same dict (keys, np.float64 values, bit
  for bit) and, with config.save_output, the same pickle and message.  tester.model decodes (Multiverse's train.py
  passes its training model, SimAug's a separate inference model); `sess` is not used.  rows_per_forward: rows per
  forward, rounded down to whole batches of config.batch_size (default_rows_per_forward)."""
  import torch
  del sess
  model, cfg = tester.model, config
  bs = int(cfg.batch_size)
  groups = max(1, int(rows_per_forward or default_rows_per_forward(bs)) // bs)
  if cfg.per_scene_eval:
    assert sum(cfg.use_grids) == 1, "per scene eval is for one grid only"
  if cfg.use_beam_search:
    assert sum(cfg.use_grids) == 1
  check_data(dataset, cfg)
  get_scene = _user_pred_utils().get_scene if (cfg.per_scene_eval or getattr(cfg, "only_scene", None) is not None) \
      else None
  res = _Results(dataset, cfg)
  eng = model._ensure_engine()
  centers_dev = {j: torch.from_numpy(np.ascontiguousarray(dataset.shared["grid_center_%d" % j]).reshape(-1, 2))
                 .to(eng.device) for j in range(len(cfg.scene_grids)) if cfg.use_grids[j]}
  group = []
  for evalbatch in dataset.get_batches(bs, full=True, shuffle=False):
    _, batch = evalbatch
    fd = model.get_feed_dict(batch, is_train=False)
    # batches fed as trajectories and batches fed dense offsets decode in separate forwards
    if group and (len(group) == groups or (model.obs_traj in fd) != (model.obs_traj in group[0][1])):
      _score_group(model, cfg, group, res, centers_dev, get_scene)
      group = []
    group.append((batch, fd))
  if group:
    _score_group(model, cfg, group, res, centers_dev, get_scene)
  return res.result()


def install(script, rows_per_forward=None):
  """Imports the script's own pred_utils (its directory after the drop-in's on sys.path) and replaces its `evaluate`
  with the device one.  Returns the module."""
  import importlib
  import os
  multifuture.add_script_dir(script)
  here = os.path.dirname(os.path.abspath(script))
  mod = sys.modules.get("pred_utils")
  if mod is not None and os.path.dirname(os.path.abspath(getattr(mod, "__file__", "") or "")) != here:
    del sys.modules["pred_utils"]
  mod = importlib.import_module("pred_utils")
  if not callable(getattr(mod, "evaluate", None)):
    raise SystemExit("%s has no evaluate() to replace" % getattr(mod, "__file__", "pred_utils"))

  def device_evaluate(dataset, config, sess, tester):
    return evaluate(dataset, config, sess, tester, rows_per_forward=rows_per_forward)

  device_evaluate.__doc__ = evaluate.__doc__
  mod.evaluate = device_evaluate
  return mod


def main(argv=None):
  argv = sys.argv[1:] if argv is None else argv
  script, script_argv, rows = multifuture.split_argv(
      argv, flag="--eval_batch_size", default=None,
      usage="python -m multiverse_b200.single_future_eval <test.py | train.py> <its arguments> [--eval_batch_size N]")
  install(script, rows)
  sys.argv = [script] + list(script_argv)
  multifuture.load_script(script, name="__main__")


if __name__ == "__main__":
  main()
