# coding=utf-8
"""NumPy restatement of the single-future evaluation: code/pred_utils.py's `evaluate` (:354-586; `simaug=True`: SimAug's,
which falls back from traj_key to seq_key and skips rows outside config.only_scene) and `Dataset.get_batches(full=True,
shuffle=False)` (:589-706).  tests/golden/single_future_eval.npz holds what the reference functions themselves return on
a synthetic set; the tests check this restatement against it on the CPU, and use it as the host truth on the GPU, where
there is no reference tree."""
import collections
import math
import pickle

import numpy as np

SCENES = ["0000", "0002", "0400", "0401", "0500"]


def get_scene(videoname_):
  """code/pred_utils.py:303-307."""
  s = videoname_.split("_S_")[-1]
  s = s.split("_")[0]
  return s[:4]


class Dataset(object):
  """code/pred_utils.py:589-706 without shuffling (the evaluation's batches)."""

  def __init__(self, data, data_type, config=None, shared=None):
    self.data, self.data_type, self.config, self.shared = data, data_type, config, shared
    self.valid_idxs = range(len(self.data["obs_traj"]))
    self.num_examples = len(self.valid_idxs)

  def get_by_idxs(self, idxs):
    out = collections.defaultdict(list)
    for key, val in self.data.items():
      out[key].extend(val[idx] for idx in idxs)
    return out

  def get_batches(self, batch_size, full=True, shuffle=False):
    assert full and not shuffle
    cfg = self.config
    for b in range(int(math.ceil(self.num_examples / float(batch_size)))):
      idxs = list(self.valid_idxs[b * batch_size:(b + 1) * batch_size])
      original = len(idxs)
      idxs += [idxs[-1]] * (batch_size - original)
      data = self.get_by_idxs(idxs)
      data.update({"original_batch_size": original})
      old2new = {}
      obs_scene = np.zeros((cfg.batch_size, cfg.obs_len, 1), dtype="int32")
      for i in range(len(data["obs_scene"])):
        for j in range(len(data["obs_scene"][i])):
          oldid = data["obs_scene"][i][j][0]
          if oldid not in old2new:
            old2new[oldid] = len(old2new)
          obs_scene[i, j, 0] = old2new[oldid]
      scene_feat = np.zeros((len(old2new), cfg.scene_h, cfg.scene_w, cfg.scene_class), dtype="float32")
      for oldid, newid in old2new.items():
        scene_feat[newid] = self.shared["scene_feat"][oldid]
      data.update({"batch_obs_scene": obs_scene, "batch_scene_feat": scene_feat})
      yield tuple(idxs), Dataset(data, self.data_type, shared=self.shared)


def evaluate(dataset, config, step, simaug=False):
  """pred_utils.evaluate with `step(batch) -> (grid_pred_class, grid_pred_reg, beam_outputs)` in place of
  tester.step(sess, (idxs, batch)).  Returns (p, out_data or None); out_data is pickled to config.save_output."""
  pred_len, ns = config.pred_len, len(config.scene_grids)
  only = getattr(config, "only_scene", None) if simaug else None
  p = {}
  if config.per_scene_eval:
    assert sum(config.use_grids) == 1
    l2dis_scenes = [[] for _ in SCENES]
  out_data = None
  if config.save_output is not None:
    out_data = {"obs_list": [], "pred_gt_list": [], "seq_ids": []}
    for i in range(ns):
      out_data.update({("grid%s_class" % i): []})
      out_data.update({("grid%s_gt_class" % i): []})
      out_data.update({("grid%s_pred_traj" % i): []})
      out_data.update({("grid_center_%d" % i): dataset.shared["grid_center_%d" % i]})
    if config.use_beam_search:
      out_data.update({"beam_grid_ids": [], "beam_logprobs": []})
  l2dis_grid = [[] for _ in range(ns)]
  l2dis_grid_c = [[] for _ in range(ns)]
  grid_class_pred = [[] for _ in range(ns)]
  grid_class_pred_at_T = [[[] for _ in range(pred_len)] for _ in range(ns)]
  for _, batch in dataset.get_batches(config.batch_size, full=True, shuffle=False):
    grid_pred_class, grid_pred_reg, beam_outputs = step(batch)
    N = batch.data["original_batch_size"]
    if config.use_beam_search:
      assert sum(config.use_grids) == 1
      _, beam_grid_ids, beam_logprobs = beam_outputs
    if simaug and "traj_key" not in batch.data:
      batch.data["traj_key"] = batch.data["seq_key"]
    for j, (H, W) in enumerate(config.scene_grids):
      if not config.use_grids[j]:
        continue
      grid_traj_d, grid_c_traj_d = [], []
      grid_class = grid_pred_class[j][:N].reshape([N, pred_len, H * W])
      sel = np.argmax(grid_class, axis=2)
      if config.use_gt_grid:
        sel = np.array([batch.data["pred_grid_class"][i][j, :] for i in range(N)])
      grid_reg = grid_pred_reg[j][:N].reshape([N, pred_len, H * W, 2])
      center_coors = batch.shared["grid_center_%s" % j].reshape([-1, 2])
      for i in range(N):
        if only is not None and get_scene(batch.data["traj_key"][i]) != only:
          continue
        gt_cls = batch.data["pred_grid_class"][i][j, :]
        grid_class_pred[j].extend(gt_cls == sel[i, :])
        grid_traj, grid_traj_c = [], []
        for t in range(pred_len):
          grid_class_pred_at_T[j][t].append(gt_cls[t] == sel[i, t])
          c = center_coors[sel[i, t]]
          grid_traj.append(c + grid_reg[i, t, sel[i, t], :])
          grid_traj_c.append(c)
        grid_traj = np.array(grid_traj)
        gt_traj = batch.data["pred_traj"][i]
        diff = np.sqrt(np.sum((gt_traj - grid_traj) ** 2, axis=1))
        grid_traj_d.append(diff)
        grid_c_traj_d.append(np.sqrt(np.sum((gt_traj - np.array(grid_traj_c)) ** 2, axis=1)))
        if config.per_scene_eval:
          l2dis_scenes[SCENES.index(get_scene(batch.data["traj_key"][i]))].append(diff)
        if out_data is not None:
          if j == 0:
            out_data["seq_ids"].append(batch.data["traj_key"][i])
            out_data["obs_list"].append(batch.data["obs_traj"][i])
            out_data["pred_gt_list"].append(batch.data["pred_traj"][i])
          out_data["grid%s_pred_traj" % j].append(grid_traj)
          out_data["grid%s_gt_class" % j].append(gt_cls)
          out_data["grid%s_class" % j].append(grid_class[i])
          if config.use_beam_search:
            out_data["beam_grid_ids"].append(beam_grid_ids[i])
            out_data["beam_logprobs"].append(beam_logprobs[i])
      l2dis_grid[j] += grid_traj_d
      l2dis_grid_c[j] += grid_c_traj_d
  for j in range(ns):
    if not config.use_grids[j]:
      continue
    p.update({("grid%d_acc" % j): np.mean(grid_class_pred[j])})
    for t in range(pred_len):
      p.update({("grid%d_acc_@T=%d" % (j, t)): np.mean(grid_class_pred_at_T[j][t])})
    for lst, tag in ((l2dis_grid[j], "traj"), (l2dis_grid_c[j], "traj_centerOnly")):
      p.update({("grid%d_%s_ade" % (j, tag)): np.mean([t for o in lst for t in o]),
                ("grid%d_%s_fde" % (j, tag)): np.mean([o[-1] for o in lst])})
  if config.per_scene_eval:
    for s, scene in enumerate(SCENES):
      ade = [t for o in l2dis_scenes[s] for t in o]
      fde = [o[-1] for o in l2dis_scenes[s]]
      p.update({("%s_ade" % scene): np.mean(ade) if ade else 0.0, ("%s_fde" % scene): np.mean(fde) if fde else 0.0})
  if out_data is not None:
    with open(config.save_output, "wb") as f:
      pickle.dump(out_data, f)
  return p, out_data


def synthetic_dataset(args, n, seed, frames=None):
  """A Dataset of n synthetic trajectories as read_data builds it (multiverse_b200.synthetic: random walks over a
  1920x1080 frame, dense targets from the float64 trajectories, pred_traj stored as float32), ActEV-style traj_key over
  the five scenes (0500 only for the last three rows).  frames: scene frames shared round-robin (default one per
  trajectory)."""
  from multiverse_b200 import synthetic
  f = synthetic.make_feeds(args, n, seed, with_pred=True)
  t, ns = args.obs_len, len(args.scene_grids)
  videos = {"0000": "000007", "0002": "000201", "0400": "040003", "0401": "040100", "0500": "050000"}
  obs_scene = f["obs_scene"] if frames is None else f["obs_scene"] % frames
  data = dict(obs_traj=f["traj64"][:, :t], pred_traj=f["traj"][:, t:], obs_scene=obs_scene[:, :, None].astype(np.int32),
              obs_grid_class=np.stack([np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(n)]),
              pred_grid_class=np.stack([np.stack([f["grid_pred_labels"][j][i] for j in range(ns)]) for i in range(n)]),
              traj_key=["VIRAT_S_%s_01_000%03d_000%03d_%d_%d" % (videos[SCENES[i % 4 if i < n - 3 else 4]], i % 1000,
                                                                 i % 1000 + 50, i, i) for i in range(n)])
  for j in range(ns):
    data["obs_grid_target_all_%d" % j] = f["grid_obs_regress"][j]
    data["pred_grid_target_all_%d" % j] = f["grid_pred_regress"][j]
  shared = {"scene_feat": f["scene_feat"] if frames is None else f["scene_feat"][:frames]}
  for j, c in enumerate(synthetic.grid_centers(args)):
    shared["grid_center_%d" % j] = c
  return Dataset(data, "test", config=args, shared=shared)


def tester_step(model, sess):
  """step(batch) of the drop-in Tester (pred_models.Tester.step)."""
  import pred_models
  tester = pred_models.Tester(model, model.config)
  return lambda batch: tester.step(sess, ((), batch))


def same_value(a, b):
  """Equal value and type, NaN equal to NaN (np.mean of an empty list)."""
  if type(a) is not type(b):
    return False
  if isinstance(a, float) and math.isnan(a):
    return math.isnan(b)
  return a == b


def assert_same_dict(got, want):
  assert list(got) == list(want)
  bad = [(k, got[k], want[k], type(got[k]), type(want[k])) for k in want if not same_value(got[k], want[k])]
  assert not bad, bad[:5]


def assert_same_out_data(got, want):
  """Two save_output dicts: the same keys in the same order, and every entry of the same type, dtype, shape and bytes
  (np.str_ keys compared as values)."""
  assert list(got) == list(want)
  for k in want:
    a, b = got[k], want[k]
    assert type(a) is type(b), k
    items = list(zip(a, b)) if isinstance(b, list) else [(a, b)]
    if isinstance(b, list):
      assert len(a) == len(b), (k, len(a), len(b))
    for x, y in items:
      assert type(x) is type(y), (k, type(x), type(y))
      if isinstance(y, np.ndarray):
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k
      else:
        assert x == y, k
