# coding=utf-8
"""The synthetic set and the cases of tests/golden/single_future_eval.npz (make_golden_single_future_eval.py), and
their reconstruction from the stored arrays."""
import types

import numpy as np

R, BS, T_OBS, T_PRED, SH, SW, SC = 23, 5, 8, 12, 12, 16, 3
STRIDES = [2, 4]
GRIDS = [(6, 8), (3, 4)]
VW, VH = 1920.0, 1080.0
SCENE_VIDEOS = {"0000": "000007", "0002": "000201", "0400": "040003", "0401": "040100", "0500": "050000"}
CASES = {
    # name: (config overrides, SimAug's evaluate)
    "greedy_two_scale": (dict(use_grids=[True, True]), False),
    "beam_grids_0_1": (dict(use_grids=[False, True], use_beam_search=True, beam_size=3), False),
    "use_gt_grid": (dict(use_grids=[True, True], use_gt_grid=True), False),
    "per_scene_eval": (dict(use_grids=[True, False], per_scene_eval=True, save_output=None), False),
    "simaug_only_scene": (dict(use_grids=[True, False], per_scene_eval=True, only_scene="0400"), True),
    "tied_logits": (dict(use_grids=[True, True]), False),
}


def centers():
  out = []
  for h, w in GRIDS:
    cx = (np.arange(w) + 0.5) * (VW / w)
    cy = (np.arange(h) + 0.5) * (VH / h)
    out.append(np.stack(np.meshgrid(cx, cy), axis=-1))
  return out


def make_set(seed=5):
  rng = np.random.default_rng(seed)
  traj = np.clip(rng.uniform([200, 150], [1700, 900], (R, 1, 2)) + np.cumsum(rng.normal(0, 30, (R, T_OBS + T_PRED, 2)),
                                                                             axis=1), 1, [VW - 1, VH - 1])
  traj = traj.astype(np.float32)
  ns = len(GRIDS)
  cls = np.zeros((R, ns, T_OBS + T_PRED), np.int64)
  for j, (h, w) in enumerate(GRIDS):
    xi = np.maximum(np.ceil(traj[..., 0] / (VW / w)).astype(np.int64), 1) - 1
    yi = np.maximum(np.ceil(traj[..., 1] / (VH / h)).astype(np.int64), 1) - 1
    cls[:, j] = yi * w + xi
  cls[3, 0, T_OBS + 4] = -1                       # numpy indexing wraps it (the last cell)
  scenes = ["0000", "0002", "0400", "0401"] * 6
  scenes[7], scenes[19] = "0500", "0500"
  keys = np.array(["VIRAT_S_%s_0%d_000%03d_000%03d_%d_%d" % (SCENE_VIDEOS[scenes[i]], i % 3, i, i + 100, 10 * i, i)
                   for i in range(R)])
  frames = rng.integers(0, 9, (R, T_OBS))
  frames.sort(axis=1)
  scene_feat = np.zeros((9, SH, SW, SC), np.float32)
  np.put_along_axis(scene_feat, rng.integers(0, SC, (9, SH, SW, 1)), 1.0, axis=-1)
  out = dict(obs_traj=traj[:, :T_OBS], pred_traj=traj[:, T_OBS:], obs_grid_class=cls[..., :T_OBS],
             pred_grid_class=cls[..., T_OBS:], obs_scene=frames[..., None].astype(np.int32), keys=keys,
             scene_feat=scene_feat)
  for j, c in enumerate(centers()):
    out["grid_center_%d" % j] = c
  return out


def case_config(name, save_output):
  over, simaug = CASES[name]
  cfg = dict(batch_size=BS, obs_len=T_OBS, pred_len=T_PRED, scene_h=SH, scene_w=SW, scene_class=SC,
             scene_grid_strides=list(STRIDES), scene_grids=list(GRIDS), use_beam_search=False, beam_size=1,
             use_gt_grid=False, per_scene_eval=False, save_output=save_output)
  if simaug:
    cfg["only_scene"] = None
  cfg.update(over)
  return types.SimpleNamespace(**cfg), simaug


def case_data(s, simaug):
  """(data, shared) as pred_utils.read_data builds them: per-row arrays, traj_key a list of str (SimAug's keys in
  seq_key only)."""
  data = {k: np.asarray(s[k]) for k in ("obs_traj", "pred_traj", "obs_grid_class", "pred_grid_class", "obs_scene")}
  data["seq_key" if simaug else "traj_key"] = [str(k) for k in s["keys"]]
  shared = {"scene_feat": np.asarray(s["scene_feat"])}
  for j in range(len(GRIDS)):
    shared["grid_center_%d" % j] = np.asarray(s["grid_center_%d" % j])
  return data, shared


def case_outputs(name, cfg, n_rows, seed=7):
  """What Tester.step returns for every batch: (grid_pred_class, grid_pred_reg, beam_outputs).  Logits and offsets
  are multiples of 1/64 (the file compresses; ties occur, and the first maximum must win)."""
  rng = np.random.default_rng(seed + sorted(CASES).index(name))
  outs = []
  for _ in range(-(-n_rows // BS)):
    cls, reg, beam = [], [], None
    for j, (h, w) in enumerate(GRIDS):
      if not cfg.use_grids[j]:
        cls.append([]); reg.append([])
        continue
      if cfg.use_beam_search:
        k = cfg.beam_size
        lg = (rng.integers(-512, 512, (BS, k, T_PRED, h * w)) / 64.0).astype(np.float32)
        beam = [lg, rng.integers(0, h * w, (BS, k, T_PRED)).astype(np.int32),
                (-np.abs(rng.standard_normal((BS, k))) * 3).astype(np.float32)]
        cls.append(lg[:, 0].reshape(BS, T_PRED, h, w, 1))
      elif name == "tied_logits":
        cls.append(rng.integers(0, 3, (BS, T_PRED, h, w, 1)).astype(np.float32))
      else:
        cls.append((rng.integers(-512, 512, (BS, T_PRED, h, w, 1)) / 64.0).astype(np.float32))
      reg.append((rng.integers(-4096, 4096, (BS, T_PRED, h, w, 2)) / 64.0).astype(np.float32))
    outs.append((cls, reg, beam))
  return outs


def store_outputs(store, name, outs):
  for b, (cls, reg, beam) in enumerate(outs):
    for j in range(len(GRIDS)):
      if len(cls[j]):
        store["%s/out%d/cls%d" % (name, b, j)] = cls[j]
        store["%s/out%d/reg%d" % (name, b, j)] = reg[j]
    if beam is not None:
      for i in range(3):
        store["%s/out%d/beam%d" % (name, b, i)] = beam[i]


def load_outputs(z, name, cfg):
  outs, b = [], 0
  while any(("%s/out%d/cls%d" % (name, b, j)) in z for j in range(len(GRIDS))):
    cls = [z["%s/out%d/cls%d" % (name, b, j)] if cfg.use_grids[j] else [] for j in range(len(GRIDS))]
    reg = [z["%s/out%d/reg%d" % (name, b, j)] if cfg.use_grids[j] else [] for j in range(len(GRIDS))]
    beam = [z["%s/out%d/beam%d" % (name, b, i)] for i in range(3)] if cfg.use_beam_search else None
    outs.append((cls, reg, beam))
    b += 1
  return outs


def load_set(z):
  return {k[len("set/"):]: z[k] for k in z.files if k.startswith("set/")}
