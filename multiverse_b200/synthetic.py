# coding=utf-8
"""Seeded synthetic weights and feeds of the reference's placeholder shapes (SURVEY.md §8d), used by
bench.py, __graft_entry__.smoke() and the drop-in demos.  No dataset or checkpoint is reachable
from this environment, so benchmarks run on these.

Feeds follow code/pred_models.py:62-115 (placeholders) and the target computation of
code/multifuture_inference.py:115-156 / code/preprocess.py:436-475: grid class = ceil(x / gap)
(0 -> 1) - 1, offsets = trajectory point - cell centre for EVERY cell (pixels of a 1920x1080
frame).  Variable names are the ones the reference creates (SURVEY.md §8a)."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np


def make_config(**kw):
  """Hyper-parameters of every published command (TRAINING.md:32-39, TESTING.md:84-93) at the
  BASELINE.json grid shape (scene 72x36 -> grids 36x18 and 18x9)."""
  cfg = dict(batch_size=4, obs_len=8, pred_len=12, scene_h=72, scene_w=36, scene_class=11,
             scene_conv_dim=64, scene_conv_kernel=3, scene_grid_strides=[2, 4],
             use_grids=[True, True], enc_hidden_size=256, dec_hidden_size=256, emb_size=32,
             convlstm_kernel=3, use_scene_enc=True, use_gnn=True, use_beam_search=False,
             beam_size=1, diverse_beam=False, diverse_gamma=1.0, fix_num_timestep=0,
             activation_func="tanh", video_h=1080, video_w=1920, keep_prob=1.0, is_train=False)
  cfg.update(kw)
  cfg = SimpleNamespace(**cfg)
  cfg.scene_grids = [(int(round(cfg.scene_h * 1.0 / s)), int(round(cfg.scene_w * 1.0 / s)))
                     for s in cfg.scene_grid_strides]          # code/pred_utils.py:127-132
  return cfg


def weight_shapes(cfg):
  k, ch, e, cs = cfg.convlstm_kernel, cfg.enc_hidden_size, cfg.emb_size, cfg.scene_conv_dim
  shp, cin = {}, cfg.scene_class
  for i in range(len(cfg.scene_grid_strides) if cfg.use_scene_enc else 0):
    shp["person_pred/scene_conv%d/W" % (i + 1)] = (3, 3, cin, cs)
    shp["person_pred/scene_conv%d/b" % (i + 1)] = (cs,)
    cin = cs
  p = "person_pred/"
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      continue
    if not cfg.use_scene_enc:
      # the class encoder's embedding of one_hot(label) (code/pred_models.py:221-225), one variable for every scale
      shp.setdefault(p + "grid_emb/W", (3, 3, 1, e))
      shp.setdefault(p + "grid_emb/b", (e,))
    shp[p + "encoder_grid_class_%d/enc_grid_%d/kernel" % (i, i)] = (k, k, (cs if cfg.use_scene_enc else e) + ch, 4 * ch)
    shp[p + "encoder_grid_class_%d/enc_grid_%d/biases" % (i, i)] = (4 * ch,)
    shp[p + "encoder_grid_reg_%d/enc_grid_regress_%d/kernel" % (i, i)] = (k, k, 2 + ch, 4 * ch)
    shp[p + "encoder_grid_reg_%d/enc_grid_regress_%d/biases" % (i, i)] = (4 * ch,)
    for kind, cell, pdim in (("class", "dec_grid_%d" % i, 1), ("reg", "dec_grid_reg_%d" % i, 2)):
      d = p + "decoder_grid_%s_%d/decoder_rnn/" % (kind, i)
      shp[d + cell + "/kernel"] = (k, k, e + ch, 4 * ch)
      shp[d + cell + "/biases"] = (4 * ch,)
      shp[d + "grid_emb/W"] = (3, 3, pdim, e)
      shp[d + "grid_emb/b"] = (e,)
      shp[p + "hidden2grid_decoder_grid_%s_%d/out_dec_grid/W" % (kind, i)] = (3, 3, ch, pdim)
  return shp


def make_weights(cfg, seed=20200614):
  """Random-init weights of the reference architecture: glorot-uniform ConvLSTM kernels (TF
  default), he-normal conv2d W (variance_scaling(2.0), code/pred_models.py:1359), small biases."""
  rng = np.random.default_rng(seed)
  out = {}
  for name, shp in weight_shapes(cfg).items():
    if name.endswith("/kernel"):
      lim = math.sqrt(6.0 / (shp[0] * shp[1] * (shp[2] + shp[3])))
      w = rng.uniform(-lim, lim, size=shp)
    elif name.endswith("/W"):
      w = np.clip(rng.standard_normal(shp), -2, 2) * math.sqrt(2.0 / (shp[0] * shp[1] * shp[2]))
      if "out_dec_grid" in name:
        w = w * 4.0
    else:
      w = rng.standard_normal(shp) * 0.05
    out[name] = w.astype(np.float32)
  return out


def grid_centers(cfg):
  out = []
  for h, w in cfg.scene_grids:
    hg, wg = cfg.video_h * 1.0 / h, cfg.video_w * 1.0 / w
    cx = (np.arange(w) + 0.5) * wg
    cy = (np.arange(h) + 0.5) * hg
    out.append(np.stack(np.meshgrid(cx, cy), axis=-1))         # [h,w,2] (x,y)
  return out


def make_feeds(cfg, n=None, seed=20200614, with_pred=False):
  """Feeds for n trajectories: one distinct segmentation frame per trajectory, smooth random
  walks, obs labels/offsets per scale.  Vectorised over the batch."""
  n = n or cfg.batch_size
  rng = np.random.default_rng(seed)
  t, tp = cfg.obs_len, cfg.pred_len
  sh, sw, sc = cfg.scene_h, cfg.scene_w, cfg.scene_class
  blocks = rng.integers(0, sc, size=(n, -(-sh // 6), -(-sw // 3)))
  seg = np.repeat(np.repeat(blocks, 6, axis=1), 3, axis=2)[:, :sh, :sw]
  scene_feat = np.zeros((n, sh, sw, sc), dtype=np.float32)
  np.put_along_axis(scene_feat, seg[..., None], 1.0, axis=-1)
  obs_scene = np.tile(np.arange(n, dtype=np.int32)[:, None], (1, t))
  start = rng.uniform([0.2 * cfg.video_w, 0.2 * cfg.video_h], [0.8 * cfg.video_w, 0.8 * cfg.video_h],
                      size=(n, 2))
  traj = np.clip(start[:, None] + np.cumsum(rng.normal(0, 25.0, size=(n, t + tp, 2)), axis=1), 1.0,
                 [cfg.video_w - 1.0, cfg.video_h - 1.0])
  feeds = dict(scene_feat=scene_feat, obs_scene=obs_scene, traj=traj.astype(np.float32), traj64=traj,
               grid_obs_labels=[], grid_obs_regress=[], grid_pred_labels=[], grid_pred_regress=[])
  for center, (h, w) in zip(grid_centers(cfg), cfg.scene_grids):
    hg, wg = cfg.video_h * 1.0 / h, cfg.video_w * 1.0 / w
    xi = np.maximum(np.ceil(traj[:, :, 0] / wg).astype(np.int64), 1) - 1
    yi = np.maximum(np.ceil(traj[:, :, 1] / hg).astype(np.int64), 1) - 1
    labels = (yi * w + xi).astype(np.int32)
    feeds["grid_obs_labels"].append(labels[:, :t])
    feeds["grid_pred_labels"].append(labels[:, t:])
    feeds["grid_obs_regress"].append(
        (traj[:, :t, None, None, :] - center[None, None]).astype(np.float32))
    if with_pred:
      feeds["grid_pred_regress"].append(
          (traj[:, t:, None, None, :] - center[None, None]).astype(np.float32))
  return feeds


def shard_feeds(feeds, rank, world):
  """Trajectory shard `rank` of `world` of a feed dict (SURVEY.md §8e): the contiguous rows
  [rank*N/world, (rank+1)*N/world) of every per-trajectory array and ONLY the scene frames those rows index,
  re-compacted and re-indexed the way the reference compacts them per batch (code/pred_utils.py:680-704).  Keys
  that are absent (grid_pred_* at inference) are skipped; lists are per-scale lists.  Used by bench.py (inference
  and training arms), tests/ddp_check.py and the gloo sharding test - one definition of "a shard"."""
  n = feeds["obs_scene"].shape[0]
  assert n % world == 0, "the global batch must divide evenly over the ranks"
  per = n // world
  sl = slice(rank * per, (rank + 1) * per)
  obs_scene = np.asarray(feeds["obs_scene"][sl])
  frames, local = np.unique(obs_scene, return_inverse=True)
  out = dict(scene_feat=feeds["scene_feat"][frames], obs_scene=local.reshape(obs_scene.shape).astype(np.int32))
  for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    if k in feeds and len(feeds[k]):
      out[k] = [a[sl] for a in feeds[k]]
  for k in ("traj", "traj64"):
    if k in feeds:
      out[k] = feeds[k][sl]
  return out


def write_npz(path, cfg, n, seed=0):
  """A data_<split>.npz in the layout code/preprocess.py writes (:670-679, :789-813, :860-864)
  and code/pred_utils.read_data (:208-300) reads, filled with synthetic trajectories."""
  f = make_feeds(cfg, n, seed, with_pred=True)
  t = cfg.obs_len
  ns = len(cfg.scene_grids)
  data = dict(
      obs_traj=f["traj64"][:, :t], pred_traj=f["traj64"][:, t:],     # float64, like the reference's preprocess output
      obs_scene=f["obs_scene"][:, :, None].astype(np.int32),
      obs_grid_class=np.stack([np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(n)]),
      pred_grid_class=np.stack([np.stack([f["grid_pred_labels"][j][i] for j in range(ns)]) for i in range(n)]),
      scene_feat=f["scene_feat"], scene_grid_strides=np.array(cfg.scene_grid_strides),
      video_wh=np.array([cfg.video_w, cfg.video_h]))
  for j, c in enumerate(grid_centers(cfg)):
    data["obs_grid_target_all_%d" % j] = f["grid_obs_regress"][j]
    data["pred_grid_target_all_%d" % j] = f["grid_pred_regress"][j]
    data["grid_center_%d" % j] = c
  np.savez(path, **data)
  return f
