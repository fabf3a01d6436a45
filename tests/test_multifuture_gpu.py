# coding=utf-8
"""GPU test of the batched multi-future driver (multiverse_b200.multifuture.infer): its pickled output_data and
beam_prob equal those of code/multifuture_inference.py's per-trajectory loop (:460-523) - one sess.run of the drop-in
Model per trajectory, fed its own N=1 feeds and its own pred_length (restated here, as the script builds them: every
trajectory's frames compacted to indices 0.., :347-376)."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

K20 = dict(scene_h=36, scene_w=64, use_grids=[True, False], use_beam_search=True, beam_size=20, diverse_beam=True,
           diverse_gamma=0.01, fix_num_timestep=1)


def make_model(monkeypatch, over, seed):
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  from multiverse_b200 import synthetic
  tf.reset_default_graph()
  cfg = synthetic.make_config(batch_size=1, **over)
  a = types.SimpleNamespace(**vars(cfg))
  a.modelname, a.use_soft_grid_class, a.use_gt_grid = "model", False, False
  w = synthetic.make_weights(cfg, seed)
  model = pred_models.get_model(a, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  return tf, cfg, model


def script_feeds(model, cfg, n, seed):
  """N=1 feed dicts shaped like Forking Paths: two frames per trajectory, lengths 10..26."""
  from multiverse_b200 import synthetic
  f = synthetic.make_feeds(cfg, n, seed)
  lengths = np.random.default_rng(seed).integers(10, 27, size=n)
  feeds = []
  for r in range(n):
    fd = {model.obs_length: np.array([cfg.obs_len], np.int32), model.pred_length: np.array([lengths[r]], np.int32),
          model.is_train: False,
          model.scene_feat: f["scene_feat"][[r, (r + 1) % n]].astype(np.float32),
          model.obs_scene: np.array([[0] * 4 + [1] * (cfg.obs_len - 4)], np.int32),
          model.obs_scene_mask: np.ones((1, cfg.obs_len), bool)}
    for j in range(len(cfg.scene_grids)):
      fd[model.grid_obs_labels[j]] = f["grid_obs_labels"][j][r:r + 1].astype(np.int32)
      if cfg.use_grids[j]:
        fd[model.grid_obs_regress[j]] = f["grid_obs_regress"][j][r:r + 1].astype(np.float64)
    feeds.append(fd)
  return feeds


def loop_outputs(tf, model, cfg, feeds, traj_ids, centers, num_out, center_only):
  """The script's loop: one sess.run per trajectory; point = centre + offset of the selected cell, float64."""
  gi = cfg.use_grids.index(True)
  c = centers.reshape([-1, 2])
  output_data, beam_prob = {}, {}
  with tf.Session() as sess:
    for tid, fd in zip(traj_ids, feeds):
      fetch = [model.grid_pred_decoded[gi], model.grid_pred_reg_decoded[gi]]
      if cfg.use_beam_search:
        fetch.append(model.beam_outputs)
      res = sess.run(fetch, feed_dict=fd)
      length = int(fd[model.pred_length][0])
      reg = res[1].reshape([1, length, -1, 2])
      if cfg.use_beam_search:
        lg, ids, lp = res[2]
      else:
        ids = np.argmax(res[0].reshape([1, length, -1]), axis=2)[:, None]
      trajs = []
      for j in range(ids.shape[1]):
        trajs.append([c[ids[0, j, t]] if center_only else c[ids[0, j, t]] + reg[0, t, ids[0, j, t], :]
                      for t in range(length)])
      output_data[tid] = trajs if cfg.use_beam_search else [trajs[0] for _ in range(num_out)]
      if cfg.use_beam_search:
        beam_prob[tid] = (lg, lp)
  return output_data, beam_prob


@pytest.mark.parametrize("case", ["k20_diverse", "greedy", "k20_center_only"])
def test_batched_driver_equals_the_per_trajectory_loop(case, monkeypatch):
  from multiverse_b200 import multifuture, synthetic
  over = dict(K20) if case != "greedy" else dict(K20, use_beam_search=False, beam_size=1, diverse_beam=False)
  n = 40 if case == "k20_diverse" else 12
  tf, cfg, model = make_model(monkeypatch, over, 21)
  feeds = script_feeds(model, cfg, n, 21)
  traj_ids = ["s%d_%d_%d_cam%d" % (r % 3, r, r + 7, r % 4) for r in range(n)]
  gi = cfg.use_grids.index(True)
  args = types.SimpleNamespace(scene_grid_centers=synthetic.grid_centers(cfg), num_out=20,
                               center_only=case == "k20_center_only")
  want = loop_outputs(tf, model, cfg, feeds, traj_ids, args.scene_grid_centers[gi], 20, args.center_only)
  got = multifuture.infer(model, feeds, 16, args, traj_ids, with_prob=cfg.use_beam_search)
  assert list(got[0]) == traj_ids
  assert pickle.dumps(got[0]) == pickle.dumps(want[0])
  assert pickle.dumps(got[1]) == pickle.dumps(want[1])
  if cfg.use_beam_search:       # the logits are fetched only when asked for
    assert multifuture.infer(model, feeds[:3], 16, args, traj_ids[:3])[1] == {}
