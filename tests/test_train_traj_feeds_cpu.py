# coding=utf-8
"""CPU tests of the training feed dict's trajectory path (SURVEY.md §8 row f-1, training half; host logic only):
Model.get_feed_dict(batch, is_train=True, train_traj=True) - what Trainer.step asks for - feeds the trajectories, the
grid centres and int32 label cells exactly when the batch allows it, and the reference's dense feed dict otherwise.
Also the host-to-device byte count of tools/time_train_feeds.py, from shapes."""
import copy
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

from multiverse_b200.pred_models import _soft_labels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 4


@pytest.fixture()
def dropin(monkeypatch):
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  return tf, pred_models


def make(tf, pm, **flags):
  from multiverse_b200 import synthetic
  tf.reset_default_graph()
  cfg = synthetic.make_config(batch_size=N, is_train=True, scene_h=36, scene_w=64, scene_grid_strides=[2, 4],
                              use_grids=[True, True])
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname = "m"; args.use_gt_grid = False; args.use_soft_grid_class = False; args.soft_grid = 1
  for k, v in flags.items():
    setattr(args, k, v)
  model = pm.get_model(args, gpuid=0)
  f = synthetic.make_feeds(cfg, N, 3, with_pred=True)
  t = cfg.obs_len
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(2)]) for i in range(N)],
              pred_grid_class=[np.stack([f["grid_pred_labels"][j][i] for j in range(2)]) for i in range(N)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None],
              obs_traj=list(f["traj64"][:, :t]), pred_traj=list(f["traj64"][:, t:]))
  for j in range(2):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  shared = {"grid_center_%d" % j: c for j, c in enumerate(synthetic.grid_centers(cfg))}
  return model, args, cfg, types.SimpleNamespace(data=data, shared=shared)


def is_traj(model, fd):
  dense = [model.grid_obs_regress[j] in fd or model.grid_pred_regress[j] in fd for j in range(2)]
  if model.pred_traj in fd:
    assert model.obs_traj in fd and not any(dense)
    return True
  assert all(dense)
  return False


@pytest.mark.parametrize("soft", [False, True], ids=["sparse", "soft"])
def test_trajectory_feeds_when_the_batch_allows(dropin, soft):
  tf, pm = dropin
  model, args, cfg, batch = make(tf, pm, use_soft_grid_class=soft, soft_grid=7)
  fd = model.get_feed_dict(batch, is_train=True, train_traj=True)
  assert is_traj(model, fd)
  assert fd[model.obs_traj].dtype == np.float64 and fd[model.obs_traj].shape == (N, cfg.obs_len, 2)
  assert fd[model.pred_traj].dtype == np.float64 and fd[model.pred_traj].shape == (N, cfg.pred_len, 2)
  dense = model.get_feed_dict(batch, is_train=True)        # the reference's feed dict, what Trainer.step replaced
  for j, (h, w) in enumerate(cfg.scene_grids):
    c = fd[model.grid_centers[j]]
    assert c.dtype == np.float64 and c.shape == (h, w, 2)
    lab = fd[model.grid_pred_labels_T[j]]
    assert lab.dtype == np.int32 and lab.shape == (N, cfg.pred_len)
    assert np.array_equal(fd[model.grid_obs_labels[j]], dense[model.grid_obs_labels[j]])
    # what the kernels compute from these feeds is what the dense feed dict holds
    obs = (fd[model.obs_traj][:, :, None, None] - c[None, None]).astype(np.float32)
    pred = (fd[model.pred_traj][:, :, None, None] - c[None, None]).astype(np.float32)
    assert np.array_equal(obs, dense[model.grid_obs_regress[j]])
    assert np.array_equal(pred, dense[model.grid_pred_regress[j]])
    want = _soft_labels(lab, h, w, 7) if soft else lab
    assert np.array_equal(want, dense[model.grid_pred_labels_T[j]])
  for k in (model.scene_feat, model.obs_scene, model.obs_scene_mask, model.obs_length, model.pred_length):
    assert np.array_equal(np.asarray(fd[k]), np.asarray(dense[k]))


def test_dense_feeds_otherwise(dropin):
  tf, pm = dropin
  model, args, cfg, batch = make(tf, pm)
  assert not is_traj(model, model.get_feed_dict(batch, is_train=True))                    # the reference's call
  args.device_grid_feeds = False
  assert not is_traj(model, model.get_feed_dict(batch, is_train=True, train_traj=True))
  args.device_grid_feeds = True

  def variant(edit):
    b = types.SimpleNamespace(data=copy.copy(batch.data), shared=copy.copy(batch.shared))
    edit(b)
    return is_traj(model, model.get_feed_dict(b, is_train=True, train_traj=True))

  assert variant(lambda b: None)
  assert not variant(lambda b: b.data.pop("pred_traj"))
  assert not variant(lambda b: b.data.pop("obs_traj"))
  assert not variant(lambda b: b.shared.pop("grid_center_1"))
  assert not variant(lambda b: setattr(b, "shared", None))
  assert not variant(lambda b: b.shared.update(grid_center_0=b.shared["grid_center_0"][:, :-1]))
  # dense targets that do not come from the trajectories (the sampled check), observed or future
  assert not variant(lambda b: b.data.update(obs_grid_target_all_0=[a + 1.0 for a in b.data["obs_grid_target_all_0"]]))
  assert not variant(lambda b: b.data.update(pred_grid_target_all_1=[a * 2.0 for a in b.data["pred_grid_target_all_1"]]))
  # a short trajectory; a partial batch (its padded rows are zeros, which no trajectory gives)
  assert not variant(lambda b: b.data.update(pred_traj=[p[:-1] for p in b.data["pred_traj"]]))
  for k in ("obs_grid_class", "pred_grid_class", "obs_traj", "pred_traj", "obs_grid_target_all_0",
            "obs_grid_target_all_1", "pred_grid_target_all_0", "pred_grid_target_all_1"):
    batch.data[k] = batch.data[k][:N - 1]
  assert not is_traj(model, model.get_feed_dict(batch, is_train=True, train_traj=True))


@pytest.mark.parametrize("flags", [dict(use_soft_grid_class=True, soft_grid=9), dict(multiview_train=True),
                                   dict(adv_train=True)], ids=["unknown_soft_grid", "multiview", "adv_train"])
def test_dense_feeds_for_other_configurations(dropin, flags):
  tf, pm = dropin
  model, args, cfg, batch = make(tf, pm)
  for k, v in flags.items():
    setattr(args, k, v)
  assert model._train_traj_feeds(batch, N) is None


def test_soft_labels_outside_the_grid_keep_the_dense_path(dropin):
  """A label cell numpy cannot index keeps the dense path (whose _soft_labels raises, as the reference does)."""
  tf, pm = dropin
  model, args, cfg, batch = make(tf, pm, use_soft_grid_class=True, soft_grid=3)
  h, w = cfg.scene_grids[1]
  lab = np.array(batch.data["pred_grid_class"][0])
  lab[1, 0] = -h * w
  batch.data["pred_grid_class"][0] = lab
  assert model._train_traj_feeds(batch, N) is not None     # counted from the end, as numpy does
  lab[1, 0] = h * w
  assert model._train_traj_feeds(batch, N) is None


def test_host_to_device_bytes_from_shapes(dropin):
  tf, pm = dropin
  spec = importlib.util.spec_from_file_location("time_train_feeds", os.path.join(ROOT, "tools", "time_train_feeds.py"))
  tool = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(tool)
  model, args, cfg, batch = make(tf, pm, use_soft_grid_class=True, soft_grid=1)
  T, Tp = cfg.obs_len, cfg.pred_len
  common = batch.data["batch_scene_feat"].size * 4 + N * T * 4 + sum(N * T * 4 for _ in cfg.scene_grids)
  hw = [h * w for h, w in cfg.scene_grids]
  dense = common + sum(N * (T + Tp) * v * 2 * 4 + N * Tp * v * 4 for v in hw)
  traj = common + N * (T + Tp) * 2 * 8 + sum(v * 2 * 8 + N * Tp * 4 for v in hw)
  assert tool.h2d_bytes(model, model.get_feed_dict(batch, is_train=True)) == dense
  assert tool.h2d_bytes(model, model.get_feed_dict(batch, is_train=True, train_traj=True)) == traj
