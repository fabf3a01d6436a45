# coding=utf-8
"""GPU tests of the device single-future evaluation (multiverse_b200.single_future_eval.evaluate).

- Scoring: the golden cases' stored decode outputs, uploaded in the engine's layouts in place of a forward, give the
  dicts and save_output pickles the reference's pred_utils.evaluate returned and wrote, bit for bit, one batch per
  forward and several.
- End to end: synthetic weights through the drop-in Model / Tester and the restated Dataset (a partial last batch):
  the device evaluate at one batch per forward and at its default grouping equals the restated host evaluate run over
  Tester.step - keys, values (==), types and the save_output pickle - for TESTING.md's test model, TRAINING.md's
  validation (the training model after two Trainer.steps), beam search, --use_gt_grid and --per_scene_eval.
- Host traffic: without --save_output nothing larger than [rows, T] comes back to the host and the fetch path
  (Model._engine_forward) is not used."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

import single_future_eval_cases as C
import single_future_eval_ref as ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "single_future_eval.npz")


# ------------------------------------------------------------------ scoring of the golden cases' stored outputs
class ReplayModel(object):
  """Stands in for the drop-in Model: get_feed_dict records the batch order, and single_future_eval._forward (patched)
  returns the stored outputs of the batches of a forward, uploaded in the engine's layouts."""

  def __init__(self, cfg, outs):
    import torch
    self.config, self.outs, self.fed = cfg, outs, 0
    h = lambda name, i=None: ("h", name, i)
    self.scene_feat, self.obs_scene, self.pred_length, self.obs_traj = (h("scene_feat"), h("obs_scene"),
                                                                        h("pred_length"), h("obs_traj"))
    self.grid_obs_labels = [h("grid_obs_labels", i) for i in range(len(cfg.scene_grids))]
    self.grid_obs_regress = [h("grid_obs_regress", i) for i in range(len(cfg.scene_grids))]
    self.grid_centers = [h("grid_centers", i) for i in range(len(cfg.scene_grids))]
    self.engine = types.SimpleNamespace(device=torch.device("cuda", 0))

  def _ensure_engine(self):
    return self.engine

  def get_feed_dict(self, batch, is_train=False):
    n = C.BS
    fd = {self.scene_feat: batch.data["batch_scene_feat"], self.obs_scene: batch.data["batch_obs_scene"][..., 0],
          self.pred_length: np.full((n,), C.T_PRED, np.int32)}
    for j in range(len(C.GRIDS)):
      fd[self.grid_obs_labels[j]] = np.zeros((n, C.T_OBS), np.int32)
      fd[self.grid_obs_regress[j]] = np.zeros((n, 1), np.float32)
    return fd

  def forward(self, model, feed):
    import torch
    n = feed[self.obs_scene].shape[0]
    outs = self.outs[self.fed:self.fed + n // C.BS]
    self.fed += len(outs)
    dev = self.engine.device
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    res = dict(grid_pred_decoded=[], grid_pred_reg_decoded=[], beam_outputs=None, _offs={})
    for j, (h, w) in enumerate(C.GRIDS):
      if not self.config.use_grids[j]:
        res["grid_pred_decoded"].append([]); res["grid_pred_reg_decoded"].append([])
        continue
      reg = np.concatenate([o[1][j] for o in outs])
      res["grid_pred_decoded"].append(up(np.concatenate([o[0][j] for o in outs])))
      res["grid_pred_reg_decoded"].append(up(reg))
      res["_offs"][j] = up(reg.reshape(n, C.T_PRED, h * w, 2).transpose(1, 0, 2, 3))     # [Tp,N,HW,2]
    if self.config.use_beam_search:
      res["beam_outputs"] = [up(np.concatenate([o[2][i] for o in outs])) for i in range(3)]
    return res


@pytest.mark.parametrize("batches_per_forward", [1, 2, None])
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_scoring_of_stored_outputs_equals_reference(name, batches_per_forward, tmp_path, monkeypatch):
  from multiverse_b200 import single_future_eval as sfe
  z = np.load(GOLDEN)
  cfg, simaug = C.case_config(name, str(tmp_path / "out.p"))
  if name == "per_scene_eval":
    cfg.save_output = None
  data, shared = C.case_data(C.load_set(z), simaug)
  ds = ref.Dataset(data, "test", config=cfg, shared=shared)
  model = ReplayModel(cfg, C.load_outputs(z, name, cfg))
  monkeypatch.setattr(sfe, "_forward", model.forward)
  monkeypatch.setitem(sys.modules, "pred_utils", ref)          # the script's get_scene
  rows = None if batches_per_forward is None else batches_per_forward * C.BS
  p = sfe.evaluate(ds, cfg, None, types.SimpleNamespace(model=model), rows_per_forward=rows)
  assert model.fed == len(model.outs)
  ref.assert_same_dict(p, pickle.loads(z[name + "/p"].tobytes()))
  if cfg.save_output is not None:
    with open(cfg.save_output, "rb") as f:
      ref.assert_same_out_data(pickle.load(f), pickle.loads(z[name + "/out_data"].tobytes()))


# ------------------------------------------------------------------ end to end through the drop-in model
TEST_MODEL = dict(scene_h=36, scene_w=64, scene_grid_strides=[2, 4], use_grids=[True, False], emb_size=32,
                  use_scene_enc=True, use_gnn=True, batch_size=16)
TRAIN_FLAGS = dict(grid_loss_weight=1.0, wd=0.001, clip_gradient_norm=10.0, optimizer="adadelta", emb_lr=1.0,
                   learning_rate_decay=0.95, num_epoch_per_decay=2.0, train_num_examples=100, use_cosine_lr=False,
                   use_soft_grid_class=False, soft_grid=1, mask_grid_regression=False, train_w_onehot=True,
                   init_lr=0.3, use_teacher_forcing=False)


def build(monkeypatch, over, n_rows, seed=3, train=False):
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  monkeypatch.setitem(sys.modules, "pred_utils", ref)
  import tensorflow as tf
  import pred_models
  from multiverse_b200 import synthetic
  tf.reset_default_graph()
  base = dict(TEST_MODEL)
  base.update(over)
  cfg = synthetic.make_config(is_train=train, **base)
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname, args.use_gt_grid, args.per_scene_eval, args.save_output = "model", False, False, None
  args.use_soft_grid_class = False
  if train:
    for k, v in TRAIN_FLAGS.items():
      setattr(args, k, v)
  for k in ("use_gt_grid", "per_scene_eval"):
    if k in over:
      setattr(args, k, over[k])
  w = synthetic.make_weights(cfg, seed)
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  return tf, pred_models, model, args, ref.synthetic_dataset(args, n_rows, seed)


def compare(tf, pred_models, model, args, ds, tmp_path, save_output=True):
  from multiverse_b200 import single_future_eval as sfe
  import torch
  args.save_output = str(tmp_path / "host.p") if save_output else None
  with tf.Session() as sess:
    want, want_out = ref.evaluate(ds, args, ref.tester_step(model, sess))
    tester = pred_models.Tester(model, args, sess)
    for rows in (args.batch_size, None):
      args.save_output = str(tmp_path / ("dev%s.p" % rows)) if save_output else None
      got = sfe.evaluate(ds, args, sess, tester, rows_per_forward=rows)
      torch.cuda.synchronize()
      ref.assert_same_dict(got, want)
      if save_output:
        with open(args.save_output, "rb") as f:
          ref.assert_same_out_data(pickle.load(f), want_out)
  return want


E2E = {
    "test_model": (dict(), 45),
    "beam_k5_diverse": (dict(use_beam_search=True, beam_size=5, diverse_beam=True, diverse_gamma=0.01), 37),
    "use_gt_grid": (dict(use_grids=[True, True], use_gt_grid=True), 40),
    "per_scene_eval": (dict(per_scene_eval=True), 45),
}


@pytest.mark.parametrize("name", sorted(E2E))
def test_device_evaluate_equals_host_evaluate(name, monkeypatch, tmp_path):
  over, n = E2E[name]
  tf, pred_models, model, args, ds = build(monkeypatch, over, n)
  assert n % args.batch_size
  p = compare(tf, pred_models, model, args, ds, tmp_path, save_output=name != "per_scene_eval")
  assert np.isfinite(p["grid0_traj_ade"])


def test_validation_of_the_training_model_equals_host_evaluate(monkeypatch, tmp_path):
  """TRAINING.md's validation: the training model itself (its TrainEngine decodes) after two Trainer.steps."""
  tf, pred_models, model, args, ds = build(monkeypatch, dict(use_grids=[True, True], batch_size=20), 50, train=True)
  trainer = pred_models.Trainer(model, args)
  with tf.Session() as sess:
    for b, batch in enumerate(ds.get_batches(args.batch_size, full=True, shuffle=False)):
      if b == 2:
        break
      trainer.step(sess, batch)
  from multiverse_b200 import train_engine
  assert isinstance(model._ensure_engine(), train_engine.TrainEngine)
  compare(tf, pred_models, model, args, ds, tmp_path)


def test_no_dense_fetch_without_save_output(monkeypatch, tmp_path):
  from multiverse_b200 import single_future_eval as sfe
  tf, pred_models, model, args, ds = build(monkeypatch, dict(use_grids=[True, True]), 45)
  shapes = []
  real = sfe._to_host
  monkeypatch.setattr(sfe, "_to_host", lambda t: shapes.append(tuple(t.shape)) or real(t))

  def no_fetch(*a, **k):
    raise AssertionError("Model._engine_forward called")

  monkeypatch.setattr(type(model), "_engine_forward", no_fetch)
  with tf.Session() as sess:
    sfe.evaluate(ds, args, sess, pred_models.Tester(model, args, sess))
  # one forward of 48 rows: per used scale the selections and the two error arrays
  assert shapes == [(48, args.pred_len)] * 6
