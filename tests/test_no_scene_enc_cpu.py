# coding=utf-8
"""Models built without --use_scene_enc pinned on executions of the reference's own code:
tests/golden/make_golden_no_scene_enc.py stored what the unmodified code/pred_models.py returned on the eager TF-1.15
stand-in, and the fp64 truth of tests/no_scene_enc_ref.py must reproduce it (<= 1e-12, ids identical), so the GPU tests
that compare against those goldens compare against the reference.  Also: the variables the drop-in Model and
synthetic.weight_shapes declare are the reference's, and the SimAug combinations are refused."""
import os
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import no_scene_enc_ref as NS  # noqa: E402
from multiverse_b200 import synthetic  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402

TOL = 1e-12
GOLD = os.path.join(ROOT, "tests", "golden")


def inputs(over, seed):
  cfg = NS.config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  return cfg, w, f, cases.checksum(*w.values()) + cases.checksum(f["traj"])


@pytest.mark.parametrize("name", sorted(NS.ROLLOUTS))
def test_truth_equals_reference_execution(name):
  cfg, w, f, ck = inputs(*NS.ROLLOUTS[name])
  g = np.load(os.path.join(GOLD, "rollout_noscene_%s.npz" % name))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  ref = NS.forward(cfg, w, f, np.float64)
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      assert ref["grid_pred_decoded"][i] == [] and "grid_pred_decoded_%d" % i not in g.files
      continue
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
      kk = "%s_%d" % (k, i)
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"], kk
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk
  if cfg.use_beam_search:
    lg, ids, lp = ref["beam_outputs"]
    assert np.array_equal(ids, g["beam_ids"])
    assert np.abs(cases.sample(lg) - g["beam_logits"]).max() <= TOL * g["beam_logits_absmax"]
    assert np.abs(lp - g["beam_logprobs"]).max() < 1e-11


def test_truth_equals_reference_training_step():
  """Losses and every (unclipped, then clipped as the Trainer does) gradient of the reference's Model + Trainer step at
  TRAINING.md's arguments without --use_scene, including the one grid_emb every scale shares."""
  over, seed = NS.TRAIN
  cfg, w, f, ck = inputs(over, seed)
  g = np.load(os.path.join(GOLD, "refexec_train_noscene.npz"))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  tot, losses, wd, grads = NS.loss_and_grads(cfg, w, f)
  assert abs(tot - float(g["loss"])) <= TOL * abs(tot) and abs(wd - float(g["wd_loss"])) <= TOL * wd
  assert np.abs(np.array(losses) - g["pred_grid_loss"]).max() <= TOL * max(losses)
  assert set(g["variables"]) == set(grads)
  for k, gr in grads.items():
    bar = TOL * max(float(g["grad_absmax/" + k]), 1e-30)
    assert np.abs(cases.sample(np.clip(gr, -10, 10), cases.NATIVE_TRAIN_SAMPLE) - g["grad/" + k]).max() <= bar, k
  # the shared embedding collects the gradient of both scales: neither scale alone accounts for it
  emb = grads[NS.ENC_EMB[0]]
  for used in ([True, False], [False, True]):
    one = NS.loss_and_grads(NS.config(**dict(over, use_grids=used)), w, f)[3][NS.ENC_EMB[0]]
    assert np.abs(one - emb).max() > 1e-3 * np.abs(emb).max()


def test_variables_are_the_references():
  """synthetic.weight_shapes (and so make_weights) and the drop-in Model declare exactly the variables, with the
  shapes, that the reference created in its execution: no scene_conv*, one person_pred/grid_emb for every scale and
  the class encoder's kernel [3,3,emb_size+256,1024]."""
  g = np.load(os.path.join(GOLD, "rollout_noscene_greedy_two_scale.npz"))
  theirs = {k: s for k, s in zip(g["variables"], g["variable_shapes"]) if k != "global_step"}
  cfg = NS.config(**NS.ROLLOUTS["greedy_two_scale"][0])
  assert {k: str(tuple(s)) for k, s in synthetic.weight_shapes(cfg).items()} == theirs
  assert theirs["person_pred/grid_emb/W"] == "(3, 3, 1, 32)"
  assert theirs["person_pred/encoder_grid_class_0/enc_grid_0/kernel"] == "(3, 3, 288, 1024)"
  assert not any("scene_conv" in k for k in theirs)
  model = dropin_model(cfg)
  assert {k: str(tuple(np.shape(v))) for k, v in model.weights().items()} == theirs


def dropin_model(cfg, **flags):
  sys.path.insert(0, os.path.join(ROOT, "multiverse_b200", "dropin"))
  try:
    import tensorflow as tf
    from multiverse_b200 import pred_models
  finally:
    sys.path.pop(0)
  tf.reset_default_graph()
  args = types.SimpleNamespace(**dict(vars(cfg), is_train=False, keep_prob=1.0, modelname="m",
                                      use_soft_grid_class=False, use_gt_grid=False), **flags)
  return pred_models.get_model(args, gpuid=0)


@pytest.mark.parametrize("flag", ["adv_train", "multiview_train", "standard_aug", "norm_input"])
def test_simaug_flags_are_refused(flag):
  """SimAug's model always encodes the scene, and its augmentations act on the scene input: without --use_scene_enc
  the engine configuration refuses them before any device work."""
  from multiverse_b200.pred_models import _engine_config
  cfg = NS.config(**NS.ROLLOUTS["greedy_two_scale"][0])
  model = dropin_model(cfg, **{flag: True})
  with pytest.raises(NotImplementedError, match="use_scene_enc"):
    _engine_config(model.config)
  _engine_config(dropin_model(cfg, **{flag: False}).config)       # the flag off: accepted


@pytest.mark.parametrize("use_gnn", [True, False])
def test_beam_replay_reproduces_the_truths_own_beam(use_gnn):
  """no_scene_enc_ref.beam_replay (the truth the GPU tests replay along the engine's selections), fed the selections
  of the fp64 beam search itself, reproduces that search's per-step logits: K = 4 diverse beam on 18x9."""
  sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
  import make_golden_no_scene_enc as M
  over = dict(batch_size=2, use_grids=[False, True], use_beam_search=True, beam_size=4, diverse_beam=True,
              diverse_gamma=0.01, fix_num_timestep=1, use_gnn=use_gnn)
  cfg, w, f, _ = inputs(over, 5)
  _, tr = M.beam_margins(cfg, w, f, 1)
  got = NS.beam_replay(cfg, w, f, 1, tr["ids"], tr["parents"])
  want = np.stack(tr["logits"])
  assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()
