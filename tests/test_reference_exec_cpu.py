# coding=utf-8
"""Pins the oracle on an EXECUTION of the reference's own graph code.

``oracle/tf1_eager`` imports the unmodified ``code/pred_models.py`` of the reference repository against an eager,
torch-fp64-backed stand-in for the TensorFlow-1.15 symbols it uses and runs ``Model.__init__ / build_forward /
build_loss`` and ``Trainer.__init__`` as written.  tests/golden/make_golden_refexec.py stored what that run returned
(tests/golden/refexec_*.npz); these tests assert that ``oracle/multiverse_ref.py`` reproduces it (fp64, <=1e-12; ids
identical) - the wiring of code/pred_models.py:123-308, 311-471, 474-806, 808-909, 961-1040, 1197-1251, 1636-1717 is
therefore pinned on executed reference code, not a restatement; only the per-op TF semantics underneath stay restated
(and torch-anchored in test_oracle_cpu.py).
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402

TOL = 1e-12
GOLD = os.path.join(ROOT, "tests", "golden")


def gold(name):
  g = np.load(os.path.join(GOLD, name))
  assert str(g["source"]).startswith("reference_exec")
  return g


def check_forward(name):
  over, seed = cases.REFEXEC_FORWARD[name]
  cfg = R.default_config(**over)
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  ref = R.forward(cfg, w, f, np.float64)
  g = gold("refexec_forward.npz")
  key = lambda k: "%s/%s" % (name, k)
  assert set(g[key("variables")]) - {"global_step"} == set(w.keys())     # TF variable names, §8a
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      assert ref["grid_pred_decoded"][i] == [] and key("grid_pred_decoded_%d" % i) not in g.files     # :170-171
      continue
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded", "scene_convs"):
      kk = key("%s_%d" % (k, i))
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"]
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk
  if cfg.use_beam_search:
    lg, ids, lp = ref["beam_outputs"]
    assert np.array_equal(ids, g[key("beam_ids")])
    assert np.abs(cases.sample(lg) - g[key("beam_logits")]).max() <= TOL * g[key("beam_logits_absmax")]
    assert np.abs(lp - g[key("beam_logprobs")]).max() < 1e-11
  else:
    assert ref["beam_outputs"] is None and key("beam_ids") not in g.files
  return ref


def test_reference_beam_k5_plain_equals_oracle_and_golden():
  """Coarse 18x9 grid, K=5 plain beam (no penalty, fix_num_timestep=0): the reference's own
  grid_decoder_beam_search + back-trace, and the committed rollout golden made from the same execution."""
  ref = check_forward("beam_k5_plain")
  g = np.load(os.path.join(GOLD, "rollout_beam_k5_plain.npz"))
  assert str(g["source"]) == "reference_exec"
  assert np.array_equal(g["beam_ids"], ref["beam_outputs"][1])
  assert np.abs(g["beam_logprobs"] - ref["beam_outputs"][2]).max() < 1e-11
  assert np.abs(g["logits_1"] - ref["grid_pred_decoded"][1]).max() < 1e-6     # stored as fp32


def test_reference_beam_k20_diverse_equals_oracle():
  """K=20 diverse beam (gamma 0.01, first step's scores zeroed) - the multifuture_inference.py
  configuration (TESTING.md:84-93) - on the coarse grid with 3 trajectories."""
  check_forward("beam_k20_diverse")


def test_reference_greedy_two_scale_equals_oracle():
  """Both scales, greedy class decoder with graph attention + regression decoder (test.py path)."""
  assert R.default_config(**cases.REFEXEC_FORWARD["greedy_two_scale"][0]).scene_grids == [(12, 8), (6, 4)]
  check_forward("greedy_two_scale")


def test_reference_ragged_pred_length_and_no_gnn():
  """use_gnn off (the reference then hands the raw state to the cell)."""
  check_forward("no_gnn")


def test_reference_training_step_equals_oracle():
  """Model.build_loss + Trainer.__init__ executed: total / class / Huber / wd losses, the clipped
  gradient of every trainable variable (tf.gradients -> clip_by_value +-10, :1698-1705) and one
  Adadelta train_op (:1672,:1716) against the oracle's torch-autograd restatement and the
  closed-form update the CUDA optimizer kernel implements."""
  from oracle import multiverse_ref_torch as RT
  over, seed, _ = cases.REFEXEC_TRAIN
  cfg = R.default_config(**over)
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  got = gold("refexec_train.npz")
  tot, losses, wd, grads = RT.loss_and_grads(cfg, w, f)
  assert abs(float(got["loss"]) - tot) < 1e-11 * abs(tot)
  assert abs(float(got["wd_loss"]) - wd) < 1e-12 * wd
  assert np.abs(got["pred_grid_loss"] - np.array(losses)).max() < 1e-11
  assert set(got["variables"]) == set(w.keys()) == set(grads)
  lr = 0.2 * 1.0 * 0.95 ** 0        # init_lr * emb_lr * decay^(floor(step/decay_steps)), step 0
  for k, g in grads.items():
    gc = np.clip(g, -10.0, 10.0)
    scale = max(np.abs(gc).max(), 1e-30)
    assert abs(float(got["grad_absmax/" + k]) - np.abs(gc).max()) <= 1e-10 * scale, k
    assert np.abs(got["grad/" + k] - cases.sample(gc)).max() <= 1e-10 * scale, k
    acc = 0.05 * gc * gc                                  # rho=.95, zero slots, eps=1e-8
    upd = np.sqrt(1e-8) / np.sqrt(acc + 1e-8) * gc
    want = w[k].astype(np.float64) - lr * upd
    assert np.abs(got["updated/" + k] - cases.sample(want)).max() < 1e-12, k
  assert int(got["global_step"]) == 1


def test_reference_native_two_scale_forward_equals_oracle():
  """The published scene 36x64 (grids 18x32 and 9x16, the only ones wider than tall), greedy decode of both scales
  with graph attention: class logits, offsets and scene convolutions (tests/golden/refexec_native.npz)."""
  cfg, w, f = cases.refexec_native_inputs()
  assert cfg.scene_grids == [(18, 32), (9, 16)] and cfg.use_grids == [True, True]
  ref = R.forward(cfg, w, f, np.float64)
  g = gold("refexec_native.npz")
  assert set(g["forward/variables"]) - {"global_step"} == set(w.keys())
  for i in range(2):
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded", "scene_convs"):
      kk = "forward/%s_%d" % (k, i)
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"], kk
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk


def test_reference_native_training_step_equals_oracle():
  """TRAINING.md's training step on the 36x64 scene: both scales, --train_w_onehot, loss weights 1.0 / 0.2, weight
  decay 0.001 and one Adadelta train_op at --init_lr 0.3: the losses, the clipped gradient of every variable and the
  updated variables against the oracle's torch-autograd restatement and the closed-form update."""
  from oracle import multiverse_ref_torch as RT
  cfg, w, f = cases.refexec_native_inputs()
  opts = cases.REFEXEC_NATIVE[2]
  assert (cfg.grid_loss_weight, cfg.grid_reg_loss_weight, cfg.wd) == (
      opts["grid_loss_weight"], opts["grid_reg_loss_weight"], opts["wd"])
  got = gold("refexec_native.npz")
  tot, losses, wd, grads = RT.loss_and_grads(cfg, w, f)
  assert abs(float(got["train/loss"]) - tot) < 1e-11 * abs(tot)
  assert abs(float(got["train/wd_loss"]) - wd) < 1e-12 * wd
  assert len(losses) == 4 and np.abs(got["train/pred_grid_loss"] - np.array(losses)).max() < 1e-11
  assert set(got["train/variables"]) == set(w.keys()) == set(grads)
  lr = opts["init_lr"] * 1.0 * 0.95 ** 0        # init_lr * emb_lr * decay^(floor(step/decay_steps)), step 0
  smp = lambda a: cases.sample(a, cases.NATIVE_TRAIN_SAMPLE)
  for k, g in grads.items():
    gc = np.clip(g, -10.0, 10.0)
    scale = max(np.abs(gc).max(), 1e-30)
    assert abs(float(got["train/grad_absmax/" + k]) - np.abs(gc).max()) <= 1e-10 * scale, k
    assert np.abs(got["train/grad/" + k] - smp(gc)).max() <= 1e-10 * scale, k
    acc = 0.05 * gc * gc                                  # rho=.95, zero slots, eps=1e-8
    upd = np.sqrt(1e-8) / np.sqrt(acc + 1e-8) * gc
    want = w[k].astype(np.float64) - lr * upd
    assert np.abs(got["train/updated/" + k] - smp(want)).max() < 1e-12, k
  assert int(got["train/global_step"]) == 1
