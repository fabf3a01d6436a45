# coding=utf-8
"""The --emb_size matrix of tests/emb_matrix_cases.py: it reaches every cell row width cpad that an accepted
--emb_size produces, with an x block narrower than its padding at each; and the fp64 oracle against the executed
reference at embedding widths that are not a multiple of 32 (tests/golden/make_golden_emb_matrix.py)."""
import os

import numpy as np
import pytest

import emb_matrix_cases as EM
from multiverse_b200 import ops


def test_matrix_reaches_every_cpad():
  """Every E in range(8, 257, 8) maps to a cpad of the table, every such cpad has a full and a padded x block, and
  the GPU matrix launches every cpad with padding and the new ones (416, 448, 480) both ways."""
  cpads = {ops.cell_cpad(e) for e in range(8, 257, 8)}
  assert cpads == set(EM.CPADS) == set(range(288, 513, 32))
  for cpad, (full, padded) in EM.CPADS.items():
    assert ops.cell_cpad(full) == ops.cell_cpad(padded) == EM.cpad_of(padded) == cpad
    assert full == cpad - 256 and padded % 8 == 0 and padded % 32 != 0 and padded < full
  assert {ops.cell_cpad(e) for e in EM.MATRIX} == cpads
  assert {e for e in EM.MATRIX if ops.cell_cpad(e) in EM.NEW_CPADS} == {
      e for c in EM.NEW_CPADS for e in EM.CPADS[c]}
  assert set(EM.PADDED) <= set(EM.MATRIX)


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-12


@pytest.mark.parametrize("name", sorted(EM.ROLLOUTS))
def test_truth_equals_reference_execution(name):
  """The fp64 oracle reproduces the executed reference (tests/golden/rollout_emb_<name>.npz) to 1e-12."""
  import cases
  from oracle import multiverse_ref as R
  from test_emb_size_cpu import golden_inputs
  cfg, w, f, ck = golden_inputs(*EM.ROLLOUTS[name])
  g = np.load(os.path.join(GOLD, "rollout_emb_%s.npz" % name))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  assert cfg.use_scene_enc and not cfg.use_beam_search
  ref = R.forward(cfg, w, f, np.float64)
  for i in range(len(cfg.scene_grids)):
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
      kk = "%s_%d" % (k, i)
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"], kk
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk
    lg = np.asarray(ref["grid_pred_decoded"][i])
    assert np.array_equal(lg.reshape(lg.shape[0], lg.shape[1], -1).argmax(-1),
                          g["logits_%d" % i].reshape(lg.shape[0], lg.shape[1], -1).argmax(-1)), i


@pytest.mark.parametrize("name", sorted(EM.TRAIN))
def test_truth_equals_reference_training_step(name):
  """The fp64 autograd truth reproduces the reference Model + Trainer step's losses and clipped gradients
  (tests/golden/refexec_train_emb_<name>.npz) to 1e-12."""
  import cases
  import no_scene_enc_ref as NS
  from oracle import multiverse_ref_torch as RT
  from test_emb_size_cpu import golden_inputs
  over, seed = EM.TRAIN[name]
  cfg, w, f, ck = golden_inputs(dict(over, **{k: v for k, v in EM.TRAIN_ARGS.items() if k != "optimizer"}), seed)
  g = np.load(os.path.join(GOLD, "refexec_train_emb_%s.npz" % name))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  tot, losses, wd, grads = (RT.loss_and_grads if cfg.use_scene_enc else NS.loss_and_grads)(cfg, w, f)
  assert abs(tot - float(g["loss"])) <= TOL * abs(tot) and abs(wd - float(g["wd_loss"])) <= TOL * wd
  assert np.abs(np.array(losses) - g["pred_grid_loss"]).max() <= TOL * max(losses)
  assert set(g["variables"]) == set(grads)
  for k, gr in grads.items():
    bar = TOL * max(float(g["grad_absmax/" + k]), 1e-30)
    assert np.abs(cases.sample(np.clip(gr, -10, 10), cases.NATIVE_TRAIN_SAMPLE) - g["grad/" + k]).max() <= bar, k
