# coding=utf-8
"""CPU pins of the training options of code/train.py:85-92 (--use_soft_grid_class, --mask_grid_regression, training
without --train_w_onehot) on executions of the unmodified reference (tests/golden/make_golden_train_options.py):

  - the drop-in's vectorised soft label maps equal the reference get_feed_dict's bit for bit, for soft_grid 1-7, and
    equal its per-(sample, step) ndimage.convolve loop on labels in every corner, edge and inside;
  - tests/train_options_ref.py - the fp64 truth the GPU tests hold the kernels and the engine to - equals the reference
    Model.build_loss + Trainer on every golden case: losses, the clipped gradients of every trainable variable and the
    variables after one Adadelta step."""
import os
import sys

import numpy as np
import pytest

import train_options_ref as TO
from oracle import multiverse_ref_torch as RT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
import make_golden_train_options as G  # noqa: E402


def gold(name):
  g = np.load(os.path.join(GOLD, name))
  assert str(g["source"]).startswith("reference_exec")
  return g


def test_soft_labels_equal_reference_feed_dict():
  from multiverse_b200.pred_models import _soft_labels
  from multiverse_b200 import synthetic
  g = gold("refexec_soft_labels.npz")
  cfg = synthetic.make_config()
  for mode in range(1, 8):
    for j, (h, w) in enumerate(cfg.scene_grids):
      want = g["mode%d/labels/%d" % (mode, j)]
      mine = _soft_labels(g["mode%d/pred_grid_class/%d" % (mode, j)], h, w, mode)
      assert mine.dtype == np.float32 and mine.shape == want.shape
      assert np.array_equal(mine, want.astype(np.float32)), (mode, j)


@pytest.mark.parametrize("mode", range(1, 8))
def test_soft_labels_equal_the_convolution_loop(mode):
  from multiverse_b200.pred_models import _soft_labels
  for h, w in ((36, 18), (18, 9)):
    rng = np.random.default_rng(mode + h)
    cls = rng.integers(0, h * w, size=(6, 12))
    cells = [0, 1, w - 1, w, (h - 1) * w, h * w - 1, h * w - 2, (h // 2) * w, (h // 2) * w + w - 1, w + 1, 2 * w + 2]
    cls[0, :len(cells)] = cells
    cls[1, :len(cells)] = cells[::-1]
    want = G.soft_maps_reference(cls, h, w, mode).astype(np.float32)
    assert np.array_equal(_soft_labels(cls, h, w, mode), want)


def test_reference_restatement_without_options_equals_the_oracle():
  """With every option off, train_options_ref is the oracle's loss_and_grads."""
  cfg, w, f = G.case_inputs("sparse_mask")
  tot, losses, wd, grads = TO.loss_and_grads(cfg, w, f)
  tot_o, losses_o, wd_o, grads_o = RT.loss_and_grads(cfg, w, f)
  assert abs(tot - tot_o) <= 1e-13 * abs(tot_o) and np.abs(np.subtract(losses, losses_o)).max() <= 1e-13
  for k in grads:
    assert np.abs(grads[k] - grads_o[k]).max() <= 1e-13 * max(np.abs(grads_o[k]).max(), 1e-30), k


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_options_reference_equals_reference_execution(case):
  mode, mask, onehot = G.CASES[case]
  cfg, w, f = G.case_inputs(case)
  got = gold("refexec_train_%s.npz" % case)
  tot, losses, wd, grads = TO.loss_and_grads(cfg, w, f, soft=bool(mode), mask=mask, onehot=onehot)
  assert abs(float(got["loss"]) - tot) <= 1e-12 * abs(tot)
  assert abs(float(got["wd_loss"]) - wd) <= 1e-12 * wd
  assert np.abs(got["pred_grid_loss"] - np.array(losses)).max() <= 1e-12 * max(losses)
  assert set(got["variables"]) == set(w) == set(grads)
  lr = 0.2                                            # init_lr * emb_lr * decay^0 at step 0
  for k, g in grads.items():
    gc = np.clip(g, -10.0, 10.0)                      # Trainer: clip_by_value +-clip_gradient_norm (:1700-1705)
    scale = max(np.abs(gc).max(), 1e-30)
    assert abs(float(got["grad_absmax/" + k]) - np.abs(gc).max()) <= 1e-12 * scale, k
    assert np.abs(got["grad/" + k] - G.sample(gc)).max() <= 1e-12 * scale, k
    upd = np.sqrt(1e-8) / np.sqrt(0.05 * gc * gc + 1e-8) * gc         # Adadelta(rho .95, eps 1e-8), zero slots
    assert np.abs(got["updated/" + k] - G.sample(w[k].astype(np.float64) - lr * upd)).max() < 1e-12, k
