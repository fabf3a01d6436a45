# coding=utf-8
"""The beam decoder without graph attention (use_gnn off: code/pred_models.py:474-806 hands the gathered parent state
straight to the cell) pinned on an execution of the reference's own code.  tests/golden/make_golden_ablation.py stored
what the unmodified code/pred_models.py returned on the eager TF-1.15 stand-in; the oracle must reproduce it (fp64,
<= 1e-12, ids identical), so the GPU tests that compare against those goldens compare against the reference."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import cases_ablation  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402

TOL = 1e-12
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("name", sorted(cases_ablation.ROLLOUTS_NO_GNN))
def test_beam_without_attention_oracle_equals_reference_execution(name):
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**over)
  assert not cfg.use_gnn and cfg.use_beam_search and cfg.use_scene_enc
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "rollout_%s.npz" % name))
  assert str(g["source"]) == "reference_exec"
  assert abs(float(g["checksum"]) - (cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"]))) < 1e-6
  # the model has the same variables with and without the attention (it has no parameters)
  assert set(g["variables"]) - {"global_step"} == set(w.keys())
  ref = R.forward(cfg, w, f, np.float64)
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      assert ref["grid_pred_decoded"][i] == [] and "grid_pred_decoded_%d" % i not in g.files
      continue
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
      kk = "%s_%d" % (k, i)
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"], kk
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk
  lg, ids, lp = ref["beam_outputs"]
  assert np.array_equal(ids, g["beam_ids"])
  assert np.abs(cases.sample(lg) - g["beam_logits"]).max() <= TOL * g["beam_logits_absmax"]
  assert np.abs(lp - g["beam_logprobs"]).max() < 1e-11
  assert np.abs(lg.max(-1) - g["beam_lg_max"]).max() <= TOL * g["beam_logits_absmax"]


def test_beam_without_attention_differs_from_beam_with_it():
  """The goldens exercise the branch: with the attention the same weights and inputs decode other beams."""
  name = "beam_k5_nognn"
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**dict(over, use_gnn=True))
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  with_gnn = R.forward(cfg, w, f, np.float64)["beam_outputs"]
  g = np.load(os.path.join(GOLD, "rollout_%s.npz" % name))
  assert np.abs(with_gnn[2] - g["beam_logprobs"]).max() > 1e-3
