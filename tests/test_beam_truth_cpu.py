# coding=utf-8
"""The fp64 truth the multi-future GPU tests replay along the engine's selections (tests/beam_truth.py: beam_replay),
fed the selections of the fp64 beam search itself (RT.decoder_beam), reproduces that search's per-step logits over the
longest future a multi-future rollout decodes (26 steps), with and without scene encoding: K = 4 diverse beam with
graph attention on a 6x8 grid."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import beam_truth as BT  # noqa: E402
from multiverse_b200 import synthetic  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402

TP = 26


@pytest.mark.parametrize("use_scene_enc", [True, False], ids=["scene_enc", "no_scene_enc"])
def test_beam_replay_reproduces_the_truths_own_beam_over_26_steps(use_scene_enc):
  over = dict(batch_size=2, scene_h=12, scene_w=16, use_grids=[True, False], use_beam_search=True, beam_size=4,
              diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=True, use_scene_enc=use_scene_enc,
              pred_len=TP)
  cfg = R.default_config(**over)
  assert cfg.scene_grids[0] == (6, 8)
  w = synthetic.make_weights(cfg, 31 + use_scene_enc)
  f = synthetic.make_feeds(cfg, cfg.batch_size, 31 + use_scene_enc)
  tr, margins, (lg, ids, scores) = BT.beam_search(cfg, w, f, 0, TP, torch.device("cpu"))
  assert tr["ids"].shape == (TP, 2, 4) and margins.shape == (TP, 2, 3)
  # the trace is the search's own: its back-trace is what the search returns
  b_ids, b_lg = BT.backtrace(tr["ids"], tr["parents"], tr["logits"], TP)
  assert np.array_equal(b_ids, ids) and np.array_equal(b_lg, lg)
  got = BT.beam_replay(cfg, w, f, 0, tr["ids"], tr["parents"], torch.device("cpu"))
  want = tr["logits"]
  assert got.shape == want.shape
  err = np.abs(got - want).max() / np.abs(want).max()
  print("scene_enc %s: beam_replay vs RT.decoder_beam over %d steps: %.1e" % (use_scene_enc, TP, err))
  assert err <= 1e-12, err
  # beam_scores (the GPU tests' log-probability truth) along the search's own selections gives the search's scores
  for j in range(cfg.batch_size):
    lp, _, bad = BT.beam_scores(cfg, got[:, j], want[:, j], tr["ids"][:, j], tr["parents"][:, j], 0.0)
    assert bad == 0 and np.abs(lp - scores[j]).max() <= 1e-12 * np.abs(scores[j]).max(), (lp, scores[j])
