# coding=utf-8
"""CPU tests of the multi-future evaluation's host side (multiverse_b200.multifuture_eval): the NumPy restatements of
code/multifuture_eval_trajs.py and code/multifuture_eval_trajs_prob.py print exactly what the unmodified scripts
printed on the golden set (tests/golden/multifuture_eval.npz); the module's packing of the ground truth and its
concatenation of per-future results, fed per-future values computed here, print the trajs script's lines byte for
byte and the prob script's counts exactly and NLL to 1e-6."""
import os

import numpy as np
import pytest

import multifuture_eval_ref as ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multifuture_eval.npz")


@pytest.fixture(scope="module")
def golden(tmp_path_factory):
  d = dict(np.load(GOLD))
  gt_dir, pred_file, prob_file = ref.golden_pickles(d, str(tmp_path_factory.mktemp("mfe")))
  import pickle
  with open(pred_file, "rb") as f:
    pred = pickle.load(f)
  with open(prob_file, "rb") as f:
    prob = pickle.load(f)
  return d, ref.load_gts(gt_dir, list(pred)), pred, prob


def test_golden_set_covers_the_cases(golden):
  d, gts, _, _ = golden
  cams = [str(t).split("_")[-1] for t in d["traj_ids"]]
  assert "cam4" in cams and len(set(cams)) == 4
  assert d["g_count"].min() == 1 and d["g_count"].max() == 15
  assert (d["gt_len"][d["gt_len"] > 0] == 1).any()
  assert all(d["gt_len"][n].max() == d["lengths"][n] for n in range(len(cams)))
  pts = d["gt"][:, :, :5][np.arange(5) < d["gt_len"][..., None]]
  assert (pts == 0).any() and (pts < 0).any() and ((pts > -1) & (pts < 0)).any()
  assert (pts[:, 0] % 60 == 0).any() and (pts[:, 1] == 1080).any()


def test_restatements_print_the_scripts_stdout(golden):
  d, gts, pred, prob = golden
  assert ref.trajs_stdout(pred, gts) == str(d["stdout_trajs"])
  assert ref.prob_stdout(prob, gts) == str(d["stdout_prob"])
  rows = ref.nll_rows(prob, gts)
  for j in range(5):
    assert np.array_equal(np.array(rows["T=%d" % (j + 1)]), d["nll"][d["count"][:, j] > 0, j])


def left_to_right_min(points, lengths, gt, gt_len):
  """Per (trajectory, future): the min-ADE prediction's per-step errors and the min FDE, with left-to-right sums."""
  n, g, tg, _ = gt.shape
  ade = np.zeros((n, g, tg))
  fde = np.zeros((n, g))
  for i in range(n):
    for j in range(g):
      ln = gt_len[i, j]
      if ln == 0:
        continue
      assert ln <= lengths[i]
      sq = (gt[i, j, None, :ln] - points[i, :, :ln]) ** 2
      err = np.sqrt(sq[..., 0] + sq[..., 1])
      tot = np.zeros(err.shape[0])
      for t in range(ln):
        tot = tot + err[:, t]
      ade[i, j, :ln] = err[tot.argmin()]
      fde[i, j] = err[:, ln - 1].min()
  return ade, fde


def test_scores_concatenate_in_the_scripts_order(golden):
  from multiverse_b200 import multifuture_eval as mfe
  d, gts, pred, prob = golden
  ids = [str(t) for t in d["traj_ids"]]
  scores = mfe.Scores()
  for c0 in (0, 17, 31):                       # batches of unequal size
    rows = ids[c0:{0: 17, 17: 31, 31: len(ids)}[c0]]
    gt, gt_len = mfe.pack_gt([gts[t] for t in rows])
    sl = slice(c0, c0 + len(rows))
    ade, fde = left_to_right_min(d["points"][sl], d["lengths"][sl], gt, gt_len)
    scores.add_trajectories(rows, ade, fde, gt_len)
  assert "\n".join(scores.trajectory_lines()) + "\n" == str(d["stdout_trajs"])
  scores.add_nll(d["nll"][:20], d["count"][:20])
  scores.add_nll(d["nll"][20:], d["count"][20:])
  got, want = scores.nll_lines(), str(d["stdout_prob"]).splitlines()
  assert got[:3] == want[:3]
  assert np.allclose(np.array(got[3].split(), float), np.array(want[3].split(), float), rtol=1e-6, atol=0)


def test_pack_gt_keeps_the_dict_order():
  from multiverse_b200 import multifuture_eval as mfe
  gts = [{"b": {"x_agent_traj": [[0, 1, 2.5, 3], [1, 1, 0, 0]]}, "a": {"x_agent_traj": [[0, 1, 7, 8.25]]}}, {}]
  gt, gt_len = mfe.pack_gt(gts)
  assert gt.dtype == np.float64 and gt.shape == (2, 2, 2, 2) and gt_len.tolist() == [[2, 1], [0, 0]]
  assert gt[0, 0].tolist() == [[2.5, 3.0], [0.0, 0.0]] and gt[0, 1, 0].tolist() == [7.0, 8.25]


def test_cell_restatement_wraps_and_refuses_like_numpy():
  assert ref.cell_of([0.0, 0.0], 18, 32, 1080, 1920) == 0
  assert ref.cell_of([60.0, 60.0], 18, 32, 1080, 1920) == 0                 # ceil(1) - 1: the cell below the line
  assert ref.cell_of([60.000001, 1080.0], 18, 32, 1080, 1920) == 17 * 32 + 1
  assert ref.cell_of([-61.0, 0.0], 18, 32, 1080, 1920) == 30                 # -2 wraps
  with pytest.raises(IndexError):
    ref.cell_of([1920.5, 0.0], 18, 32, 1080, 1920)


def test_eval_flag_is_split_off():
  from multiverse_b200 import multifuture
  assert multifuture.split_eval(["s.py", "a", "--eval", "--batch_size", "8"]) == (["s.py", "a", "--batch_size", "8"],
                                                                                 True)
  assert multifuture.split_eval(["s.py", "a"]) == (["s.py", "a"], False)
