# coding=utf-8
"""GPU tests of the multi-future evaluation on the device (multiverse_b200.multifuture_eval and its kernels):
  - mvb_min_ade_fde_cells at N 512, K 20, up to 15 futures of ragged lengths, beam / center_only / greedy K = 1:
    errors, minima and indices bit-exact against a NumPy restatement (centre + offset in fp64, left-to-right sums,
    first index on ties);
  - mvb_points_to_cells bit-exact against xys_to_indexes restated per point, cell boundaries, 0 and wrapped negative
    indices included; an index numpy refuses raises IndexError;
  - the ragged NLL within 1e-5 of the prob script's own per-trajectory NLL on the golden set, and bit-identical to
    mvb_beam_nll when every row has the same length;
  - both command lines print the golden stdout of the unmodified scripts (ADE/FDE byte for byte, NLL to 1e-6);
  - `multifuture --eval` (infer with an Evaluation) prints what infer's pickles give through the restated scripts,
    for a K = 20 diverse beam with graph attention and for greedy, without copying a beam-logit tensor to the host."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import multifuture_eval_ref as ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "multifuture_eval.npz")


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def up(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def ref_min_ade_fde_cells(ids, offs, centers, gt, gt_len, center_only):
  """The trajs script's selection on the points multifuture_inference.py forms (fp64 centre + fp32 offset):
  per-step errors with both squares rounded before the add, left-to-right sums, first index on ties."""
  pts = centers[ids] if center_only else centers[ids] + offs.astype(np.float64)     # [N,K,Tp,2]
  tg = gt.shape[2]
  diff = gt[:, :, None] - pts[:, None, :, :tg]                                        # [N,G,K,Tg,2]
  sq = diff ** 2
  d = np.sqrt(sq[..., 0] + sq[..., 1])
  ln = gt_len[:, :, None]
  tot = np.zeros(d.shape[:3])
  for t in range(tg):
    tot = np.where(t < ln, tot + d[..., t], tot)
  last = np.take_along_axis(d, np.maximum(ln - 1, 0)[..., None], -1)[..., 0]
  ade_idx, fde_idx = tot.argmin(-1), last.argmin(-1)
  ade_err = np.take_along_axis(d, ade_idx[:, :, None, None], 2)[:, :, 0] * (np.arange(tg) < gt_len[..., None])
  fde = np.take_along_axis(last, fde_idx[..., None], -1)[..., 0]
  none = gt_len == 0
  ade_idx[none], fde_idx[none], fde[none] = -1, -1, 0.0
  return ade_err, ade_idx.astype(np.int32), fde, fde_idx.astype(np.int32)


def at_size_case(k, seed):
  """512 trajectories of lengths 1..26, up to 15 futures each (lengths 1..the row's, absent ones 0), on the 18x32
  grid over 1920x1080; futures near one prediction, duplicated predictions, coordinates of unlike magnitude."""
  rng = np.random.default_rng(seed)
  n, tp, h, w = 512, 26, 18, 32
  centers = np.stack(np.meshgrid((np.arange(w) + 0.5) * 60.0, (np.arange(h) + 0.5) * 60.0), -1).reshape(-1, 2)
  lengths = rng.integers(1, tp + 1, n).astype(np.int32)
  lengths[0] = tp
  ids = rng.integers(0, h * w, (n, k, tp)).astype(np.int32)
  offs = rng.normal(0, 25, (n, k, tp, 2)).astype(np.float32)
  offs[::7, :, :, 1] = rng.uniform(-1e-3, 1e-3, offs[::7, :, :, 1].shape)
  if k > 4:
    ids[::3, 4], offs[::3, 4] = ids[::3, 1], offs[::3, 1]                 # duplicates: index 1 must win
  gg = 15
  gt_len = np.zeros((n, gg), np.int32)
  for r in range(n):
    c = rng.integers(1, gg + 1)
    gt_len[r, :c] = rng.integers(1, lengths[r] + 1, c)
  pts = centers[ids] + offs.astype(np.float64)
  near = rng.integers(0, k, (n, gg))
  gt = np.take_along_axis(pts, near[:, :, None, None], 1) + rng.normal(0, 3, (n, gg, tp, 2))
  if k > 4:
    gt[::3, 0] = pts[::3, 1] + rng.normal(0, 0.01, (len(gt[::3]), tp, 2))
  gt[np.arange(tp) >= gt_len[..., None]] = 0.0
  return ids, offs, centers, lengths, gt, gt_len


@pytest.mark.parametrize("mode", ["beam", "center_only", "greedy"])
def test_min_ade_fde_cells_at_size(dev, mode):
  from multiverse_b200 import ops
  k = 1 if mode == "greedy" else 20
  ids, offs, centers, lengths, gt, gt_len = at_size_case(k, 900 + k)
  center_only = mode == "center_only"
  want = ref_min_ade_fde_cells(ids, offs, centers, gt, gt_len, center_only)
  got = ops.min_ade_fde_cells(up(ids, dev), up(offs, dev), up(centers, dev), up(lengths, dev), up(gt, dev),
                              up(gt_len, dev), center_only)
  assert int(got[4].item()) == 0
  got = [a.cpu().numpy() for a in got[:4]]
  names = ("ade_err", "ade_idx", "fde", "fde_idx")
  diff = {nm: int((a != b).sum()) for nm, a, b in zip(names, got, want)}
  print("min_ade_fde_cells %s: %d futures, elements that differ from numpy %s" % (mode, int((gt_len > 0).sum()),
                                                                                  diff))
  for nm, a, b in zip(names, got, want):
    assert np.array_equal(a, b), (nm, diff[nm])
  if k > 4:
    assert (want[1][::3, 0] == 1).mean() > 0.9
  if mode == "greedy":
    assert set(np.unique(got[1])) <= {-1, 0}


def test_min_ade_fde_cells_refuses_a_future_longer_than_its_predictions(dev):
  from multiverse_b200 import multifuture_eval as mfe
  ids, offs, centers, lengths, gt, gt_len = at_size_case(20, 5)
  r = int(np.argmin(lengths))
  gt_len[r, 0] = lengths[r] + 1
  with pytest.raises(AssertionError):
    mfe.score_trajectories(up(ids, dev), up(offs, dev), up(centers, dev), up(lengths, dev), up(gt, dev),
                           up(gt_len, dev))


def test_points_to_cells_bit_exact(dev):
  from multiverse_b200 import multifuture_eval as mfe, ops
  rng = np.random.default_rng(3)
  pts = rng.uniform([-119.0, -59.0], [1920.0, 1080.0], (20000, 2))
  bx, by = np.meshgrid(np.arange(-1, 33) * 60.0, np.arange(-1, 19) * 60.0)
  edge = np.stack([bx.ravel(), by.ravel()], -1)
  special = np.array([[0.0, 0.0], [-0.0, -0.0], [-1e-300, 5e-324], [-0.5, -59.99], [-60.0, -60.0], [-61.0, 1080.0],
                      [1920.0, 0.0], [np.nextafter(60.0, 0), np.nextafter(60.0, 100)], [1919.9999999999998, 1.0]])
  pts = np.concatenate([pts, edge, special])
  want = np.array([ref.cell_of(p, 18, 32, 1080, 1920) for p in pts], np.int32)
  cells, err = ops.points_to_cells(up(pts, dev), 18, 32, 1080, 1920)
  assert int(err.item()) == 0
  got = cells.cpu().numpy()
  print("points_to_cells: %d points, %d differ" % (len(pts), int((got != want).sum())))
  assert np.array_equal(got, want)
  assert (want[-len(special):-3] >= 0).all() and want[-4] == 17 * 32 + 30
  for bad in ([1920.5, 0.0], [0.0, 1140.5], [-1921.0, 0.0], [np.nan, 0.0]):
    cells, err = ops.points_to_cells(up(np.array([[1.0, 1.0], bad]), dev), 18, 32, 1080, 1920)
    assert int(err.item()) == 1 and cells.cpu().tolist() == [0, -1]
  gt = np.zeros((1, 1, 5, 2))
  gt[0, 0, 2] = [1920.5, 3.0]
  logits = torch.zeros((1, 2, 5, 576), device=dev)
  with pytest.raises(IndexError):
    mfe.score_nll(logits, torch.zeros((1, 2), device=dev), up(np.array([5], np.int32), dev), up(gt, dev),
                  up(np.array([[5]], np.int32), dev), 18, 32)


def golden_device(dev):
  d = dict(np.load(GOLD))
  logits = ref.golden_logits(d)
  return d, up(logits, dev), up(d["logprobs"], dev), up(d["lengths"], dev)


def test_ragged_nll_matches_the_scripts_per_trajectory_nll(dev, tmp_path):
  from multiverse_b200 import multifuture_eval as mfe
  d, logits, logprobs, lengths = golden_device(dev)
  gt_dir, _, _ = ref.golden_pickles(d, str(tmp_path))
  ids = [str(t) for t in d["traj_ids"]]
  gt, gt_len = mfe.pack_gt([ref.load_gts(gt_dir, ids)[t] for t in ids])
  nll, cnt = mfe.score_nll(logits, logprobs, lengths, up(gt, dev), up(gt_len, dev), 18, 32)
  nll, cnt = nll.cpu().numpy(), cnt.cpu().numpy()
  assert np.array_equal(cnt, d["count"])
  err = float(np.abs(nll - d["nll"]).max())
  print("ragged NLL vs the script's per-trajectory NLL: max |diff| %.3e" % err)
  assert err < 1e-5
  with pytest.raises(IndexError):
    mfe.score_nll(logits, logprobs, torch.clamp(lengths, max=4), up(gt, dev), up(gt_len, dev), 18, 32)


def test_ragged_nll_with_equal_lengths_is_beam_nll(dev):
  from multiverse_b200 import ops
  g = torch.Generator(device=dev)
  g.manual_seed(8)
  n, k, tp, v = 256, 20, 12, 576
  logits = torch.randn((n, k, tp, v), generator=g, device=dev) * 3
  logprobs = -torch.randn((n, k), generator=g, device=dev).abs() * 4
  steps = torch.arange(5, dtype=torch.int32, device=dev)
  gt_idx = torch.randint(-1, v, (n, 5, 15), generator=g, device=dev, dtype=torch.int32)
  want = ops.beam_nll(logits, logprobs, gt_idx, steps)
  got = ops.beam_nll_ragged(logits, logprobs, torch.full((n,), tp, dtype=torch.int32, device=dev), gt_idx, steps)
  assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def run_cli(*args):
  r = subprocess.run([sys.executable, "-m", "multiverse_b200.multifuture_eval"] + list(args), cwd=ROOT,
                     capture_output=True, text=True)
  assert r.returncode == 0, r.stderr
  return r.stdout


def test_command_lines_print_the_golden_stdout(dev, tmp_path):
  d = dict(np.load(GOLD))
  gt_dir, pred_file, prob_file = ref.golden_pickles(d, str(tmp_path))
  assert run_cli("trajs", gt_dir, pred_file) == str(d["stdout_trajs"])
  got, want = run_cli("prob", gt_dir, prob_file).splitlines(), str(d["stdout_prob"]).splitlines()
  assert got[:3] == want[:3]
  a, b = np.array(got[3].split(), float), np.array(want[3].split(), float)
  print("prob command line: NLL max |diff| from the script's %.3e" % float(np.abs(a - b).max()))
  assert np.all(np.abs(a - b) <= 1e-6)


def synthetic_gt(lengths, seed):
  rng = np.random.default_rng(seed)
  out = []
  for r, ln in enumerate(lengths):
    c = int(rng.integers(1, 16))
    gl = rng.integers(1, ln + 1, c)
    gl[0] = ln
    pts = rng.uniform([-30.0, -30.0], [1920.0, 1080.0], (c, ln, 2))
    out.append(ref.gt_dict(pts, gl, r))
  return out


@pytest.mark.parametrize("case", ["k20_diverse", "greedy"])
def test_eval_equals_the_pickle_path(dev, case, monkeypatch):
  from test_multifuture_gpu import K20, make_model, script_feeds
  from multiverse_b200 import multifuture, multifuture_eval as mfe, synthetic
  over = dict(K20) if case != "greedy" else dict(K20, use_beam_search=False, beam_size=1, diverse_beam=False)
  n = 40
  tf, cfg, model = make_model(monkeypatch, over, 33)
  feeds = script_feeds(model, cfg, n, 33)
  traj_ids = ["%04d_%d_%d_cam%d" % (r, r + 3, r + 7, 1 + r % 4) for r in range(n)]
  lengths = [int(fd[model.pred_length][0]) for fd in feeds]
  gts = dict(zip(traj_ids, synthetic_gt(lengths, 34)))
  gi = cfg.use_grids.index(True)
  args = types.SimpleNamespace(scene_grid_centers=synthetic.grid_centers(cfg), num_out=20, center_only=False,
                               video_h=1080, video_w=1920)
  evaluation = multifuture.make_evaluation(model, args, gts)
  v = cfg.scene_grids[gi][0] * cfg.scene_grids[gi][1]
  fetched = []
  cpu, to = torch.Tensor.cpu, torch.Tensor.to

  def spy_cpu(t, *a, **kw):
    fetched.append(tuple(t.shape))
    return cpu(t, *a, **kw)

  def spy_to(t, *a, **kw):
    out = to(t, *a, **kw)
    if t.is_cuda and not out.is_cuda:
      fetched.append(tuple(t.shape))
    return out

  monkeypatch.setattr(torch.Tensor, "cpu", spy_cpu)
  monkeypatch.setattr(torch.Tensor, "to", spy_to)
  got = multifuture.infer(model, feeds, 16, args, traj_ids, evaluation=evaluation)
  monkeypatch.setattr(torch.Tensor, "cpu", cpu)
  monkeypatch.setattr(torch.Tensor, "to", to)
  assert not [s for s in fetched if len(s) == 4 and s[-1] == v], fetched
  output_data, beam_prob = multifuture.infer(model, feeds, 16, args, traj_ids, with_prob=cfg.use_beam_search)
  assert got[0].keys() == output_data.keys()
  lines = evaluation.lines()
  assert "\n".join(lines[:3]) + "\n" == ref.trajs_stdout(output_data, gts)
  if not cfg.use_beam_search:
    assert len(lines) == 3
    return
  want = ref.prob_stdout(beam_prob, gts, cfg.scene_grids[gi][0], cfg.scene_grids[gi][1]).splitlines()
  assert lines[3:6] == want[:3]
  a, b = np.array(lines[6].split(), float), np.array(want[3].split(), float)
  print("--eval NLL max |diff| from the restated script %.3e" % float(np.abs(a - b).max()))
  assert np.all(np.abs(a - b) <= 1e-6 * np.abs(b))
