# coding=utf-8
"""GPU tests of decoding trajectories of different lengths in one batch (ConvRNNEngine.forward(pred_lengths=...)):
every row, unsorted in the batch, is byte-identical to its own N=1 forward at its own length and zero after it; equal
lengths give forward(pred_len=T); every step launches only the rows still running.  The ragged back-trace and the
offset gather are bit-exact against NumPy."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from multiverse_b200 import ops, synthetic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# multifuture_inference.py as TESTING.md runs it (scene 36x64, grid 18x32, emb 32): K = 20 diverse beam, gamma 0.01,
# the first selection's scores zeroed, graph attention, scene encoding
CASES = {
    "k20_diverse": dict(scene_h=36, scene_w=64, use_grids=[True, False], use_beam_search=True, beam_size=20,
                        diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1),
    "k5_plain_nognn": dict(use_grids=[False, True], use_beam_search=True, beam_size=5, use_gnn=False),
    "greedy_two_scale": dict(),
}
# 24 rows, unsorted, repeated lengths, 1 and 2 (no band tracker in a rollout of their own), 26 (the longest future)
LENGTHS = [12, 3, 26, 1, 7, 12, 2, 26, 5, 1, 19, 3, 12, 9, 2, 26, 14, 4, 12, 6, 1, 21, 3, 8]


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _release_memory():
  yield
  gc.collect()
  if torch.cuda.is_available():
    torch.cuda.empty_cache()


def up(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def make_case(name, n, dev, seed=11):
  from multiverse_b200.engine import ConvRNNEngine
  cfg = synthetic.make_config(batch_size=n, **CASES[name])
  w = synthetic.make_weights(cfg, seed)
  f = synthetic.make_feeds(cfg, n, seed)
  feeds = dict(scene_feat=up(f["scene_feat"], dev), obs_scene=up(f["obs_scene"], dev),
               grid_obs_labels=[up(a, dev) for a in f["grid_obs_labels"]],
               grid_obs_regress=[up(a, dev) for a in f["grid_obs_regress"]])
  return cfg, ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev), feeds


def row_feeds(feeds, r):
  """Row r alone (make_feeds gives every trajectory its own frame: frame r)."""
  return dict(scene_feat=feeds["scene_feat"][r:r + 1], obs_scene=torch.zeros_like(feeds["obs_scene"][r:r + 1]),
              grid_obs_labels=[a[r:r + 1] for a in feeds["grid_obs_labels"]],
              grid_obs_regress=[a[r:r + 1] for a in feeds["grid_obs_regress"]])


def host(out):
  """Every fetched output as numpy: (name, index) -> array."""
  res = {}
  for name in ("grid_pred_decoded", "grid_pred_reg_decoded"):
    for i, t in enumerate(out[name]):
      if torch.is_tensor(t):
        res[(name, i)] = t.cpu().numpy()
  if out["beam_outputs"] is not None:
    for j, t in enumerate(out["beam_outputs"]):
      res[("beam_outputs", j)] = t.cpu().numpy()
  return res


def time_axis(key):
  """Axis of the rollout steps in a fetched output without its row axis (None: no step axis)."""
  if key[0] == "beam_outputs":
    return (1, 1, None)[key[1]]
  return 0


def assert_rows_equal_their_own_forward(name, dev, lengths=LENGTHS):
  cfg, eng, feeds = make_case(name, len(lengths), dev)
  batch = host(eng.forward(feeds, pred_lengths=np.array(lengths, dtype=np.int32)))
  tp = max(lengths)
  for r, length in enumerate(lengths):
    alone = host(eng.forward(row_feeds(feeds, r), pred_len=length))
    assert set(alone) == set(batch)
    for key, a in alone.items():
      b = batch[key][r]
      ax = time_axis(key)
      if ax is None:
        assert a[0].tobytes() == b.tobytes(), "row %d (length %d): %s differs" % (r, length, key)
        continue
      assert b.shape[ax] == tp
      head = np.take(b, np.arange(length), axis=ax)
      assert head.dtype == a.dtype and head.tobytes() == np.ascontiguousarray(a[0]).tobytes(), \
          "row %d (length %d): %s differs from its own forward" % (r, length, key)
      tail = np.take(b, np.arange(length, tp), axis=ax)
      assert not tail.any(), "row %d (length %d): %s is not zero after the row's length" % (r, length, key)


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_equal_their_own_forward(name, dev):
  assert_rows_equal_their_own_forward(name, dev)


@pytest.mark.parametrize("name", ["k20_diverse", "k5_plain_nognn"])
def test_rows_equal_their_own_forward_without_bands(name, dev):
  """MVB_BEAM_BAND=0 (every beam row computed at every step), in a process of its own."""
  code = ("import sys; sys.path.insert(0, %r); import torch, test_ragged_decode_gpu as T; "
          "T.assert_rows_equal_their_own_forward(%r, torch.device('cuda:0'))" % (os.path.join(ROOT, "tests"), name))
  env = dict(os.environ, MVB_BEAM_BAND="0")
  r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("name", sorted(CASES))
def test_equal_lengths_are_the_fixed_length_forward(name, dev):
  cfg, eng, feeds = make_case(name, 6, dev)
  a = host(eng.forward(feeds, pred_len=14))
  b = host(eng.forward(feeds, pred_lengths=[14] * 6))
  assert set(a) == set(b)
  for key in a:
    assert a[key].tobytes() == b[key].tobytes(), key


@pytest.mark.parametrize("name", sorted(CASES))
def test_cell_launches_cover_the_running_rows(name, dev):
  """The rows of every decoder cell launch, summed over the rollout, are those of the rows still running."""
  cfg, eng, feeds = make_case(name, len(LENGTHS), dev)
  lens = np.array(LENGTHS)
  act = [int((lens > t).sum()) for t in range(lens.max())]
  eng.cell_events = []
  ops.reset_launch_count()
  eng.forward(feeds, pred_lengths=lens)
  torch.cuda.synchronize()
  rows = {}
  for tag, (_, _, ns), _, _ in eng.cell_events:
    rows[tag] = rows.get(tag, 0) + ns
  eng.cell_events = None
  scales = sum(cfg.use_grids)
  assert rows["dec_reg"] == scales * sum(act)                      # step t: the rows longer than t
  if cfg.use_beam_search:
    k = cfg.beam_size
    assert rows["beam_t0"] == len(lens)                            # time 0: every row, once per sample
    assert rows["beam_fanout"] == act[1]                            # time 1: the parents of the rows longer than 1
    assert rows["beam"] == k * sum(act[2:])                         # time t >= 2: K beams of the rows longer than t
    if "beam_base" in rows:
      assert rows["beam_base"] == sum(act[2:])
  else:
    assert rows["dec_class"] == scales * sum(act)
  assert ops.launch_count() > 0


def test_ragged_backtrace_matches_numpy(dev):
  tp, n, b, v = 26, 512, 20, 576
  rng = np.random.default_rng(3)
  lens = rng.integers(1, tp + 1, size=n).astype(np.int32)
  lens[:4] = (1, 2, tp, tp)
  ids = rng.integers(0, v, size=(tp, n, b)).astype(np.int32)
  par = rng.integers(0, b, size=(tp, n, b)).astype(np.int32)
  logits = rng.standard_normal((tp, n, b, v)).astype(np.float32)
  out_ids = torch.full((n, b, tp), -1, dtype=torch.int32, device=dev)
  out_lg = torch.full((n, b, tp, v), np.nan, dtype=torch.float32, device=dev)
  ops.beam_backtrace_ragged(up(ids, dev), up(par, dev), up(logits, dev), up(lens, dev), out_ids, out_lg)
  got_ids, got_lg = out_ids.cpu().numpy(), out_lg.cpu().numpy()
  want_ids = np.zeros((n, b, tp), np.int32)
  src = np.zeros((n, b, tp), np.int64)
  for i in range(n):
    for k in range(b):
      p = k
      for tau in range(lens[i] - 1, -1, -1):
        src[i, k, tau] = p
        want_ids[i, k, tau] = ids[tau, i, p]
        p = par[tau, i, p]
  tau = np.arange(tp)
  want_lg = logits[tau[None, None, :], np.arange(n)[:, None, None], src]
  want_lg[np.broadcast_to(tau[None, None, :] >= lens[:, None, None], (n, b, tp))] = 0
  assert np.array_equal(got_ids, want_ids)
  assert got_lg.tobytes() == want_lg.tobytes()


def test_gather_offsets_matches_numpy(dev):
  tp, n, k, v = 26, 64, 20, 576
  rng = np.random.default_rng(4)
  lens = rng.integers(1, tp + 1, size=n).astype(np.int32)
  ids = rng.integers(0, v, size=(n, k, tp)).astype(np.int32)
  offs = (rng.standard_normal((tp, n, v, 2)) * 500).astype(np.float32)
  got = ops.gather_offsets(up(ids, dev), up(offs, dev), up(lens, dev)).cpu().numpy()
  want = offs[np.arange(tp)[None, None, :], np.arange(n)[:, None, None], ids]
  want[np.broadcast_to(np.arange(tp)[None, None, :] >= lens[:, None, None], (n, k, tp))] = 0
  assert got.tobytes() == want.tobytes()
