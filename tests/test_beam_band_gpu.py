# coding=utf-8
"""GPU tests of the beam decoder's image-row bands (ops.beam_band, DESIGN.md 3.2): outside its band a beam's c and h
are those of its sample's base rollout, so the beam cell computes only the bands' rows (a work list of M tiles) and the
rest is copied from the base.  That is not an approximation: with the bands on (default) and off (MVB_BEAM_BAND=0),
every beam step's c' and h32 are byte-identical, and so are the final logits, ids, log-probabilities and offsets.
The tracker's bands and work lists equal a NumPy replay of the step's ids and parents."""
import gc

import numpy as np
import pytest
import torch

from multiverse_b200 import ops, synthetic

pytestmark = pytest.mark.gpu

C4 = dict(use_grids=[True, False], use_beam_search=True, beam_size=20, diverse_beam=True, diverse_gamma=0.01,
          fix_num_timestep=1)


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


def make_case(n, dev, seed=7, **over):
  from multiverse_b200.engine import ConvRNNEngine
  cfg = synthetic.make_config(batch_size=n, **dict(C4, **over))
  w = synthetic.make_weights(cfg, seed)
  f = synthetic.make_feeds(cfg, n, seed)
  feeds = dict(scene_feat=up(f["scene_feat"], dev), obs_scene=up(f["obs_scene"], dev),
               grid_obs_labels=[up(a, dev) for a in f["grid_obs_labels"]],
               grid_obs_regress=[up(a, dev) for a in f["grid_obs_regress"]])
  return cfg, ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev), feeds


def band_replay(ids, parents, radius, h, w):
  """NumPy bands of one step: ids, parents [N, K]; returns the new bands [N*K, 2] given the parents' (or None)."""
  def step(band_in):
    k = ids.shape[1]
    y = ids.reshape(-1).astype(np.int64) // w
    lo, hi = y - 2, y + 2
    if band_in is not None:
      p = np.arange(ids.size) // k * k + parents.reshape(-1)
      lo, hi = np.minimum(lo, band_in[p, 0] - radius), np.maximum(hi, band_in[p, 1] + radius)
    return np.stack([np.maximum(lo, 0), np.minimum(hi, h - 1)], 1)
  return step


def tiles_replay(bands, h, w):
  """128-row tiles over the GEMM rows of every band; bands that meet across a sample boundary form one run."""
  s_rows, wp = (h + 1) * (w + 1), w + 1
  runs = []
  for k, (lo, hi) in enumerate(bands.tolist()):
    s = k * s_rows + lo * wp
    e = (k + 1) * s_rows if hi == h - 1 else k * s_rows + (hi + 1) * wp
    if runs and runs[-1][1] == s:
      runs[-1][1] = e
    else:
      runs.append([s, e])
  return np.array([(m0, min(m0 + 128, e)) for s, e in runs for m0 in range(s, e, 128)], dtype=np.int64).reshape(-1, 2)


def rollout(monkeypatch, eng, feeds, band, ns, graph=False, force_ids=None):
  """One forward with the bands on or off.  Returns the outputs and, unless graph, every beam step's c (as the next
  step's cell reads it) and h32 (as the next head reads it), plus the final state buffers."""
  monkeypatch.setenv("MVB_BEAM_BAND", "1" if band else "0")
  steps = []
  real_cell, real_head, real_step = ops.cell_fwd_onehot, ops.head_class_fwd, ops.beam_step
  if not graph:
    def cell(*a, **kw):
      if a[10] == ns:
        steps.append(("c", a[4].clone()))
      return real_cell(*a, **kw)

    def head(*a, **kw):
      if a[9] == ns:
        steps.append(("h", a[0].clone()))
      return real_head(*a, **kw)
    monkeypatch.setattr(ops, "cell_fwd_onehot", cell)
    monkeypatch.setattr(ops, "head_class_fwd", head)
  if force_ids is not None:
    calls = [0]

    def step(logits, s_in, s_out, ids_out, *a, **kw):
      real_step(logits, s_in, s_out, ids_out, *a, **kw)
      ids_out.copy_(force_ids(calls[0], ids_out))
      calls[0] += 1
    monkeypatch.setattr(ops, "beam_step", step)
  if graph:
    eng.forward_graph(feeds)
    out = eng.forward_graph(feeds)
  else:
    out = eng.forward(feeds)
  torch.cuda.synchronize()
  monkeypatch.setattr(ops, "cell_fwd_onehot", real_cell)
  monkeypatch.setattr(ops, "head_class_fwd", real_head)
  monkeypatch.setattr(ops, "beam_step", real_step)
  res = [t.clone() for t in out["beam_outputs"]] + [out["grid_pred_reg_decoded"][0].clone()]
  finals = [eng._bufs[k].clone() for k in sorted(eng._bufs, key=str) if isinstance(k, tuple) and
            k[0] in ("beam_c0", "beam_c1", "beam_h32") and k[1] == ns]
  return res, steps, finals


def assert_band_identical(monkeypatch, n, dev, graph=False, force_ids=None, **over):
  cfg, eng, feeds = make_case(n, dev, **over)
  ns = n * cfg.beam_size
  runs = [rollout(monkeypatch, eng, feeds, band, ns, graph, force_ids) for band in (False, True)]
  (r0, s0, f0), (r1, s1, f1) = runs
  for name, a, b in zip(("logits", "ids", "logprobs", "offsets"), r0, r1):
    assert torch.equal(a, b), "%s differ with the bands on" % name
  assert len(f0) == 3 and all(torch.equal(a, b) for a, b in zip(f0, f1)), "final beam states differ"
  assert [k for k, _ in s0] == [k for k, _ in s1]
  if not graph:
    assert len(s0) == 2 * (cfg.pred_len - 1) - 1
  for j, ((kind, a), (_, b)) in enumerate(zip(s0, s1)):
    assert a.view(torch.int32).equal(b.view(torch.int32)), "%s of record %d differs with the bands on" % (kind, j)
  return cfg, eng, feeds


def test_band_identical_k20_diverse_n16(monkeypatch, dev):
  assert_band_identical(monkeypatch, 16, dev)


def test_band_identical_k20_epilogue_warpgroup_kernel(monkeypatch, dev):
  """96 x 20 beam rows of 36x18: over 64 M tiles per SM, so the beam launch runs cell_fwd_epi_kernel on the list."""
  assert_band_identical(monkeypatch, 96, dev)


def test_band_identical_graph_shard(monkeypatch, dev):
  """The 8-GPU shard of c4 (64 x 20 = 1 280 beam rows) replayed from CUDA graphs."""
  assert_band_identical(monkeypatch, 64, dev, graph=True)


def test_band_identical_k5_plain(monkeypatch, dev):
  assert_band_identical(monkeypatch, 16, dev, beam_size=5, diverse_beam=False, diverse_gamma=1.0, fix_num_timestep=0)


def test_band_identical_without_attention(monkeypatch, dev):
  """use_gnn off: the parents' h is copied into the cell's operands, so a band widens by one row per step."""
  assert_band_identical(monkeypatch, 16, dev, use_gnn=False)


def test_band_identical_native_grid(monkeypatch, dev):
  """The published 36x64 scene: grids 18x32 and 9x16 (beam on the 18x32 one)."""
  assert_band_identical(monkeypatch, 8, dev, scene_h=36, scene_w=64)


@pytest.mark.parametrize("rows", ["first", "last", "alternate"])
def test_band_identical_forced_edge_rows(monkeypatch, dev, rows):
  """Selections forced onto the first or last image row (bands clamped at the grid's edge, runs across sample
  boundaries), or alternating between them (the bands cover the whole image from the second step)."""
  cfg = synthetic.make_config(batch_size=8, **C4)
  h, w = cfg.scene_grids[0]

  def force(call, ids):
    y = {"first": 0, "last": h - 1, "alternate": (h - 1) * (call % 2)}[rows]
    return y * w + ids % w
  assert_band_identical(monkeypatch, 8, dev, force_ids=force)


def test_tracker_matches_numpy(monkeypatch, dev):
  """Every step's bands, work list and tile count against the NumPy replay of its ids and parents, with and without
  the graph attention; the lists cover exactly the bands' valid rows."""
  for over in (dict(), dict(use_gnn=False)):
    cfg, eng, feeds = make_case(24, dev, **over)
    h, w = cfg.scene_grids[0]
    radius = 2 if cfg.use_gnn else 1
    rec = []
    real = ops.beam_band

    def track(ids, parents, band_in, band_out, tiles, tile_count, *a):
      real(ids, parents, band_in, band_out, tiles, tile_count, *a)
      rec.append((ids.clone(), parents.clone(), band_out.clone(), tiles.clone(), tile_count.clone()))
    monkeypatch.setattr(ops, "beam_band", track)
    monkeypatch.setenv("MVB_BEAM_BAND", "1")
    eng.forward(feeds)
    torch.cuda.synchronize()
    monkeypatch.setattr(ops, "beam_band", real)
    assert len(rec) == cfg.pred_len - 1
    prev = None
    for t, (ids, par, bands, tiles, count) in enumerate(rec):
      want = band_replay(ids.cpu().numpy(), par.cpu().numpy(), radius, h, w)(prev)
      assert np.array_equal(bands.cpu().numpy(), want), "bands of step %d" % (t + 1)
      wt = tiles_replay(want, h, w)
      assert int(count.item()) == len(wt), "tile count of step %d" % (t + 1)
      assert np.array_equal(tiles[:len(wt)].cpu().numpy(), wt), "work list of step %d" % (t + 1)
      prev = want
