# coding=utf-8
"""The multi-future decode against the fp64 truth at the configuration code/multifuture_inference.py runs (TESTING.md:
scene 36x64, so the beam runs on the 18x32 grid; --emb_size 32, --use_scene_enc, --use_gnn; K = 20 diverse beam, gamma
0.01, fix_num_timestep 1): one trajectory per forward, each decoded to its own length (up to 26 steps), ragged batches
and multifuture.infer end to end.  The truths (tests/beam_truth.py) run in fp64 on the device.

- Beam logits: every live beam row at every step within BAR of the fp64 replay along the engine's own selections
  (max |diff| / max |truth| per step); the returned beam outputs are the back-trace of that trace.
- Log-probabilities: within BAR of the fp64 sums along each beam's path (log-softmax of the truth's logits plus
  log(gamma) x the rank in the parent's row, scores zeroed up to fix_num_timestep).  Where the truth's rank of a
  selected cell lies within the engine's logit error of a tie, either rank is admitted (counted and printed).
- Ids: the selections (cells and parents) equal the fp64 beam search's own, in its order, at every step before its
  first selection within 2e-4 of a tie (the rule of test_emb_size_gpu.test_rollout_beam_against_reference_execution,
  plus the diverse penalty's in-row rank: beam_truth.beam_search's margins), and the returned ids equal its ids for
  every rollout with no such selection; the others are reported.
- Offsets (regression decoder): within BAR of fp64.
The worst error of every step t = 1..26 is printed (pytest -s)."""
import gc
import types

import numpy as np
import pytest
import torch

import beam_truth as BT
from test_beam_no_gnn_gpu import rel, to_dev
from test_multifuture_gpu import K20

pytestmark = pytest.mark.gpu
BAR = 1e-4
TMAX = 26                                   # the longest future multifuture_inference.py decodes
LENGTHS = [26, 20, 12, 3, 2, 1]
SEEDS = [601, 602, 603, 604]
TIE = 2e-4                                  # selection margin below which the truth's ids are not asserted
# 12 rows, unsorted: lengths 1, 2 and 26, repeats, both parities
RAGGED = [12, 1, 26, 3, 2, 20, 7, 26, 2, 15, 1, 12]


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


def config(n, **over):
  from multiverse_b200 import synthetic
  return synthetic.make_config(batch_size=n, pred_len=TMAX, **dict(K20, **over))


def engine(cfg, w, dev):
  from multiverse_b200.engine import ConvRNNEngine
  return ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev)


def traced_forward(eng, feeds, **kw):
  """eng.forward(feeds, **kw) and the per-step trace of decode_class_beam (cells, parents and logits of every step;
  rows in the order the engine runs them)."""
  trace, beam = [], eng.decode_class_beam

  def traced(*a, **k):
    r = beam(*a, **k)
    trace.append({name: v.cpu().numpy() for name, v in r[3].items()})
    return r
  eng.decode_class_beam = traced
  try:
    out = eng.forward(feeds, **kw)
    torch.cuda.synchronize()
  finally:
    del eng.decode_class_beam
  return out, (trace[0] if trace else None)


class Curve(object):
  """Worst error per step t = 1..TMAX over the cases of a test ("-": no case measured at that step)."""

  def __init__(self, *names):
    self.v = {k: np.full(TMAX, np.nan) for k in names}

  def add(self, name, errs, at=0):
    v = self.v[name][at:at + len(errs)]
    v[:] = np.fmax(v, errs)

  def show(self, title):
    print("\n%s: worst error per step t = 1..%d" % (title, TMAX))
    for k, v in self.v.items():
      print("  %-8s %s" % (k, " ".join("-" if np.isnan(x) else "%.1e" % x for x in v)))
      print("  %-8s max t<=20 %.2e, t>20 %.2e" % ("", np.nanmax(v[:20]), np.nanmax(v[20:])))


def per_step(got, want):
  """rel of every step of [T, ...] arrays."""
  return np.array([rel(got[t], want[t]) for t in range(len(want))])


def check_sample(cfg, length, tr, truth, bo, tag):
  """One sample of a beam decode of `length` steps: tr ids / parents [T,K] and logits [T,K,V] of its trace (T >=
  length), truth [length,K,V] the fp64 replay along it, bo = (logits [K,Tmax,V], ids [K,Tmax], log-probabilities [K])
  as forward returns them for this sample.  Returns (per-step logit errors, log-probability error, ambiguous ranks)."""
  ids, par, lgt = tr["ids"][:length], tr["parents"][:length], tr["logits"][:length]
  errs = per_step(lgt, truth)
  assert errs.max() < BAR, "%s: logits along the engine's selections %s" % (tag, errs)
  blg, bids, blp = bo
  want_ids, want_lg = BT.backtrace(ids[:, None], par[:, None], lgt[:, None], length)
  assert np.array_equal(bids[:, :length], want_ids[0]), "%s: ids are not the back-trace of the trace" % tag
  assert np.array_equal(blg[:, :length], want_lg[0]), "%s: logits are not the back-trace of the trace" % tag
  assert not bids[:, length:].any() and not blg[:, length:].any(), "%s: outputs after the length" % tag
  lp, amb, bad = BT.beam_scores(cfg, truth, lgt, ids, par, float(np.abs(blp).max()))
  assert bad == 0, "%s: %d ranks outside the truth's admissible range" % (tag, bad)
  lp_err = rel(blp, lp) if np.abs(lp).max() > 0 else float(np.abs(blp).max())
  assert lp_err < BAR, "%s: log-probabilities %s vs fp64 %s" % (tag, blp, lp)
  return errs, lp_err, amb, lp


# --------------------------------------------------------------------------- N = 1, every length
@pytest.fixture(scope="module")
def n1(dev):
  """Per seed: config, weights, feeds of one trajectory, its engine, the fp64 beam search over 26 steps and the fp64
  offsets; replays along engine traces are cached (a replay of T steps holds every shorter one along the same
  selections)."""
  from multiverse_b200 import synthetic
  cfg = config(1)
  cases = {}
  for seed in SEEDS:
    w, f = synthetic.make_weights(cfg, seed), synthetic.make_feeds(cfg, 1, seed)
    tr, margins, _ = BT.beam_search(cfg, w, f, 0, TMAX, dev)
    cases[seed] = types.SimpleNamespace(
        cfg=cfg, w=w, f=f, feeds=to_dev(f, dev), eng=engine(cfg, w, dev), beam=tr, margins=margins,
        reg=BT.reg_truth(cfg, w, f["grid_obs_regress"][0], 0, TMAX, dev), replays=[])
  return cases


def replay(case, tr, length, dev):
  ids, par = tr["ids"][:length], tr["parents"][:length]
  for r_ids, r_par, r_lg in case.replays:
    if len(r_lg) >= length and np.array_equal(r_ids[:length - 1], ids[:length - 1]) and \
        np.array_equal(r_par[:length - 1], par[:length - 1]):
      return r_lg[:length]
  lg = BT.beam_replay(case.cfg, case.w, case.f, 0, ids, par, dev)
  case.replays.append((ids, par, lg))
  return lg[:length]


@pytest.mark.parametrize("band", ["1", "0"], ids=["bands", "no_bands"])
def test_n1_beam_against_fp64_at_every_length(dev, n1, monkeypatch, band):
  """N = 1 per forward (the script's loop), lengths 1, 2, 3, 12, 20, 26, four seeds, with and without the image-row
  bands (MVB_BEAM_BAND)."""
  monkeypatch.setenv("MVB_BEAM_BAND", band)
  curve = Curve("logits", "offsets", "logprob")
  clear, report = 0, []
  amb_total = 0
  for seed, case in n1.items():
    for length in LENGTHS:
      tag = "seed %d length %d bands %s" % (seed, length, band)
      out, tr = traced_forward(case.eng, case.feeds, pred_len=length)
      tr = {k: v[:, 0] for k, v in tr.items()}
      truth = replay(case, tr, length, dev)[:, 0]
      bo = [t[0].cpu().numpy() for t in out["beam_outputs"]]
      errs, lp_err, amb, _ = check_sample(case.cfg, length, tr, truth, bo, tag)
      amb_total += amb
      curve.add("logits", errs)
      curve.add("logprob", [lp_err], at=length - 1)    # after the last selection
      off = per_step(out["grid_pred_reg_decoded"][0][0].cpu().numpy(), case.reg[0, :length])
      assert off.max() < BAR, "%s: offsets %s" % (tag, off)
      curve.add("offsets", off)
      # the fp64 search's own selections, in its order, at every step before its first one near a tie; its ids
      # where none is
      gap = case.margins[:length, 0].min(-1)
      first = int(np.argmax(gap <= TIE)) if (gap <= TIE).any() else length
      for k in ("ids", "parents"):
        assert np.array_equal(tr[k][:first], case.beam[k][:first, 0]), \
            "%s: %s differ from the fp64 beam search's before its first selection near a tie (time %d)" % (
                tag, k, first + 1)
      want, _ = BT.backtrace(case.beam["ids"], case.beam["parents"], case.beam["logits"], length)
      if first == length:
        clear += 1
        assert np.array_equal(bo[1][:, :length], want[0]), "%s: ids differ from the fp64 beam search's" % tag
      elif length == TMAX:
        shared = len(set(map(tuple, bo[1].tolist())) & set(map(tuple, want[0].tolist())))
        report.append("seed %d: first selection near a tie at time %d (gap %.1e), %d of %d id sequences shared "
                      "at 26 steps" % (seed, first + 1, gap[first], shared, case.cfg.beam_size))
  curve.show("N=1 K=20 diverse beam on 18x32, bands %s (%d runs)" % (band, len(n1) * len(LENGTHS)))
  print("  ids equal the fp64 search's in %d of %d runs clear of ties; ranks within the logit error of a tie: %d"
        % (clear, len(n1) * len(LENGTHS), amb_total))
  print("  " + ("\n  ".join(report) or "no seed near a tie"))


def test_n1_greedy_against_fp64_at_every_length(dev):
  """--greedy at N = 1 on 18x32: the fp64 class decoder fed the engine's own arg-max ids; ids equal the truth's
  arg-max wherever its top-2 gap exceeds 1e-4 x max|logit| (and that holds on at least 90 % of the steps); logits and
  offsets within BAR."""
  from multiverse_b200 import synthetic
  cfg = config(1, use_beam_search=False, beam_size=1, diverse_beam=False)
  curve = Curve("logits", "offsets")
  h, w_ = cfg.scene_grids[0]
  n_clear = n_steps = 0
  for seed in SEEDS:
    w, f = synthetic.make_weights(cfg, seed), synthetic.make_feeds(cfg, 1, seed)
    eng, feeds = engine(cfg, w, dev), to_dev(f, dev)
    reg = BT.reg_truth(cfg, w, f["grid_obs_regress"][0], 0, TMAX, dev)
    for length in LENGTHS:
      tag = "greedy seed %d length %d" % (seed, length)
      out = eng.forward(feeds, pred_len=length)
      lg = out["grid_pred_decoded"][0].cpu().numpy().reshape(length, h * w_)
      ids = lg.argmax(-1)
      truth = BT.greedy_replay(cfg, w, f, 0, ids[None], dev)[0]
      errs = per_step(lg, truth)
      assert errs.max() < BAR, "%s: logits %s" % (tag, errs)
      srt = np.sort(truth, -1)
      clear = srt[:, -1] - srt[:, -2] > 1e-4 * np.abs(truth).max()
      assert (ids == truth.argmax(-1))[clear].all(), "%s: ids differ from the fp64 arg-max" % tag
      n_clear += int(clear.sum())
      n_steps += length
      off = per_step(out["grid_pred_reg_decoded"][0][0].cpu().numpy(), reg[0, :length])
      assert off.max() < BAR, "%s: offsets %s" % (tag, off)
      curve.add("logits", errs)
      curve.add("offsets", off)
    del eng
  curve.show("N=1 greedy on 18x32")
  print("  steps whose fp64 top-2 gap clears 1e-4 x max|logit|: %d of %d" % (n_clear, n_steps))
  assert n_clear >= 0.9 * n_steps


# --------------------------------------------------------------------------- ragged batch
def row_feeds(f, r):
  """Row r of make_feeds' output alone (every trajectory has its own frame: frame r)."""
  return dict(scene_feat=f["scene_feat"][r:r + 1], obs_scene=np.zeros_like(f["obs_scene"][r:r + 1]),
              grid_obs_labels=[a[r:r + 1] for a in f["grid_obs_labels"]],
              grid_obs_regress=[a[r:r + 1] for a in f["grid_obs_regress"]])


@pytest.mark.parametrize("band", ["1", "0"], ids=["bands", "no_bands"])
def test_ragged_batch_against_fp64(dev, monkeypatch, band):
  """forward(pred_lengths=RAGGED): every row against its own fp64 truth at its own length - logits along its own
  trace, back-trace, offsets, log-probabilities (read from its own last selection's score buffer, both parities of
  the length), zeros after the length - and ops.beam_nll_ragged on the output against the NLL formed in fp64 from the
  truth's logits and log-probabilities along the same selections."""
  from multiverse_b200 import ops, synthetic
  monkeypatch.setenv("MVB_BEAM_BAND", band)
  lens = np.array(RAGGED)
  n = len(lens)
  cfg, cfg1 = config(n), config(1)
  w, f = synthetic.make_weights(cfg, 611), synthetic.make_feeds(cfg, n, 611)
  eng = engine(cfg, w, dev)
  out, tr = traced_forward(eng, to_dev(f, dev), pred_lengths=lens.astype(np.int32))
  pos = np.argsort(np.argsort(-lens, kind="stable"))         # row i runs at position pos[i]
  bo = [t.cpu().numpy() for t in out["beam_outputs"]]
  reg = BT.reg_truth(cfg, w, f["grid_obs_regress"][0], 0, TMAX, dev)
  reg_e = out["grid_pred_reg_decoded"][0].cpu().numpy()
  curve = Curve("logits", "offsets", "logprob")
  truth_lg, truth_lp, amb_total = [], [], 0
  for i, length in enumerate(lens):
    tag = "row %d (length %d, bands %s)" % (i, length, band)
    rt = {k: v[:, pos[i]] for k, v in tr.items()}
    truth = BT.beam_replay(cfg1, w, row_feeds(f, i), 0, rt["ids"][:length, None], rt["parents"][:length, None],
                           dev)[:, 0]
    errs, lp_err, amb, lp = check_sample(cfg, length, rt, truth, [b[i] for b in bo], tag)
    amb_total += amb
    curve.add("logits", errs)
    curve.add("logprob", [lp_err], at=length - 1)    # after the last selection
    off = per_step(reg_e[i, :length], reg[i, :length])
    assert off.max() < BAR, "%s: offsets %s" % (tag, off)
    assert not reg_e[i, length:].any(), "%s: offsets after the length" % tag
    curve.add("offsets", off)
    truth_lg.append(BT.backtrace(rt["ids"][:length, None], rt["parents"][:length, None], truth[:, None],
                                 length)[1][0])
    truth_lp.append(lp)
  curve.show("ragged K=20 batch of %d rows, lengths %s, bands %s" % (n, RAGGED, band))
  print("  ranks within the logit error of a tie: %d" % amb_total)
  # NLL at T = 1..5 of ground-truth cells (absent ones -1) under the beam mixture
  v = cfg.scene_grids[0][0] * cfg.scene_grids[0][1]
  rng = np.random.default_rng(612)
  gt = rng.integers(0, v, size=(n, 5, 3)).astype(np.int32)
  gt[rng.random(gt.shape) < 0.3] = -1
  gt[:, :, 0] = np.abs(gt[:, :, 0])
  steps = np.arange(5, dtype=np.int32)
  nll, cnt = ops.beam_nll_ragged(out["beam_outputs"][0], out["beam_outputs"][2], out["_lengths"],
                                 torch.from_numpy(gt).to(dev), torch.from_numpy(steps).to(dev))
  nll, cnt = nll.cpu().numpy(), cnt.cpu().numpy()
  eps = np.finfo(float).eps
  worst = 0.0
  for i, length in enumerate(lens):
    lp = truth_lp[i]
    wk = np.exp(lp - lp.max())
    wk /= wk.sum()
    for j, s in enumerate(steps):
      cells = gt[i, j][gt[i, j] >= 0]
      if s >= length:
        assert cnt[i, j] == 0, (i, s)
        continue
      assert cnt[i, j] == len(cells), (i, s)
      b = truth_lg[i][:, s]
      e = np.exp(b - b.max(-1, keepdims=True))
      grid = ((e / e.sum(-1, keepdims=True)) * wk[:, None]).sum(0)
      want = np.mean(-np.log(grid[cells] + eps))
      worst = max(worst, abs(nll[i, j] - want))
  print("  beam_nll_ragged vs fp64 NLL along the same selections: max |diff| %.2e" % worst)
  assert worst < 1e-5, worst


# --------------------------------------------------------------------------- multifuture.infer end to end
@pytest.mark.parametrize("case", ["k20_diverse", "k20_center_only", "greedy"])
def test_infer_points_against_fp64(dev, monkeypatch, case):
  """multifuture.infer on 10 trajectories of lengths 10..26 in batches of 4 (the last one partial): every point of
  output_data is centre + offset of the engine's selected cell, the offset within BAR x max|offset| of the fp64
  regression decoder's (the centre alone with --center_only, exactly)."""
  from multiverse_b200 import multifuture, synthetic
  import test_multifuture_gpu as MF
  over = dict(K20) if case != "greedy" else dict(K20, use_beam_search=False, beam_size=1, diverse_beam=False)
  seed, n = 621, 10
  tf, cfg, model = MF.make_model(monkeypatch, over, seed)
  w = synthetic.make_weights(cfg, seed)
  feeds = MF.script_feeds(model, cfg, n, seed)
  traj_ids = ["t%d_cam%d" % (r, r % 4) for r in range(n)]
  gi = cfg.use_grids.index(True)
  args = types.SimpleNamespace(scene_grid_centers=synthetic.grid_centers(cfg), num_out=20,
                               center_only=case == "k20_center_only")
  eng = model._ensure_engine()
  fwd, sel = eng.forward, []

  def recording(*a, **kw):
    out = fwd(*a, **kw)
    if out["beam_outputs"] is not None:
      ids = out["beam_outputs"][1].cpu().numpy()
    else:
      lg = out["grid_pred_decoded"][gi]
      ids = lg.reshape(lg.shape[0], lg.shape[1], -1).argmax(-1)[:, None].cpu().numpy()
    sel.append(ids)
    return out
  monkeypatch.setattr(eng, "forward", recording)
  got, _ = multifuture.infer(model, feeds, 4, args, traj_ids)
  assert [len(a) for a in sel] == [4, 4, 4]                    # the last batch: 2 trajectories + 2 padding rows
  ids = [row for a in sel for row in a][:n]
  centers = np.asarray(args.scene_grid_centers[gi], np.float64).reshape(-1, 2)
  worst = 0.0
  for r, tid in enumerate(traj_ids):
    length = int(feeds[r][model.pred_length][0])
    pts = np.asarray(got[tid], np.float64)
    k = pts.shape[0]
    assert pts.shape == (k, length, 2) and k == 20
    cells = ids[r][:, :length] if case != "greedy" else np.repeat(ids[r][:1, :length], k, 0)
    if args.center_only:
      assert np.array_equal(pts, centers[cells]), tid
      continue
    truth = BT.reg_truth(cfg, w, feeds[r][model.grid_obs_regress[gi]], gi, length, dev)[0].reshape(length, -1, 2)
    want = centers[cells] + truth[np.arange(length)[None], cells]
    err = np.abs(pts - want).max() / np.abs(truth).max()
    worst = max(worst, err)
    assert err < BAR, (tid, err)
  print("infer %s: %d trajectories in batches of 4, points vs centre + fp64 offset: %.1e" % (case, n, worst))
