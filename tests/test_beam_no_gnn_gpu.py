# coding=utf-8
"""GPU tests of the K-way beam decoder without graph attention (use_gnn off): the parent-state gather kernel
(mvb_beam_gather_h_f16f8) at the benchmark's 10 240 beam rows, and whole rollouts against the goldens of the executed
reference (tests/golden/make_golden_ablation.py, pinned by tests/test_beam_no_gnn_cpu.py).

Bars: ids bit-exact where the reference's selection is unambiguous at fp32 accuracy; against the small goldens, logits
and offsets <= BAR = 1.6e-5 relative (max|diff| / max|ref| per tensor: the accuracy smoke() reports for the c4 path);
at size, the at-size rule and 1e-4 bar of test_parity_gpu.test_rollout_atsize."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

import cases
import cases_ablation
from oracle import multiverse_ref as R
from test_dropin_gpu import make_batch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TOL = 1e-4       # the at-size bar
BAR = 1.6e-5     # logits / offsets against the small goldens
SENT = 0x5A      # byte sentinel in every operand byte the gather must not write


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


def rel(a, b):
  a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
  return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def up(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def to_dev(feeds, dev):
  return dict(scene_feat=up(feeds["scene_feat"], dev), obs_scene=up(feeds["obs_scene"], dev),
              grid_obs_labels=[up(a, dev) for a in feeds["grid_obs_labels"]],
              grid_obs_regress=[up(a, dev) for a in feeds["grid_obs_regress"]])


def test_gather_h_at_beam_size(dev):
  """10 240 beam rows of 36x18 (512 trajectories x K = 20) with a beam row map (parents repeat and are not monotone):
  the h block of every grid cell is bit-identical to a torch gather followed by the f16f8 split (fp16 value, e4m3 of
  it, e4m3 of the residual x 2^12), and every other byte - x block, channel padding, halo rows - keeps its sentinel."""
  from multiverse_b200 import ops
  n, b, h, w = 512, 20, 36, 18
  ns, s_rows = n * b, (h + 1) * (w + 1)
  cpad = ops.cell_cpad(32)
  cxp = cpad - ops.HIDDEN
  rows = ops.halo_rows(ns, h, w)
  g = torch.Generator(device=dev).manual_seed(5)
  h32 = torch.tanh(torch.randn((rows, ops.HIDDEN), device=dev, generator=g) * 2)
  parents = torch.randint(0, b, (n, b), device=dev, generator=g, dtype=torch.int32)
  row_map = (torch.arange(n, device=dev, dtype=torch.int32)[:, None] * b + parents).reshape(-1).contiguous()
  xh = ops.alloc_xh(ns, h, w, cpad, ops.PLANES_F16F8, dev)
  xh.view(torch.uint8).fill_(SENT)
  want = xh.clone()
  ops.beam_gather_h(h32, row_map, xh, h, w, ns)
  # the expected bytes, written chunk by chunk into the sentinel copy
  raw = want.view(torch.uint8).reshape(-1)
  f16 = raw[:2 * rows * cpad].view(torch.float16).view(rows, cpad)
  f8 = raw[2 * rows * cpad:].view(rows, 2 * cpad)
  c = torch.arange(ops.HIDDEN, device=dev)
  off0 = 2 * cxp + (c // 64) * 128 + c % 64           # inside an fp8 row: per 64 h channels [e0 (64) | e1 (64)]
  yy, xx = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
  cells = (yy * (w + 1) + xx).reshape(-1)
  for s0 in range(0, ns, 512):
    s = torch.arange(s0, min(ns, s0 + 512), device=dev)
    dst = (s[:, None] * s_rows + cells[None]).reshape(-1)
    src = (row_map[s].long()[:, None] * s_rows + cells[None]).reshape(-1)
    v = h32[src]
    a0 = v.half()
    e0 = a0.float().to(torch.float8_e4m3fn).view(torch.uint8)
    e1 = ((v - a0.float()) * 4096.0).to(torch.float8_e4m3fn).view(torch.uint8)
    f16[dst[:, None], (cxp + c)[None]] = a0
    f8[dst[:, None], off0[None]] = e0
    f8[dst[:, None], (off0 + 64)[None]] = e1
  torch.cuda.synchronize()
  got_b, want_b = xh.view(torch.uint8), want.view(torch.uint8)
  assert torch.equal(got_b, want_b), "%d bytes differ" % int((got_b != want_b).sum())
  # (implied by the equality; stated for the reader) halo rows and x blocks still hold the sentinel
  v = xh.view(torch.uint8).view(2, ns, h + 1, w + 1, 2 * cpad)
  assert bool((v[:, :, h] == SENT).all()) and bool((v[:, :, :, w] == SENT).all())
  assert bool((v[..., :2 * cxp] == SENT).all())


def test_gather_h_refuses_a_buffer_of_another_shape(dev):
  from multiverse_b200 import ops
  h, w, ns = 6, 5, 4
  xh = ops.alloc_xh(ns + 1, h, w, ops.cell_cpad(32), ops.PLANES_F16F8, dev)
  h32 = ops.alloc_state(ns, h, w, dev)
  rm = torch.zeros((ns,), dtype=torch.int32, device=dev)
  with pytest.raises(AssertionError):
    ops.beam_gather_h(h32, rm, xh, h, w, ns)
  with pytest.raises(RuntimeError, match="plane stride"):
    from multiverse_b200 import _lib
    _lib.call("mvb_beam_gather_h_f16f8", ops._p(h32), ops._p(rm), ops._p(xh), xh.stride(0), xh.shape[2], ns, h, w,
              ops._stream())


def run_case(name, dev):
  from multiverse_b200 import ops
  from multiverse_b200.engine import ConvRNNEngine
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**over)
  w = R.make_weights(cfg, seed); f = R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "rollout_%s.npz" % name))
  assert abs(float(g["checksum"]) - (cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"]))) < 1e-6
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
  out = eng.forward(to_dev(f, dev))
  seen = ops.cell_variants_seen()
  return cfg, g, eng, w, f, out, seen


def test_rollout_beam_k5_without_attention(dev):
  """test.py --use_beam_search without --use_gnn (K = 5 plain beam, 18x9): beam ids bit-exact (the reference's
  selection margins are >= 2.4e-4 at every step), logits and offsets within the bar."""
  from multiverse_b200 import ops
  cfg, g, eng, w, f, out, seen = run_case("beam_k5_nognn", dev)
  assert g["beam_margins"].min() > 2e-4
  assert (ops.PLANES_F16F8, False) in seen, seen
  blg, ids, lp = [t.cpu().numpy() for t in out["beam_outputs"]]
  assert ids.dtype == np.int32 and np.array_equal(ids, g["beam_ids"])
  assert np.abs(lp - g["beam_logprobs"]).max() < 1e-3
  errs = dict(beam_logits=rel(blg[:, :3], g["beam_logits_top3"]),
              logits=rel(out["grid_pred_decoded"][1].cpu().numpy(), g["logits_1"]),
              offsets=rel(out["grid_pred_reg_decoded"][1].cpu().numpy(), g["reg_1"]))
  print("beam_k5_nognn rel errs", {k: "%.1e" % v for k, v in errs.items()})
  assert max(errs.values()) < BAR, errs
  assert_offsets_as_with_attention(cfg, w, f, out, dev)
  out2 = eng.forward(to_dev(f, dev))             # buffer reuse: bit-identical
  for a, b in zip(out["beam_outputs"], out2["beam_outputs"]):
    assert torch.equal(a, b)


def test_rollout_beam_k20_without_attention(dev):
  """multifuture_inference.py without --use_gnn (K = 20 diverse beam, 36x18, 60 beam rows: the CTA-pair f16f8 cell
  kernel).  The reference's K-th / (K+1)-th candidate gap is >= 4 at every step, but children of different parents
  tie to ~1e-9 inside the beam, so their ORDER is not defined at fp32 accuracy (the at-size rule of
  test_parity_gpu.test_rollout_atsize): the set of id sequences is bit-exact per sample, log-probabilities and
  per-beam logit statistics compared sorted over the beam axis."""
  from multiverse_b200 import ops
  cfg, g, eng, w, f, out, seen = run_case("beam_k20_nognn", dev)
  assert g["beam_margins"][..., 1].min() > 2e-4
  assert (ops.PLANES_F16F8, True) in seen, "the CTA-pair f16f8 cell kernel did not run: %s" % sorted(seen)
  blg, ids, lp = [t.cpu().numpy() for t in out["beam_outputs"]]
  seqs = lambda a: sorted(map(tuple, a.tolist()))
  for j in range(cfg.batch_size):
    assert seqs(ids[j]) == seqs(g["beam_ids"][j]), "beam id sets differ from the reference in sample %d" % j
  assert np.abs(np.sort(lp, 1) - np.sort(g["beam_logprobs"], 1)).max() < 1e-3
  scale = np.abs(g["beam_lg_max"]).max()
  errs = {k: float(np.abs(np.sort(fn(blg), 1) - np.sort(g[k], 1)).max() / scale)
          for k, fn in (("beam_lg_max", lambda a: a.max(-1)), ("beam_lg_mean", lambda a: a.mean(-1)))}
  errs["offsets"] = rel(out["grid_pred_reg_decoded"][0].cpu().numpy(), g["reg_0"])
  exact = sum(np.array_equal(ids[j], g["beam_ids"][j]) for j in range(cfg.batch_size))
  print("beam_k20_nognn: id sets equal in all %d samples, beam for beam in %d; rel errs %s"
        % (cfg.batch_size, exact, {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < BAR, errs
  assert_offsets_as_with_attention(cfg, w, f, out, dev)


def assert_offsets_as_with_attention(cfg, w, f, out, dev):
  """The offset decoder does not depend on use_gnn: its outputs equal, bit for bit, those of the model with the
  attention on the same weights and feeds."""
  from multiverse_b200.engine import ConvRNNEngine
  i = cfg.use_grids.index(True)
  cfg_g = R.default_config(**dict(vars(cfg), use_gnn=True))
  with_gnn = ConvRNNEngine(cfg_g, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2).forward(to_dev(f, dev))
  assert torch.equal(with_gnn["grid_pred_reg_decoded"][i], out["grid_pred_reg_decoded"][i])


def test_graph_replay_is_bit_identical_without_attention(dev):
  """forward_graph (the drop-in's path below 2000 beam rows) replays the no-attention beam decoder bit-identically."""
  cfg, g, eng, w, f, out, seen = run_case("beam_k5_nognn", dev)
  ref = [t.clone() for t in out["beam_outputs"]]
  feeds = to_dev(f, dev)
  for _ in range(3):                 # eager, capture, replay
    got = eng.forward_graph(feeds)
    torch.cuda.synchronize()
    for a, b in zip(got["beam_outputs"], ref):
      assert torch.equal(a, b)


def test_batch_is_its_shards_without_attention(dev):
  """64 trajectories x K = 20 on 36x18 (1 280 beam rows): every trajectory's beam outputs inside the batch are
  bit-identical to its outputs inside a 16-trajectory shard - the gather reads only its own sample's parents - plus
  the properties of a rollout that need no oracle."""
  from multiverse_b200 import ops, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  n = 64
  cfg = synthetic.make_config(batch_size=n, use_grids=[True, False], use_beam_search=True, beam_size=20,
                              diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=False)
  w = synthetic.make_weights(cfg, 3)
  full = synthetic.make_feeds(cfg, n, 3)
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
  lg, ids, lp = [t.clone() for t in eng.forward(to_dev(full, dev))["beam_outputs"]]
  assert (ops.PLANES_F16F8, True) in ops.cell_variants_seen()
  assert int(ids.min()) >= 0 and int(ids.max()) < 648 and bool(torch.isfinite(lg).all())
  assert bool((lp[:, :-1] >= lp[:, 1:]).all())
  world = 4
  for rank in (0, 3):
    part = eng.forward(to_dev(synthetic.shard_feeds(full, rank, world), dev))
    lo, hi = rank * (n // world), (rank + 1) * (n // world)
    for a, b in zip(part["beam_outputs"], (lg, ids, lp)):
      assert torch.equal(a, b[lo:hi])


def test_rollout_atsize_without_attention(dev):
  """K = 20 diverse beam of 16 trajectories on 36x18 without the attention against the fp64 oracle's statistics
  (tests/golden/atsize_beam_k20_nognn_n16.npz), under the at-size rule of test_parity_gpu.test_rollout_atsize: on the
  boundary-safe samples (gap between the K-th selected and the best unselected candidate > 2e-4 at every step) the
  set of id sequences is bit-exact, log-probabilities and per-beam logit statistics agree sorted over the beam axis;
  offsets within the 1e-4 bar on every sample."""
  from multiverse_b200 import ops
  from multiverse_b200.engine import ConvRNNEngine
  name = "beam_k20_nognn_n16"
  over, seed = cases_ablation.ROLLOUTS_NO_GNN_ATSIZE[name]
  cfg = R.default_config(**over)
  w = R.make_weights(cfg, seed); f = R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "atsize_%s.npz" % name))
  assert abs(float(g["checksum"]) - (cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"]))) < 1e-6
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
  out = eng.forward(to_dev(f, dev))
  assert (ops.PLANES_F16F8, True) in ops.cell_variants_seen()
  res = dict(grid_pred_decoded=[t.cpu().numpy() if torch.is_tensor(t) else t for t in out["grid_pred_decoded"]],
             grid_pred_reg_decoded=[t.cpu().numpy() if torch.is_tensor(t) else t for t in out["grid_pred_reg_decoded"]],
             beam_outputs=[t.cpu().numpy() for t in out["beam_outputs"]])
  st = cases.rollout_stats(cfg, res)
  n = cfg.batch_size
  safe = g["beam_margins"][:, :, 1].min(1) > 2e-4
  assert safe.mean() >= 0.75, "too few boundary-safe samples: %.2f" % safe.mean()
  seqs = lambda a: sorted(map(tuple, a.tolist()))
  same_set = np.array([seqs(st["beam_ids"][j]) == seqs(g["beam_ids"][j]) for j in range(n)])
  assert same_set[safe].all(), "beam id sets differ on boundary-safe samples %s" % np.nonzero(safe & ~same_set)[0]
  assert np.abs(np.sort(st["beam_logprobs"], 1) - np.sort(g["beam_logprobs"], 1))[safe].max() < 1e-3
  worst = {}
  bs = np.abs(g["beam_lg_max"]).max()
  for k in ("beam_lg_max", "beam_lg_mean"):
    worst[k] = float(np.abs(np.sort(st[k], 1) - np.sort(g[k], 1))[safe].max() / bs)
  rs = np.abs(g["reg_at_0"]).max()
  for k in ("reg_mean_0", "reg_at_0"):
    worst[k] = float(np.abs(st[k] - g[k]).max() / rs)
  print("atsize %s: %d of %d samples boundary-safe, id sets equal on all of them; rel errs %s"
        % (name, int(safe.sum()), n, {k: "%.1e" % v for k, v in worst.items()}))
  assert max(worst.values()) < TOL, worst


def dropin_model(monkeypatch, cfg, w):
  """The reference-facing surface (multiverse_b200/dropin) with the weights w loaded: get_model as code/test.py and
  code/multifuture_inference.py call it."""
  import types
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  tf.reset_default_graph()
  args = types.SimpleNamespace(**dict(vars(cfg), is_train=False, keep_prob=1.0))     # as test.py's inference args
  args.modelname, args.use_soft_grid_class, args.use_gt_grid = "m", False, False
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  return tf, pred_models, model, args


def test_dropin_tester_step_beam_without_attention(dev, monkeypatch):
  """code/test.py --use_beam_search without --use_gnn: Tester.step through the shim's Session (code/pred_utils.py:415)
  returns what the executed reference returned: beam ids bit-exact, class and offset maps within BAR."""
  name = "beam_k5_nognn"
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**over)
  w = R.make_weights(cfg, seed); f = R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "rollout_%s.npz" % name))
  tf, pred_models, model, args = dropin_model(monkeypatch, cfg, w)
  with tf.Session(config=tf.ConfigProto(allow_soft_placement=True)) as sess:
    tester = pred_models.Tester(model, args, sess)
    for _ in range(3):           # eager, then CUDA-graph capture and replay (fewer than 2000 beam rows)
      cls, reg, (lg, ids, lp) = tester.step(sess, make_batch(cfg, f, cfg.batch_size))
      assert cls[0] == [] and reg[0] == []
      assert ids.dtype == np.int32 and np.array_equal(ids, g["beam_ids"])
      assert np.abs(lp - g["beam_logprobs"]).max() < 1e-3
      assert rel(cls[1], g["logits_1"]) < BAR and rel(reg[1], g["reg_1"]) < BAR


def test_dropin_session_run_beam_without_attention(dev, monkeypatch):
  """code/multifuture_inference.py without --use_gnn: sess.run of the beam outputs and the offset maps on
  Model.get_feed_dict (:304-385, :471) - K = 20 diverse beam on 36x18, id sets equal to the executed reference's per
  sample (the in-beam order of near-tied twins is not defined at fp32 accuracy, see
  test_rollout_beam_k20_without_attention)."""
  name = "beam_k20_nognn"
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**over)
  w = R.make_weights(cfg, seed); f = R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "rollout_%s.npz" % name))
  tf, _, model, _ = dropin_model(monkeypatch, cfg, w)
  fd = model.get_feed_dict(make_batch(cfg, f, cfg.batch_size)[1])
  with tf.Session() as sess:
    (lg, ids, lp), reg = sess.run([model.beam_outputs, model.grid_pred_reg_decoded[0]], fd)
  seqs = lambda a: sorted(map(tuple, a.tolist()))
  for j in range(cfg.batch_size):
    assert seqs(ids[j]) == seqs(g["beam_ids"][j]), j
  assert np.abs(np.sort(lp, 1) - np.sort(g["beam_logprobs"], 1)).max() < 1e-3
  assert rel(reg, g["reg_0"]) < BAR
