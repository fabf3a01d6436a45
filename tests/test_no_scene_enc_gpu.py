# coding=utf-8
"""GPU tests of models built without --use_scene_enc: the class encoder's embedded one-hot input runs folded into the
cell epilogue (ops.cell_fwd_onehot, no x chunk in the GEMM) at inference, and through emb_onehot_fwd / emb_bwd into the
one grid_emb every scale shares in training; there is no scene CNN and the graph attention sees h alone.

Against the goldens of the executed reference (tests/golden/make_golden_no_scene_enc.py, pinned by
tests/test_no_scene_enc_cpu.py): ids bit-exact where the reference's selection is unambiguous at fp32 accuracy,
logits and offsets <= BAR = 1.6e-5 relative (greedy logits: the 1e-4 bar of test_parity_gpu); the training step's
whole-model gradient within the 2e-4 bar of the fp64 truth (tests/no_scene_enc_ref.py)."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
import no_scene_enc_ref as NS
from oracle import multiverse_ref as R
from test_beam_no_gnn_gpu import dropin_model, rel, to_dev
from test_dropin_gpu import make_batch
from test_train_atsize_gpu import FRAMES, GTOL, LTOL, T_PRED, chunk_feeds, on, shared_frame_feeds
from test_train_atsize_gpu import NS as MB
from test_train_options_gpu import _dropin_model, check_step_against_reference_execution

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TOL = 1e-4       # test_parity_gpu's bar of the greedy rollouts
BAR = 1.6e-5     # logits / offsets against the small goldens
WM_SEED = 337


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


def inputs(over, seed):
  from multiverse_b200 import synthetic
  cfg = NS.config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  return cfg, w, f, cases.checksum(*w.values()) + cases.checksum(f["traj"])


def run_case(name, dev, table=NS.ROLLOUTS, prefix="rollout_noscene_"):
  from multiverse_b200 import ops
  from multiverse_b200.engine import ConvRNNEngine
  cfg, w, f, ck = inputs(*table[name])
  g = np.load(os.path.join(GOLD, prefix + name + ".npz"))
  assert abs(float(g["checksum"]) - ck) < 1e-6
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  assert eng.scene_w == [] and all(sw is None or sw.enc_emb is not None for sw in eng.scales)
  ops.cell_variants_seen(reset=True)
  out = eng.forward(to_dev(f, dev))
  seen = ops.cell_variants_seen()
  return cfg, g, eng, w, f, out, seen


def test_rollout_greedy_two_scale(dev):
  """test.py without --use_scene_enc (greedy decode of both scales, graph attention over h alone): the decoded arg-max
  ids bit-exact (the reference's top-2 gaps clear the logit error), offsets within BAR and logits within the 1e-4 bar
  of test_parity_gpu's greedy rollouts (the class logits of this model measure 2.0e-5 on the 36x18 grid)."""
  cfg, g, eng, w, f, out, seen = run_case("greedy_two_scale", dev)
  errs = {}
  for i in range(2):
    lg = out["grid_pred_decoded"][i].cpu().numpy()
    n, tp = lg.shape[:2]
    assert g["margin_%d" % i].min() > 1e-3 * np.abs(g["logits_%d" % i]).max()
    assert np.array_equal(lg.reshape(n, tp, -1).argmax(-1), g["logits_%d" % i].reshape(n, tp, -1).argmax(-1))
    errs["logits_%d" % i] = rel(lg, g["logits_%d" % i])
    errs["offsets_%d" % i] = rel(out["grid_pred_reg_decoded"][i].cpu().numpy(), g["reg_%d" % i])
  print("greedy_two_scale rel errs", {k: "%.1e" % v for k, v in errs.items()})
  assert max(errs["logits_0"], errs["logits_1"]) < TOL and max(errs["offsets_0"], errs["offsets_1"]) < BAR, errs


def test_rollout_beam_k5_without_attention(dev):
  """test.py --use_beam_search without --use_gnn or --use_scene_enc (K = 5 plain beam, 18x9): beam ids bit-exact,
  logits and offsets within the bar."""
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


def beam_trace(eng, cfg, f, dev):
  """ConvRNNEngine.forward's class chain of a beam model, keeping the per-step trace of decode_class_beam (cells,
  parents and logits of every step).  Returns (beam outputs, trace) after checking that the outputs are forward()'s,
  bit for bit."""
  i = cfg.use_grids.index(True)
  feeds = to_dev(f, dev)
  labels_t = feeds["grid_obs_labels"][i].to(torch.int32).t().contiguous()
  obs_scene_t = feeds["obs_scene"].to(torch.int32).t().contiguous()
  c_e, h_e = eng.encode_class(i, None, obs_scene_t, labels_t, None)
  lg, ids, lp, tr = eng.decode_class_beam(i, c_e, h_e, labels_t[-1].contiguous(), None, cfg.pred_len)
  outs = [t.clone() for t in (lg, ids, lp)]
  tr = {k: v.clone() for k, v in tr.items()}
  for a, b in zip(eng.forward(feeds)["beam_outputs"], outs):
    assert torch.equal(a, b)
  return [t.cpu().numpy() for t in outs], {k: v.cpu().numpy() for k, v in tr.items()}


def check_beam_with_attention(cfg, w, f, dev, bar):
  """The beam decoder with graph attention (no scene features) against the fp64 truth replayed along the engine's own
  selections (no_scene_enc_ref.beam_replay): every live row's logits at every step within `bar`; the beam outputs are
  the back-trace of that trace.  Returns (engine outputs, relative logit error)."""
  from multiverse_b200 import ops
  from multiverse_b200.engine import ConvRNNEngine
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
  (blg, ids, lp), tr = beam_trace(eng, cfg, f, dev)
  assert (ops.PLANES_F16F8, True) in ops.cell_variants_seen(), "the CTA-pair f16f8 cell kernel did not run"
  truth = NS.beam_replay(cfg, w, f, cfg.use_grids.index(True), tr["ids"], tr["parents"], device=dev)
  err = rel(tr["logits"], truth)
  n, b, tp = ids.shape
  for j in range(n):                                    # the outputs are the back-trace of the checked trace
    par = np.arange(b)
    for t in range(tp - 1, -1, -1):
      assert np.array_equal(ids[j, :, t], tr["ids"][t, j, par]) and np.array_equal(blg[j, :, t], tr["logits"][t, j, par])
      par = tr["parents"][t, j, par]
  assert bool((lp[:, :-1] >= lp[:, 1:]).all())
  assert err < bar, err
  return (blg, ids, lp), err


def test_rollout_beam_k20_with_attention(dev):
  """multifuture_inference.py --use_gnn without --use_scene_enc (K = 20 diverse beam, 36x18, 60 beam rows: the CTA-pair
  f16f8 cell kernel; the attention runs without scene features).  Without scene features, far cells' log-probabilities
  inside a parent's row tie to 0-3e-5 (below the fp32 logit error), and the diverse penalty (log 0.01 = -4.6 per rank in
  the row) turns a swap of two such siblings into other selections further on: the executed reference's id sets are
  not a well-posed target at fp32.  So the fp64 truth is replayed along the engine's own selections, and every live
  row's logits at every step must be within the 1e-4 rollout bar; the offsets against the executed reference within
  BAR.  The agreement of the id sets with the reference's is reported."""
  cfg, w, f, ck = inputs(*NS.ROLLOUTS["beam_k20_gnn"])
  g = np.load(os.path.join(GOLD, "rollout_noscene_beam_k20_gnn.npz"))
  assert abs(float(g["checksum"]) - ck) < 1e-6
  (blg, ids, lp), err = check_beam_with_attention(cfg, w, f, dev, TOL)
  shared = [len(set(map(tuple, ids[j].tolist())) & set(map(tuple, g["beam_ids"][j].tolist())))
            for j in range(cfg.batch_size)]
  from multiverse_b200.engine import ConvRNNEngine
  out = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2).forward(to_dev(f, dev))
  reg = rel(out["grid_pred_reg_decoded"][0].cpu().numpy(), g["reg_0"])
  print("beam_k20_gnn: logits along the engine's selections %.1e, offsets %.1e; id sequences shared with the executed "
        "reference per sample %s of %d" % (err, reg, shared, cfg.beam_size))
  assert reg < BAR


def test_rollout_atsize_beam_k20_with_attention(dev):
  """At size: K = 20 diverse beam with attention of 16 trajectories on 36x18 (320 beam rows), the fp64 truth replayed
  along the engine's selections, every live row's logits at every step within the 1e-4 at-size bar."""
  from multiverse_b200 import synthetic
  over = dict(batch_size=16, use_grids=[True, False], use_beam_search=True, beam_size=20, diverse_beam=True,
              diverse_gamma=0.01, fix_num_timestep=1, use_gnn=True)
  cfg = NS.config(**over)
  w, f = synthetic.make_weights(cfg, 74), R.make_inputs(cfg, 74)
  _, err = check_beam_with_attention(cfg, w, f, dev, TOL)
  print("at size, K = 20, N = 16: logits along the engine's selections %.1e" % err)


def test_graph_replay_is_bit_identical(dev):
  """forward_graph replays the folded class encoder and the decoders bit-identically to the eager forward."""
  for name in ("greedy_two_scale", "beam_k5_nognn", "beam_k20_gnn"):
    cfg, g, eng, w, f, out, seen = run_case(name, dev)
    keys = [("grid_pred_decoded", i) for i in range(2) if cfg.use_grids[i]]
    ref = {k: out[k[0]][k[1]].clone() for k in keys}
    if out["beam_outputs"] is not None:
      ref.update((("beam_outputs", j), t.clone()) for j, t in enumerate(out["beam_outputs"]))
    feeds = to_dev(f, dev)
    for _ in range(3):                 # eager, capture, replay
      got = eng.forward_graph(feeds)
      torch.cuda.synchronize()
      for (k, j), t in ref.items():
        assert torch.equal(got[k][j], t), (name, k, j)


def test_batch_is_its_shards(dev):
  """64 trajectories, both scales, greedy with attention: every trajectory's outputs inside the batch are
  bit-identical to its outputs inside a 16-trajectory shard."""
  from multiverse_b200 import synthetic
  from multiverse_b200.engine import ConvRNNEngine
  n = 64
  cfg = synthetic.make_config(batch_size=n, use_scene_enc=False)
  w = synthetic.make_weights(cfg, 3)
  full = synthetic.make_feeds(cfg, n, 3)
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  out = eng.forward(to_dev(full, dev))
  whole = [t.clone() for t in out["grid_pred_decoded"] + out["grid_pred_reg_decoded"]]
  assert all(bool(torch.isfinite(t).all()) for t in whole)
  world = 4
  for rank in (0, 3):
    part = eng.forward(to_dev(synthetic.shard_feeds(full, rank, world), dev))
    lo, hi = rank * (n // world), (rank + 1) * (n // world)
    for a, b in zip(part["grid_pred_decoded"] + part["grid_pred_reg_decoded"], whole):
      assert torch.equal(a, b[lo:hi])


def test_whole_model_gradient_at_micro_batch(dev):
  """TrainEngine.loss_and_grads on 256 trajectories of shared frames in two micro-batches of 128 (both scales, graph
  attention) against the fp64 truth on the GPU over chunks of 16: losses within 1e-4, every variable's gradient - the
  shared grid_emb's, summed over both scales, 8 steps and both micro-batches, included - within 2e-4 of its largest
  element.  Without scene features the class logits of cells far from the trajectory nearly tie (the smallest top-2
  gap of the fp64 reference is below 1e-4 x max|logit| for every seed from 337 to 345), so the arg-max fed back is not
  well-posed at fp32; the truth therefore follows the engine's arg-max path (no gradient flows through the arg-max),
  and the engine's logits must be within the 1e-4 rollout bar of the truth's on that path.  Wherever the truth's top-2
  gap exceeds twice that logit error (a flip needs the errors of the two logits to differ by the gap), the engine's
  arg-max must be the truth's."""
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  n, mb, chunk = 256, MB, 16
  over = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001)
  cfg = synthetic.make_config(batch_size=mb, clip_gradient_norm=10.0, use_scene_enc=False, **over)
  rcfg = NS.config(batch_size=chunk, **over)
  w = synthetic.make_weights(cfg, WM_SEED)
  assert NS.ENC_EMB[0] in w and not any("scene_conv" in k for k in w)
  f = shared_frame_feeds(synthetic.make_config(batch_size=n, use_scene_enc=False), n, FRAMES, WM_SEED)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  got, ids, mine = 0.0, [[], []], [[], []]
  for lo in range(0, n, mb):
    part = chunk_feeds(f, slice(lo, lo + mb))
    feeds = {k: ([on(dev, a) for a in v] if isinstance(v, list) else on(dev, v)) for k, v in part.items()}
    l, _ = eng.loss_and_grads(feeds, loss_scale=mb / n, zero=(lo == 0))
    got = got + l.cpu().numpy()
    for i in range(2):
      ids[i].append(eng._store[("ids", i, mb)][0].cpu().numpy().T)               # [Tp, mb] -> [mb, Tp]
      mine[i].append(eng.last_logits[i].cpu().numpy().transpose(1, 0, 2))      # [mb, Tp, HW]
  torch.cuda.synchronize()
  ids = [np.concatenate(a) for a in ids]
  mine = [np.concatenate(a) for a in mine]
  grads = {k: np.zeros(v.shape) for k, v in w.items()}
  losses = np.zeros(4)
  logits = [[], []]
  for lo in range(0, n, chunk):
    sl = slice(lo, lo + chunk)
    _, l, _, gr, lg = NS.loss_and_grads(rcfg, w, chunk_feeds(f, sl), device=dev, return_logits=True,
                                        fed_ids=[a[sl] for a in ids])
    losses += np.array(l) * chunk / n
    for k in grads:
      grads[k] += gr[k] * chunk / n
    for i in range(2):
      logits[i].append(lg[i].reshape(chunk, T_PRED, -1))
  for k in grads:
    if k.endswith("/W"):
      grads[k] -= cfg.wd * w[k]
  for i in range(2):
    ref = np.concatenate(logits[i])
    err = rel(mine[i], ref)
    # the path is the engine's arg-max: where the truth's top-2 gap exceeds twice the logit error, it is the truth's
    srt = np.sort(ref, -1)
    clear = srt[..., -1] - srt[..., -2] > 2 * err * np.abs(ref).max()
    agree = ref.argmax(-1) == ids[i]
    print("scale %d: logit error on the engine's arg-max path %.2e; arg-max checked at %.1f %% of the steps"
          % (i, err, 100.0 * clear.mean()))
    assert err < TOL and agree[clear].all() and clear.mean() > 0.25
  assert np.abs(got - losses).max() < LTOL * np.abs(losses).max(), (got, losses)
  worst = {k: rel(eng.grads[k].cpu().numpy(), grads[k]) for k in sorted(grads)}
  print("whole model without scene encoding, 256 trajectories in micro-batches of 128: losses %.1e, grid_emb %.1e, "
        "worst gradient errors %s" % (np.abs(got - losses).max() / np.abs(losses).max(), worst[NS.ENC_EMB[0]],
                                      sorted(worst.items(), key=lambda kv: -kv[1])[:4]))
  bad = {k: v for k, v in worst.items() if v > GTOL}
  assert not bad, bad


def test_two_ranks_equal_one_rank():
  """tests/ddp_check_no_scene_enc.py: two ranks on one GPU over gloo, each on its shard, all-reduced, equal one rank's
  step on the whole batch (losses, gradients - grid_emb's included - and the updated weights)."""
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
         "127.0.0.1", "--master-port", "29543", os.path.join(ROOT, "tests", "ddp_check_no_scene_enc.py")]
  r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  assert "DDP_CHECK" in r.stdout
  print(r.stdout[r.stdout.index("DDP_CHECK"):].splitlines()[0])


def test_dropin_trainer_step_equals_reference_execution(dev, monkeypatch):
  """One Trainer.step through the drop-in with TRAINING.md's arguments without --use_scene (scene 36x64, both scales,
  loss weights 1.0 / 0.2, --init_lr 0.3) on the inputs of tests/golden/refexec_train_noscene.npz: losses, every
  clipped gradient and the variables after Adadelta equal the unmodified reference Model + Trainer's."""
  over, seed = NS.TRAIN
  cfg, w, f, ck = inputs(over, seed)
  got = np.load(os.path.join(GOLD, "refexec_train_noscene.npz"))
  assert abs(float(got["checksum"]) - ck) < 1e-6
  dover = dict(scene_h=cfg.scene_h, scene_w=cfg.scene_w, use_grids=[True, True], use_scene_enc=False,
               grid_loss_weight=over["grid_loss_weight"], grid_reg_loss_weight=over["grid_reg_loss_weight"],
               wd=over["wd"])
  tf, pred_models, model, args, _, _, _, batch = _dropin_model(monkeypatch, w=w, f=f, n=cfg.batch_size, over=dover,
                                                               train_w_onehot=True, init_lr=over["init_lr"])
  assert set(model.weights()) == set(got["variables"])
  check_step_against_reference_execution("no_scene_enc", tf, pred_models, model, args, batch, w, got, "")


def test_dropin_tester_step_and_session_run(dev, monkeypatch):
  """code/test.py --use_beam_search without --use_gnn / --use_scene_enc: Tester.step through the shim's Session
  (eager, then graph capture and replay) returns the executed reference's beam ids, class and offset maps; and
  code/multifuture_inference.py --use_gnn's sess.run of the beam outputs on Model.get_feed_dict (K = 20 diverse beam
  with attention): bit-identical to ConvRNNEngine.forward, which test_rollout_beam_k20_with_attention checks."""
  cfg, w, f, _ = inputs(*NS.ROLLOUTS["beam_k5_nognn"])
  g = np.load(os.path.join(GOLD, "rollout_noscene_beam_k5_nognn.npz"))
  tf, pred_models, model, args = dropin_model(monkeypatch, cfg, w)
  assert set(model.weights()) == set(g["variables"]) - {"global_step"}
  with tf.Session(config=tf.ConfigProto(allow_soft_placement=True)) as sess:
    tester = pred_models.Tester(model, args, sess)
    for _ in range(3):
      cls, reg, (lg, ids, lp) = tester.step(sess, make_batch(cfg, f, cfg.batch_size))
      assert np.array_equal(ids, g["beam_ids"]) and np.abs(lp - g["beam_logprobs"]).max() < 1e-3
      assert rel(cls[1], g["logits_1"]) < BAR and rel(reg[1], g["reg_1"]) < BAR
  from multiverse_b200.engine import ConvRNNEngine
  cfg, w, f, _ = inputs(*NS.ROLLOUTS["beam_k20_gnn"])
  want = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2).forward(to_dev(f, dev))
  tf, _, model, _ = dropin_model(monkeypatch, cfg, w)
  fd = model.get_feed_dict(make_batch(cfg, f, cfg.batch_size)[1])
  with tf.Session() as sess:
    for _ in range(3):           # eager, then CUDA-graph capture and replay (fewer than 2000 beam rows)
      got = sess.run([model.beam_outputs, model.grid_pred_reg_decoded[0]], fd)
      for a, b in zip(list(got[0]) + [got[1]], want["beam_outputs"] + [want["grid_pred_reg_decoded"][0]]):
        assert np.array_equal(a, b.cpu().numpy())
