# coding=utf-8
"""GPU parity tests of the backward (BPTT) kernels against torch autograd on the oracle's
torch-CPU restatement (fp64)."""
import os

import numpy as np
import pytest
import torch

import cases
from oracle import multiverse_ref_torch as RT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu
GTOL = 2e-4   # gradients: relative to the largest entry of each gradient tensor


def rel(a, b):
  a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
  return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def T(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.parametrize("name", ["dec_cx32", "enc_class_cx64", "tile_edge", "enc_reg_cx2"])
def test_cell_backward_with_direct_wgrad_matches_autograd(dev, name):
  from multiverse_b200 import ops
  d = cases.cell_case(name)
  ns, h, w, cx = d["x"].shape
  rng = np.random.default_rng(5)
  dh = rng.standard_normal((ns, h, w, 256)).astype(np.float32)
  dc = rng.standard_normal((ns, h, w, 256)).astype(np.float32)
  # truth: autograd through the torch restatement
  t = {k: torch.from_numpy(v).double().requires_grad_(True) for k, v in d.items()}
  c1, h1 = RT.convlstm_cell(t["x"], t["c"], t["h"], t["kernel"], t["biases"])
  ((h1 * torch.from_numpy(dh).double()).sum() + (c1 * torch.from_numpy(dc).double()).sum()).backward()
  comp = name == "enc_reg_cx2"
  planes = 2
  pk = ops.PackedCell(T(d["kernel"], dev), T(d["biases"], dev), planes, comp=comp)
  wd = ops.pack_dgrad(pk, T(d["kernel"], dev))
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(T(d["x"], dev), xh, 0, h, w, comp=pk.comp)
  ops.nhwc_to_planes(T(d["h"], dev), xh, pk.cxp, h, w)
  c_in = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(d["c"], dev), c_in, h, w)
  c_out = ops.alloc_state(ns, h, w, dev); h_out = ops.alloc_state(ns, h, w, dev)
  R = ops.halo_rows(ns, h, w)
  gates = torch.zeros((R, 1024), device=dev)
  ops.cell_fwd_train(xh, pk, c_in, c_out, h_out, None, gates, h, w, ns)
  dh_h = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(dh, dev), dh_h, h, w)
  dc_h = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(dc, dev), dc_h, h, w)
  dg = torch.zeros((planes, R, 1024), dtype=torch.bfloat16, device=dev)
  dc_prev = ops.alloc_state(ns, h, w, dev)
  dbp = torch.zeros((1024,), device=dev)
  ops.lstm_gates_bwd(gates, c_in, c_out, dh_h, dc_h, dg, dc_prev, dbp, h, w, ns)
  # dc_{t-1}
  dcp = torch.empty((ns, h, w, 256), device=dev); ops.halo_to_nhwc(dc_prev, dcp, h, w)
  assert rel(dcp.cpu().numpy(), t["c"].grad.numpy()) < GTOL
  # dgrad
  dxh = torch.zeros((R, pk.cpad), device=dev)
  ops.cell_dgrad(dg, wd, dxh, h, w, ns)
  dxh_v = dxh.view(ns, h + 1, w + 1, pk.cpad)[:, :h, :w].cpu().numpy()
  assert rel(dxh_v[..., pk.cxp:], t["h"].grad.numpy()) < GTOL
  if not comp:
    assert rel(dxh_v[..., :cx], t["x"].grad.numpy()) < GTOL
  # wgrad: MN-major operands straight from the row-major planes; a second run accumulates to exactly 2x
  dwp = torch.zeros((ops.wgrad_slabs(pk.cpad), 1024, 9 * pk.cpad), device=dev)
  ops.cell_wgrad_direct(dg, xh, dwp, h, w, ns)
  dwp1 = dwp.clone()
  ops.cell_wgrad_direct(dg, xh, dwp, h, w, ns)
  assert torch.equal(dwp, 2 * dwp1)
  dk = torch.empty((3, 3, cx + 256, 1024), device=dev); db = torch.empty((1024,), device=dev)
  ops.unpack_cell_wgrad(dwp, dbp, dk, db, cx, comp=pk.comp)
  assert rel(0.5 * dk.cpu().numpy(), t["kernel"].grad.numpy()) < GTOL
  assert rel(db.cpu().numpy(), t["biases"].grad.numpy()) < GTOL
  # the same bf16 planes the kernel multiplies, in fp64: a0b0 + a0b1 + a1b0 per tap shift of the activation rows
  ref = torch.zeros((1024, 9 * pk.cpad), dtype=torch.float64, device=dev)
  for tap in range(9):
    shift = (tap // 3 - 1) * (w + 1) + (tap % 3 - 1)
    xs = torch.zeros((2, R, pk.cpad), dtype=torch.float64, device=dev)
    lo, hi = max(0, -shift), min(R, R - shift)
    xs[:, lo:hi] = xh[:, lo + shift:hi + shift].double()
    ref[:, tap * pk.cpad:(tap + 1) * pk.cpad] = sum(dg[a].double().t() @ xs[b] for a, b in ((0, 0), (0, 1), (1, 0)))
  err = rel(dwp1.sum(0).double().cpu().numpy(), ref.cpu().numpy())
  print("cell %s: wgrad against the fp64 product of its bf16 planes: rel err %.2e" % (name, err))
  assert err < 1e-5


def test_loss_kernel(dev):
  from multiverse_b200 import ops
  import torch.nn.functional as F
  rng = np.random.default_rng(1)
  lg = (rng.standard_normal((7, 3, 50)) * 3).astype(np.float32)
  lab = rng.integers(0, 50, size=(7, 3)).astype(np.int32)
  pr = (rng.standard_normal((7, 3, 50, 2)) * 2).astype(np.float32)
  tg = (rng.standard_normal((7, 3, 50, 2)) * 2).astype(np.float32)
  tl = torch.from_numpy(lg).double().requires_grad_(True); tp = torch.from_numpy(pr).double().requires_grad_(True)
  l1 = F.cross_entropy(tl.reshape(-1, 50), torch.from_numpy(lab).long().reshape(-1)) * 1.5
  l2 = F.huber_loss(tp, torch.from_numpy(tg).double(), delta=1.0) * 0.2
  (l1 + l2).backward()
  dl = torch.empty(7, 3, 50, device=dev); dp = torch.empty(7, 3, 50, 2, device=dev)
  out = torch.zeros(2, device=dev)
  ops.loss_fwd_bwd(T(lg, dev), T(lab, dev), dl, 1.5, T(pr, dev), T(tg, dev), dp, 0.2, out)
  assert abs(out[0].item() - l1.item()) < 1e-5 * abs(l1.item()) and abs(out[1].item() - l2.item()) < 1e-5 * abs(l2.item())
  assert rel(dl.cpu().numpy(), tl.grad.numpy()) < 1e-5 and rel(dp.cpu().numpy(), tp.grad.numpy()) < 1e-5


@pytest.mark.parametrize("pout", [1, 2])
def test_head_and_emb_backward(dev, pout):
  from multiverse_b200 import ops
  d = cases.head_case()
  ns, h, w, _ = d["h"].shape
  rng = np.random.default_rng(2)
  Wo = d["Wo1"] if pout == 1 else d["Wo2"]
  dout = rng.standard_normal((ns, h * w, pout)).astype(np.float32)
  th = torch.from_numpy(d["h"]).double().requires_grad_(True); tW = torch.from_numpy(Wo).double().requires_grad_(True)
  o = RT.conv2d_same(th, tW)
  (o.reshape(ns, h * w, pout) * torch.from_numpy(dout).double()).sum().backward()
  h32 = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(d["h"], dev), h32, h, w)
  dWo = torch.zeros(3, 3, 256, pout, device=dev); dh = ops.alloc_state(ns, h, w, dev)
  ops.head_bwd(h32, T(dout, dev), T(Wo, dev), dWo, dh, False, h, w, ns)
  ops.head_bwd(h32, T(dout, dev), T(Wo, dev), dWo, dh, True, h, w, ns)      # accumulate: 2x
  dhn = torch.empty(ns, h, w, 256, device=dev); ops.halo_to_nhwc(dh, dhn, h, w)
  assert rel(0.5 * dhn.cpu().numpy(), th.grad.numpy()) < 1e-5
  assert rel(0.5 * dWo.cpu().numpy(), tW.grad.numpy()) < 1e-5
  # embedding backward
  e = 32
  We = d["We1"] if pout == 1 else d["We2"]
  dx = rng.standard_normal((ns, h, w, e)).astype(np.float32)
  tWe = torch.from_numpy(We).double().requires_grad_(True); tbe = torch.from_numpy(d["be"]).double().requires_grad_(True)
  if pout == 1:
    ids = rng.integers(0, h * w, size=ns).astype(np.int32); ids[0] = 0
    tin = RT.one_hot_map(torch.from_numpy(ids), h, w, torch.float64)
  else:
    inm = rng.standard_normal((ns, h, w, 2)).astype(np.float32)
    tin = torch.from_numpy(inm).double().requires_grad_(True)
  (RT.grid_emb(tin, tWe, tbe) * torch.from_numpy(dx).double()).sum().backward()
  dxh = torch.zeros(ops.halo_rows(ns, h, w), 288, device=dev)
  dxh.view(ns, h + 1, w + 1, 288)[:, :h, :w, :e] = T(dx, dev)
  dWe = torch.zeros_like(T(We, dev)); dbe = torch.zeros(e, device=dev)
  if pout == 1:
    ops.emb_bwd(dxh, T(ids, dev), None, T(We, dev), T(d["be"], dev), dWe, dbe, None, False, h, w, ns)
  else:
    din = torch.ones(ns, h * w, 2, device=dev)
    ops.emb_bwd(dxh, None, T(inm.reshape(ns, h * w, 2), dev), T(We, dev), T(d["be"], dev), dWe, dbe, din, True, h, w, ns)
    assert rel(din.cpu().numpy() - 1.0, tin.grad.numpy().reshape(ns, h * w, 2)) < 1e-5
  assert rel(dWe.cpu().numpy(), tWe.grad.numpy()) < 1e-5 and rel(dbe.cpu().numpy(), tbe.grad.numpy()) < 1e-5


@pytest.mark.parametrize("with_scene", [True, False])
def test_gnn_backward(dev, with_scene):
  from multiverse_b200 import ops
  d = cases.gnn_case()
  ns, h, w, _ = d["h"].shape
  rng = np.random.default_rng(3)
  g = rng.standard_normal((ns, h, w, 256)).astype(np.float32)
  hh = d["h"].copy(); hh[0, 0, 0] = 0.0                                  # a zero-norm cell (eps clamp)
  th = torch.from_numpy(hh).double().requires_grad_(True)
  ts = torch.from_numpy(d["scene"] * (0.0 if not with_scene else 1.0)).double().requires_grad_(True)
  out = RT.gnn_dense(th, ts if with_scene else None, RT.neighbour_mask(h, w, torch.float64))
  (out * torch.from_numpy(g).double()).sum().backward()
  h32 = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(hh, dev), h32, h, w)
  gh = ops.alloc_state(ns, h, w, dev); ops.nhwc_to_halo(T(g, dev), gh, h, w)
  work = torch.empty(19 * ns * h * w, device=dev)
  dh = ops.alloc_state(ns, h, w, dev); ds = torch.zeros(ns, h, w, 64, device=dev)
  ops.gnn_bwd(h32, T(d["scene"], dev) if with_scene else None, gh, work, dh, False, ds if with_scene else None, h, w, ns)
  dhn = torch.empty(ns, h, w, 256, device=dev); ops.halo_to_nhwc(dh, dhn, h, w)
  if with_scene:
    assert rel(dhn.cpu().numpy(), th.grad.numpy()) < 2e-5
    assert rel(ds.cpu().numpy(), ts.grad.numpy()) < 2e-5
  else:
    ref = th.grad.numpy().copy()
    # the zero-norm cell: autograd of rsqrt(clamp(...)) passes the gradient straight through
    assert rel(dhn.cpu().numpy(), ref) < 2e-5


def test_scene_backward(dev):
  from multiverse_b200 import ops
  d = cases.scene_case()
  rng = np.random.default_rng(4)
  x = torch.from_numpy(d["scene_feat"]).double()
  W1 = torch.from_numpy(d["W1"]).double().requires_grad_(True); b1 = torch.from_numpy(d["b1"]).double().requires_grad_(True)
  W2 = torch.from_numpy(d["W2"]).double().requires_grad_(True); b2 = torch.from_numpy(d["b2"]).double().requires_grad_(True)
  c1 = torch.tanh(RT.conv2d_same(x, W1, 2) + b1); c2 = torch.tanh(RT.conv2d_same(c1, W2, 2) + b2)
  g1 = rng.standard_normal(tuple(c1.shape)).astype(np.float32); g2 = rng.standard_normal(tuple(c2.shape)).astype(np.float32)
  ((c1 * torch.from_numpy(g1).double()).sum() + (c2 * torch.from_numpy(g2).double()).sum()).backward()
  xd = T(d["scene_feat"], dev)
  o1 = ops.scene_conv_fwd(xd, T(d["W1"], dev), T(d["b1"], dev)); o2 = ops.scene_conv_fwd(o1, T(d["W2"], dev), T(d["b2"], dev))
  d1 = T(g1, dev).clone(); d2 = T(g2, dev)
  dW1 = torch.zeros(3, 3, 11, 64, device=dev); db1 = torch.zeros(64, device=dev)
  dW2 = torch.zeros(3, 3, 64, 64, device=dev); db2 = torch.zeros(64, device=dev)
  ops.scene_conv_bwd(o1, T(d["W2"], dev), o2, d2, dW2, db2, d1)
  ops.scene_conv_bwd(xd, T(d["W1"], dev), o1, d1, dW1, db1, None)
  for a, b in ((dW2, W2), (db2, b2), (dW1, W1), (db1, b1)):
    assert rel(a.cpu().numpy(), b.grad.numpy()) < 2e-5
  # time-mean and one-hot-mask backward are scatters
  idx = T(d["obs_scene"], dev)
  dmean = torch.randn(4, 6, 5, 64, device=dev); ds = torch.zeros_like(o1)
  ops.scene_time_mean_bwd(dmean, idx, ds)
  ref = torch.zeros_like(o1)
  for n in range(4):
    for t in range(8):
      ref[int(idx[n, t])] += dmean[n] / 8
  assert float((ds - ref).abs().max()) < 1e-5


def test_clip_adadelta_matches_tf_formula(dev):
  from multiverse_b200 import ops
  rng = np.random.default_rng(6)
  w = rng.standard_normal(1000); g = rng.standard_normal(1000) * 8
  acc = np.abs(rng.standard_normal(1000)); au = np.abs(rng.standard_normal(1000)) * 1e-3
  lr, rho, eps, clip, wd = 0.3, 0.95, 1e-8, 10.0, 0.001
  gg = np.clip(g * 0.5 + wd * w, -clip, clip)
  a2 = rho * acc + (1 - rho) * gg * gg
  u = np.sqrt(au + eps) / np.sqrt(a2 + eps) * gg
  au2 = rho * au + (1 - rho) * u * u
  w2 = w - lr * u
  tw, tg, ta, tu = [T(v.astype(np.float32), dev) for v in (w, g, acc, au)]
  ops.clip_adadelta(tw, tg, ta, tu, lr, clip, wd, grad_scale=0.5)
  assert rel(tw.cpu().numpy(), w2) < 1e-5 and rel(ta.cpu().numpy(), a2) < 1e-5 and rel(tu.cpu().numpy(), au2) < 1e-4


@pytest.mark.parametrize("use_grids,scene_in_gnn", [([False, True], True), ([True, True], True), ([False, True], False)])
def test_whole_model_loss_and_gradients(dev, use_grids, scene_in_gnn):
  """TrainEngine.loss_and_grads (train-mode forward + loss + hand-written BPTT) against torch
  autograd through the oracle's torch restatement, every trainable variable.  scene_in_gnn=False: SimAug's model
  variant (graph attention of the greedy decoder over h alone)."""
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  over = dict(batch_size=2, use_grids=use_grids, gnn_scene_in_greedy=scene_in_gnn)
  cfg = synthetic.make_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                              clip_gradient_norm=10.0, **over)
  w = synthetic.make_weights(cfg, 31)
  f = synthetic.make_feeds(cfg, 2, 31, with_pred=True)
  rcfg = R.default_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, **over)
  tot, losses, wd, grads = RT.loss_and_grads(rcfg, w, f)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = dict(scene_feat=T(f["scene_feat"], dev), obs_scene=T(f["obs_scene"], dev),
               grid_obs_labels=[T(a, dev) for a in f["grid_obs_labels"]],
               grid_obs_regress=[T(a, dev) for a in f["grid_obs_regress"]],
               grid_pred_labels=[T(a, dev) for a in f["grid_pred_labels"]],
               grid_pred_regress=[T(a, dev) for a in f["grid_pred_regress"]])
  got_losses, got_wd = eng.loss_and_grads(feeds)
  got_losses = got_losses.cpu().numpy()
  assert np.abs(got_losses - np.array(losses)).max() < 1e-4 * max(np.abs(losses))
  assert abs(float(got_wd) - wd) < 1e-5 * wd
  worst = {}
  for k in sorted(grads):
    ref = grads[k] - (cfg.wd * w[k] if k.endswith("/W") else 0.0)     # engine grads exclude the wd term
    e = rel(eng.grads[k].cpu().numpy(), ref)
    worst[k] = e
  bad = {k: v for k, v in worst.items() if v > 1e-3}
  print("worst gradient errors:", sorted(worst.items(), key=lambda kv: -kv[1])[:5])
  assert not bad, bad


def test_trainer_step_through_session_and_micro_batching(dev, monkeypatch):
  """Trainer.step via the shim Session (what code/train.py calls, :253): loss values equal the
  oracle's, parameters move, global_step advances, micro-batched gradients equal full-batch ones."""
  import os, sys, types
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  tf.reset_default_graph()
  over = dict(batch_size=4, use_grids=[False, True])
  cfg = synthetic.make_config(is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                              clip_gradient_norm=10.0, **over)
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname = "m"; args.use_soft_grid_class = False; args.use_gt_grid = False; args.train_w_onehot = True
  args.optimizer = "adadelta"; args.init_lr = 0.2; args.emb_lr = 1.0; args.learning_rate_decay = 0.95
  args.num_epoch_per_decay = 2.0; args.train_num_examples = 100; args.use_cosine_lr = False
  args.mask_grid_regression = False
  w = synthetic.make_weights(cfg, 5); f = synthetic.make_feeds(cfg, 4, 5, with_pred=True)
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  ns = 2
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(4)],
              pred_grid_class=[np.stack([f["grid_pred_labels"][j][i] for j in range(ns)]) for i in range(4)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None])
  for j in range(ns):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  batch = (tuple(range(4)), types.SimpleNamespace(data=data))
  rcfg = R.default_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, **over)
  tot, losses, wd, grads = RT.loss_and_grads(rcfg, w, f)
  with tf.Session() as sess:
    trainer = pred_models.Trainer(model, args)
    loss, _, wd_loss, pgl = trainer.step(sess, batch)
    assert abs(loss - tot) < 1e-4 * abs(tot) and abs(wd_loss - wd) < 1e-5 * wd
    assert np.abs(np.array(pgl) - np.array(losses)).max() < 1e-4 * max(losses)
    assert int(sess.run(model.global_step)) == 1
    # one Adadelta step moved every trained variable, and Saver sees the new values
    moved = model.global_step.owner
    k = "person_pred/decoder_grid_class_1/decoder_rnn/dec_grid_1/kernel"
    new = [v for v in tf.global_variables() if v.name == k + ":0"][0].eval()
    assert np.abs(new - w[k]).max() > 0
  # micro-batched gradients == full-batch gradients
  eng = TrainEngine(cfg, {kk: torch.from_numpy(v) for kk, v in w.items()}, dev, 2)
  feeds = {kk: ([T(a, dev) for a in v] if isinstance(v, list) else T(v, dev)) for kk, v in f.items() if kk != "traj"}
  l_full, _ = eng.loss_and_grads(feeds)
  g_full = eng.flat_grad.clone()
  l_mb, _ = eng.loss_and_grads_chunked(feeds, 2)
  assert float((l_full - l_mb).abs().max()) < 1e-4 * float(l_full.abs().max())
  assert float((g_full - eng.flat_grad).abs().max()) < 2e-4 * float(g_full.abs().max())


def test_simaug_scene_input_gradient_and_attack(dev):
  """SURVEY.md section 8 row f-4 (first part): the gradient of the targeted classification loss with respect to
  the scene features - what SimAug's white_box_attack differentiates (SimAug/code/pred_models.py:96-115) - against
  torch autograd through the oracle, and one FGSM / PGD / mixup pass of the attack's update rule."""
  from types import SimpleNamespace
  from multiverse_b200 import ops, simaug, synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  over = dict(batch_size=2, use_grids=[False, True])
  cfg = synthetic.make_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, clip_gradient_norm=10.0, **over)
  w = synthetic.make_weights(cfg, 31); f = synthetic.make_feeds(cfg, 2, 31, with_pred=True)
  # soft (non one-hot) scene features in (-1, 1): an attacked input is not one-hot any more
  rng = np.random.default_rng(3)
  f["scene_feat"] = np.clip(f["scene_feat"] * 0.8 + rng.uniform(-0.1, 0.1, f["scene_feat"].shape), -1, 1).astype(np.float32)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = {k: ([T(a, dev) for a in v] if isinstance(v, list) else T(v, dev)) for k, v in f.items() if not k.startswith("traj")}
  target = simaug.create_random_target(f["grid_pred_labels"][1], 18 * 9, np.random.default_rng(5))
  assert not (target == f["grid_pred_labels"][1]).any() and target.min() >= 0 and target.max() < 162
  g = simaug.scene_input_grad(eng, feeds, T(target, dev), 1).cpu().numpy().astype(np.float64)
  rcfg = R.default_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, **over)
  g_ref = RT.scene_input_grad(rcfg, w, f, target, 1)
  scale = float((g * g_ref).sum() / (g_ref * g_ref).sum())        # the engine differentiates the MEAN: a positive factor
  assert scale > 0
  err = np.abs(g / scale - g_ref).max() / np.abs(g_ref).max()
  big = np.abs(g_ref) > 1e-3 * np.abs(g_ref).max()
  print("scene input gradient: rel err %.2e, factor %.4g (1/(N*Tp) = %.4g), sign agreement %.5f"
        % (err, scale, 1.0 / target.size, (np.sign(g[big]) == np.sign(g_ref[big])).mean()))
  assert err < 2e-3 and abs(scale * target.size - 1.0) < 1e-3
  assert (np.sign(g[big]) == np.sign(g_ref[big])).mean() > 0.999
  # the attack: FGSM, PGD and mixup keep the reference's bounds and move every pixel the way the sign says
  x = feeds["scene_feat"]
  acfg = SimpleNamespace(use_grids=[False, True], scene_grids=cfg.scene_grids, adv_epsilon=0.1, adv_step_size=0.02,
                         adv_num_iter=3, adv_start_from_clean_prob=1.0, adv_use_fgsm=True, use_mixup=False)
  adv, tl = simaug.white_box_attack(eng, feeds, f["grid_pred_labels"][1], acfg, np.random.default_rng(5))
  assert np.array_equal(tl, target)
  lo = torch.clamp(x - 0.1, -1, 1); hi = torch.clamp(x + 0.1, -1, 1)
  want = torch.minimum(torch.maximum(x - 0.1 * torch.sign(T(g.astype(np.float32), dev)), lo), hi)
  assert torch.equal(adv, want)
  acfg.adv_use_fgsm = False; acfg.adv_start_from_clean_prob = 0.0
  adv_pgd, _ = simaug.white_box_attack(eng, feeds, f["grid_pred_labels"][1], acfg, np.random.default_rng(5))
  assert bool((adv_pgd >= lo).all()) and bool((adv_pgd <= hi).all()) and float((adv_pgd - x).abs().max()) > 0.02
  acfg.adv_use_fgsm = True; acfg.use_mixup = True; acfg.mixup_alpha = 1.0; acfg.mixup_mix_adv = False
  adv_mix, _ = simaug.white_box_attack(eng, feeds, f["grid_pred_labels"][1], acfg, np.random.default_rng(5))
  assert bool(((adv_mix - x).abs() <= 0.1 + 1e-6).all())


@pytest.mark.parametrize("exp", [1, 4, 3])
def test_simaug_against_reference_execution(dev, exp):
  """Row f-4 against the reference itself: multiview_augmentation (and, for experiment 3, the label-mixed training
  objective with focal weights and all its variable gradients) on the GPU vs tests/golden/simaug_multiview.npz, which
  holds what the UNMODIFIED SimAug/code/pred_models.py computes for the same seeded inputs when it is executed on the
  eager TF stand-in (tests/golden/make_golden_simaug.py; tests/test_simaug_reference_cpu.py re-runs it).  SimAug's
  model variant: the greedy decoder's graph attention sees h alone (gnn_scene_in_greedy=False)."""
  from types import SimpleNamespace
  from multiverse_b200 import simaug
  from multiverse_b200.train_engine import TrainEngine
  cfg, w, f, extra, spec = cases.simaug_case()
  g = np.load(os.path.join(ROOT, "tests", "golden", "simaug_multiview.npz"))
  assert str(g["source"]).startswith("reference_exec") and cfg.gnn_scene_in_greedy is False
  n, m, eps = spec["n"], spec["m"], spec["eps"]
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = {k: ([T(a, dev) for a in v] if isinstance(v, list) else T(v, dev)) for k, v in f.items() if not k.startswith("traj")}
  feeds["grid_pred_labels_extra"] = extra["grid_pred_labels_extra"]
  feeds["obs_scene_extra"] = extra["obs_scene_extra"]
  acfg = SimpleNamespace(use_grids=cfg.use_grids, scene_grids=cfg.scene_grids, adv_epsilon=eps,
                         adv_start_from_clean_prob=1.0, multiview_max_num=m, multiview_exp=exp,
                         multiview_use_adv_for_loss=False, multiview_random=False, fl_gamma=2.0, mixup_alpha=1.0,
                         multiview_max_weight_for_first=True)
  draw = SimpleNamespace(beta=lambda a, b: spec["beta_draw"])                 # the injected Beta sample
  out, info = simaug.multiview_augmentation(eng, feeds, acfg, draw)
  assert abs(info["beta_weight"] - float(g["exp%d_beta" % exp])) < 1e-12
  got = out.cpu().numpy().reshape(-1)[::cases.ADV_SAMPLE_STRIDE]
  want = g["exp%d_adv_final_sample" % exp]
  close = np.abs(got - want) <= 1e-6
  print("multiview exp %d vs the reference execution: %.5f of the sampled pixels equal, max diff %.3g"
        % (exp, close.mean(), np.abs(got - want).max()))
  assert close.mean() > 0.999 and np.abs(got - want).max() <= 2 * eps + 1e-6
  if exp != 3:
    return
  assert np.array_equal(info["selected_extra_indices"].cpu().numpy(), g["exp3_selected"])
  assert np.abs(info["focal_loss_weight"].cpu().numpy() - g["exp3_focal"]).max() < 1e-4
  # the training step's objective on the augmented, label-mixed batch (double_weighting on)
  t_obs = cfg.obs_len
  rows = torch.arange(n, device=dev)
  sel = info["selected_extra_indices"].long()
  pick = lambda a: T(np.asarray(a), dev).to(torch.int32)[rows, sel]
  ft = dict(feeds, scene_feat=out, obs_scene=torch.arange(n * t_obs, device=dev, dtype=torch.int32).reshape(n, t_obs))
  ft["mixup"] = dict(beta=info["beta_weight"], obs_labels2=[None, pick(extra["grid_obs_labels_extra"][1])],
                     pred_labels2=[None, pick(extra["grid_pred_labels_extra"][1])], focal=info["focal_loss_weight"])
  losses, _ = eng.loss_and_grads(ft)
  got_l = losses.cpu().numpy()
  assert np.abs(got_l - g["exp3_losses"]).max() < 2e-4 * g["exp3_losses"].max()
  worst = {}
  for k in eng.names:
    key = "exp3_grad_sample/" + k
    if key not in g.files:                     # a variable of the unused scale: the reference never creates it
      assert float(eng.grads[k].abs().max()) == 0.0, k
      continue
    ref = g[key].astype(np.float64)
    if k.endswith("/W"):                       # the golden holds d(total)/dW incl. the weight decay term wd * W
      ref = ref - cfg.wd * w[k].reshape(-1)[::cases.grad_sample_stride(w[k].size)]
    mine = eng.grads[k].reshape(-1)[::cases.grad_sample_stride(eng.grads[k].numel())].cpu().numpy()
    scale = max(float(g["exp3_grad_norms/" + k][2]), 1e-30)
    if float(g["exp3_grad_norms/" + k][2]) == 0:
      assert np.abs(mine).max() == 0
      continue
    worst[k] = float(np.abs(mine - ref).max() / scale)
  print("exp 3 gradients vs the reference execution: worst %s" % sorted(worst.items(), key=lambda kv: -kv[1])[:5])
  # Variables upstream of the scene features see the handful of FGSM tie pixels (input-gradient entries ~0 whose sign
  # fp32 BPTT and fp64 autograd resolve differently, < 0.1 % above): in SimAug's variant the scene reaches the loss
  # through the labelled cells' receptive fields only, and flipping 6 such pixels by 0.14 moves scene_conv1/W by
  # 1.8 %, scene_conv2/W by 1.1 % (measured on the oracle).  Everything else must agree to 2e-3; the exact gradient
  # check of the mixed objective on identical inputs is test_mixup_of_two_views_loss_and_gradients.
  upstream = ("person_pred/scene_conv", "person_pred/encoder_grid_class")
  assert max(v for k, v in worst.items() if not k.startswith(upstream)) < 2e-3, worst
  assert max(v for k, v in worst.items() if k.startswith(upstream)) < 6e-2, worst


@pytest.mark.parametrize("focal,scene_in_gnn", [(False, True), (True, True), (True, False)])
def test_mixup_of_two_views_loss_and_gradients(dev, focal, scene_in_gnn):
  """The label side of SimAug's multiview_exp 3 (SimAug/code/pred_models.py:616-638, :1371-1405): observed class maps
  (encoder input, decoder's first input) and loss labels mixed from two views with weight beta, optional per-sample
  focal weights - loss and every variable gradient against torch autograd on the oracle with the same mix.  One
  sample's two views share a cell at some steps (the single-pixel case of the mixed input)."""
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  n = 3
  over = dict(batch_size=n, use_grids=[False, True], gnn_scene_in_greedy=scene_in_gnn)    # False: SimAug's variant
  cfg = synthetic.make_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, clip_gradient_norm=10.0, **over)
  w = synthetic.make_weights(cfg, 23); f = synthetic.make_feeds(cfg, n, 23, with_pred=True)
  rng = np.random.default_rng(4)
  hw = 18 * 9
  obs2 = rng.integers(0, hw, size=(n, cfg.obs_len)).astype(np.int32)
  pred2 = rng.integers(0, hw, size=(n, cfg.pred_len)).astype(np.int32)
  obs2[0] = f["grid_obs_labels"][1][0]                 # sample 0: both views in the same cells
  pred2[0, ::2] = f["grid_pred_labels"][1][0, ::2]
  mix = dict(beta=0.7, obs_labels2=[None, obs2], pred_labels2=[None, pred2],
             focal=(rng.uniform(0.2, 1.0, n).astype(np.float32) if focal else None))
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = {k: ([T(a, dev) for a in v] if isinstance(v, list) else T(v, dev)) for k, v in f.items() if not k.startswith("traj")}
  feeds["mixup"] = dict(beta=0.7, obs_labels2=[None, T(obs2, dev)], pred_labels2=[None, T(pred2, dev)],
                        focal=None if not focal else T(mix["focal"], dev))
  losses, wd = eng.loss_and_grads(feeds)
  rcfg = R.default_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, **over)
  tot, ref_losses, ref_wd, grads = RT.loss_and_grads(rcfg, w, dict(f, mixup=mix))
  plain = RT.loss_and_grads(rcfg, w, f)[1]
  assert abs(ref_losses[0] - plain[0]) > 1e-3            # the mix changes the objective
  got = losses.cpu().numpy()
  assert np.abs(got - np.array(ref_losses)).max() < 1e-4 * max(ref_losses)
  worst = {}
  for k in eng.names:
    ref = grads[k] - (cfg.wd * w[k] if k.endswith("/W") else 0.0)
    if np.abs(ref).max() == 0:
      assert float(eng.grads[k].abs().max()) == 0
      continue
    worst[k] = rel(eng.grads[k].cpu().numpy(), ref)
  bad = {k: v for k, v in worst.items() if v > 1e-3}
  print("mixup (focal=%s): worst gradient errors %s" % (focal, sorted(worst.items(), key=lambda kv: -kv[1])[:3]))
  assert not bad, bad
  # micro-batched == full batch with the mix sliced along
  g_full = eng.flat_grad.clone()
  l_mb, _ = eng.loss_and_grads_chunked(feeds, 1)
  assert float((losses - l_mb).abs().max()) < 1e-4 * float(losses.abs().max())
  assert float((g_full - eng.flat_grad).abs().max()) < 2e-4 * float(g_full.abs().max())


@pytest.mark.parametrize("mode", ["adv_train", "multiview_train", "standard_aug"])
def test_simaug_training_variants_through_the_dropin_trainer(dev, monkeypatch, mode):
  """SimAug's training-time augmentations behind the reference-facing surface (SimAug/code/pred_models.py:286-325,
  feeds :1517-1555): Trainer.step on a Model whose config switches adv_train / multiview_train / standard_aug on.
  With epsilon = 0 every augmentation is the identity, so the step must reproduce the plain step's losses; with
  epsilon > 0 the losses change, stay finite and the variables move."""
  import sys, types
  from multiverse_b200 import synthetic
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  n, m = 2, 3
  over = dict(batch_size=n, use_grids=[False, True])
  cfg = synthetic.make_config(is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                              clip_gradient_norm=10.0, **over)
  w = synthetic.make_weights(cfg, 6); f = synthetic.make_feeds(cfg, n, 6, with_pred=True)
  rng = np.random.default_rng(2)
  ns = 2
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(n)],
              pred_grid_class=[np.stack([f["grid_pred_labels"][j][i] for j in range(ns)]) for i in range(n)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None])
  for j in range(ns):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  # the other camera views: same geometry, labels of their own, frames drawn from the batch's frame set
  data["extra"] = []
  for i in range(n):
    ex = dict(obs_grid_class=[], pred_grid_class=[])
    for j, (h, ww) in enumerate(cfg.scene_grids):
      ex["obs_grid_target_all_%d" % j] = [f["grid_obs_regress"][j][i]] * m
      ex["pred_grid_target_all_%d" % j] = [f["grid_pred_regress"][j][i]] * m
    for k in range(m):
      ex["obs_grid_class"].append(np.stack([rng.integers(0, h * ww, cfg.obs_len) for (h, ww) in cfg.scene_grids]))
      ex["pred_grid_class"].append(np.stack([rng.integers(0, h * ww, cfg.pred_len) for (h, ww) in cfg.scene_grids]))
    data["extra"].append(ex)
  data["batch_extra_obs_scene"] = rng.integers(0, f["scene_feat"].shape[0], size=(n, m, cfg.obs_len, 1))
  batch = (tuple(range(n)), types.SimpleNamespace(data=data))

  def run(eps, **flags):
    for mod in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
      sys.modules.pop(mod, None)
    import tensorflow as tf
    import pred_models
    tf.reset_default_graph()
    args = types.SimpleNamespace(**vars(cfg))
    args.modelname = "m"; args.use_soft_grid_class = False; args.use_gt_grid = False; args.train_w_onehot = True
    args.optimizer = "adadelta"; args.init_lr = 0.2; args.emb_lr = 1.0; args.learning_rate_decay = 0.95
    args.num_epoch_per_decay = 2.0; args.train_num_examples = 100; args.use_cosine_lr = False
    args.mask_grid_regression = False
    args.adv_epsilon, args.adv_step_size, args.adv_num_iter, args.adv_use_fgsm = eps, eps / 4, 2, True
    args.adv_start_from_clean_prob, args.use_mixup, args.mixup_alpha, args.norm_feat = 0.0, False, 1.0, False
    args.multiview_max_num, args.multiview_exp, args.multiview_max_weight_for_first, args.seed = m, 1, True, 11
    for k, v in flags.items():
      setattr(args, k, v)
    model = pred_models.get_model(args, gpuid=0)
    tf.global_variables_initializer().run()
    for v in tf.global_variables():
      if v.name.split(":")[0] in w:
        v.assign(w[v.name.split(":")[0]])
    with tf.Session() as sess:
      trainer = pred_models.Trainer(model, args)
      loss, _, wd_loss, pgl = trainer.step(sess, batch)
      k = "person_pred/decoder_grid_class_1/decoder_rnn/dec_grid_1/kernel"
      new = [v for v in tf.global_variables() if v.name == k + ":0"][0].eval()
    return float(loss), np.array(pgl, dtype=np.float64), new

  # a config that carries SimAug's flags selects SimAug's model variant (graph attention of the greedy decoder over
  # h alone); the plain run is given the same variant explicitly
  plain = run(0.0, gnn_scene_in_greedy=False)
  kw = {mode: True}
  if mode == "standard_aug":        # not one of the two flags that mark a SimAug config: name the variant
    kw["gnn_scene_in_greedy"] = False
  same = run(0.0, **kw)
  assert abs(same[0] - plain[0]) < 1e-6 * abs(plain[0]) and np.allclose(same[1], plain[1], rtol=1e-6)
  aug = run(0.1, **kw)
  assert np.isfinite(aug[0]) and np.isfinite(aug[1]).all() and abs(aug[0] - plain[0]) > 1e-6
  assert np.abs(aug[2] - w["person_pred/decoder_grid_class_1/decoder_rnn/dec_grid_1/kernel"]).max() > 0
  if mode == "multiview_train":      # experiment 3: label mixing and focal weights on top of the feature mix
    exp3 = run(0.1, multiview_train=True, multiview_exp=3, double_weighting=True, fl_gamma=2.0,
               multiview_use_adv_for_loss=False, multiview_random=False)
    assert np.isfinite(exp3[0]) and abs(exp3[0] - aug[0]) > 1e-6


@pytest.mark.parametrize("exp", [1, 4, 2, 3])
def test_simaug_multiview_augmentation(dev, exp):
  """Row f-4, second part: SimAug's multiview_augmentation (SimAug/code/pred_models.py:346-541) - the batch tiled over
  M camera views, one FGSM step per view against that view's labels, views ranked by their per-sample classification
  loss, two picked per multiview_exp and mixed - against the same pipeline written with the oracle's autograd
  gradient and per-sample losses."""
  from types import SimpleNamespace
  from multiverse_b200 import simaug, synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  n, m = 2, 3
  over = dict(use_grids=[False, True])
  cfg = synthetic.make_config(batch_size=n, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                              clip_gradient_norm=10.0, **over)
  w = synthetic.make_weights(cfg, 41); f = synthetic.make_feeds(cfg, n, 41, with_pred=True)
  rng = np.random.default_rng(9)
  f["scene_feat"] = np.clip(f["scene_feat"] * 0.8 + rng.uniform(-0.1, 0.1, f["scene_feat"].shape), -1, 1).astype(np.float32)
  t_obs, tp, hw = cfg.obs_len, cfg.pred_len, 18 * 9
  extra_labels = rng.integers(0, hw, size=(n, m, tp)).astype(np.int32)
  extra_scene = rng.integers(0, f["scene_feat"].shape[0], size=(n, m, t_obs)).astype(np.int32)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = {k: ([T(a, dev) for a in v] if isinstance(v, list) else T(v, dev)) for k, v in f.items() if not k.startswith("traj")}
  feeds["grid_pred_labels_extra"] = [None, extra_labels]
  feeds["obs_scene_extra"] = extra_scene
  eps = 0.1
  acfg = SimpleNamespace(use_grids=[False, True], scene_grids=cfg.scene_grids, adv_epsilon=eps,
                         adv_start_from_clean_prob=1.0, multiview_max_num=m, multiview_exp=exp,
                         multiview_use_adv_for_loss=False, multiview_random=False, fl_gamma=2.0, mixup_alpha=1.0,
                         multiview_max_weight_for_first=True)
  out, info = simaug.multiview_augmentation(eng, feeds, acfg, np.random.default_rng(17))
  # ---- the same pipeline on the oracle: tiled feeds, autograd gradient, per-sample losses
  tile = lambda a: np.repeat(np.asarray(a), m, axis=0)
  clean = f["scene_feat"][f["obs_scene"]]                                   # [N,T,SH,SW,SC]
  tf = dict(scene_feat=tile(clean).reshape((n * m * t_obs,) + clean.shape[2:]),
            obs_scene=np.arange(n * m * t_obs, dtype=np.int32).reshape(n * m, t_obs))
  for key in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    tf[key] = [None if a is None else tile(a) for a in f[key]]
  target = extra_labels.reshape(n * m, tp)
  rcfg = R.default_config(batch_size=n * m, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, **over)
  g_ref, loss_ref = RT.scene_input_grad(rcfg, w, tf, target, 1, per_sample=True)
  loss_ref = loss_ref.reshape(n, m)
  got_loss = info["adv_loss"].cpu().numpy()
  assert np.abs(got_loss - loss_ref).max() / np.abs(loss_ref).max() < 1e-4
  order_ref = np.argsort(-loss_ref, axis=1, kind="stable")
  gaps = np.abs(np.diff(np.sort(loss_ref, axis=1), axis=1)).min()
  assert gaps > 1e-3, "degenerate test data: view losses too close to rank"
  assert np.array_equal(info["loss_indices"].cpu().numpy(), order_ref)
  x = tf["scene_feat"].astype(np.float32)
  lo, hi = np.clip(x - np.float32(eps), -1, 1), np.clip(x + np.float32(eps), -1, 1)
  adv_ref = np.minimum(np.maximum(x - np.float32(eps) * np.sign(g_ref).astype(np.float32), lo), hi)
  adv_ref = adv_ref.reshape((n, m, t_obs) + clean.shape[2:])
  rows = np.arange(n)
  r2 = np.random.default_rng(17)
  if exp == 1:
    f1, f2 = adv_ref[rows, order_ref[:, 0]], adv_ref[rows, order_ref[:, 1]]
  elif exp == 4:
    f1, f2 = adv_ref[rows, order_ref[:, m - 1]], adv_ref[rows, order_ref[:, m - 2]]
  elif exp == 2:
    a = r2.integers(0, m, size=n); b = (a + r2.integers(1, m, size=n)) % m
    assert (a != b).all()
    f1, f2 = adv_ref[rows, a], adv_ref[rows, b]
  else:
    f1 = adv_ref[rows, order_ref[:, 0]]
    f2 = f["scene_feat"][extra_scene[rows, order_ref[:, 0]]]
    assert np.array_equal(info["selected_extra_indices"].cpu().numpy(), order_ref[:, 0])
    fl = (1.0 - np.exp(-np.sort(loss_ref, axis=1)[:, -1])) ** 2.0
    assert np.abs(info["focal_loss_weight"].cpu().numpy() - fl).max() < 1e-4
  wgt = r2.beta(1.0, 1.0); wgt = max(wgt, 1.0 - wgt)
  assert abs(info["beta_weight"] - wgt) < 1e-12 and wgt >= 0.5
  want = (f1 * np.float32(wgt) + f2 * (np.float32(1.0) - np.float32(wgt))).reshape((n * t_obs,) + clean.shape[2:])
  got = out.cpu().numpy()
  assert got.shape == want.shape
  # the sign of a gradient entry that is ~0 next to the others may differ between fp32 BPTT and fp64 autograd
  close = np.abs(got - want) <= 1e-6
  print("multiview exp %d: %.5f of the pixels equal, max diff %.3g" % (exp, close.mean(), np.abs(got - want).max()))
  assert close.mean() > 0.999 and np.abs(got - want).max() <= 2 * eps + 1e-6


@pytest.mark.parametrize("opt", ["momentum", "adam", "rmsprop"])
def test_other_optimizers_match_tf_semantics(dev, opt):
  """Trainer's non-default optimizers (code/pred_models.py:1667-1681) - MomentumOptimizer(lr, 0.9), AdamOptimizer(lr),
  RMSPropOptimizer(lr) - fused with weight decay, 1/G scaling and the element-wise clip (mvb_clip_update), three steps
  against the optimizer classes of the eager TF-1.15 stand-in (oracle/tf1_eager: python/training/{momentum,adam,
  rmsprop}.py restated) and against closed forms."""
  import sys
  from multiverse_b200 import ops
  sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_eager"))
  saved = {k: v for k, v in sys.modules.items() if k == "tensorflow" or k.startswith("tensorflow.")}
  for k in saved:
    del sys.modules[k]
  try:
    import tensorflow as tfe
    assert tfe.__version__.endswith("eager-standin")
  finally:
    sys.path.remove(os.path.join(ROOT, "oracle", "tf1_eager"))
    for k in [k for k in sys.modules if k == "tensorflow" or k.startswith("tensorflow.")]:
      del sys.modules[k]
    sys.modules.update(saved)
  rng = np.random.default_rng(8)
  n, lr, clip, wd, gs = 4096, 0.05, 10.0, 0.001, 0.5
  w0 = rng.standard_normal(n); grads = [rng.standard_normal(n) * 8 for _ in range(3)]
  tfe.reset_default_graph()
  var = tfe.Variable(torch.from_numpy(w0.copy()), "w", True)
  O = dict(momentum=lambda: tfe.train.MomentumOptimizer(lr, momentum=0.9), adam=lambda: tfe.train.AdamOptimizer(lr),
           rmsprop=lambda: tfe.train.RMSPropOptimizer(lr))[opt]()
  tw = T(w0.astype(np.float32), dev)
  s1 = torch.ones_like(tw) if opt == "rmsprop" else torch.zeros_like(tw)
  s2 = torch.zeros_like(tw)
  for t, g in enumerate(grads, 1):
    gg = np.clip(g * gs + wd * var.numpy(), -clip, clip)                    # what Trainer hands to apply_gradients
    O.apply_gradients([(tfe.Tensor(torch.from_numpy(gg)), var)]).run()
    kind, p1, p2, eps = dict(momentum=(1, 0.9, 0.0, 0.0), adam=(2, 0.9, 0.999, 1e-8), rmsprop=(3, 0.9, 0.0, 1e-10))[opt]
    lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) if opt == "adam" else lr
    ops.clip_update(tw, T(g.astype(np.float32), dev), s1, s2, kind, lr_t, p1, p2, eps, clip, wd, grad_scale=gs)
    err = np.abs(tw.cpu().numpy() - var.numpy()).max() / np.abs(var.numpy()).max()
    assert err < 2e-5, (opt, t, err)
