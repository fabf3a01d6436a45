# coding=utf-8
"""Training from trajectories (SURVEY.md §8 row f-1, training half): the kernels that compute the regression encoder's
input, the regression targets and the soft label maps from the trajectories, the grid centres and the label cells
(traj_to_planes, huber_traj_fwd_bwd, soft_ce_label_fwd_bwd, fg_count_label, masked_huber_traj_fwd_bwd) against their
dense counterparts fed the tensors the host builds from the same data, and whole training steps fed either way.

Every element a kernel writes - operand planes, dlogits, dreg, the foreground count - must be byte-identical.  The
loss sums are accumulated in fp32 with one atomic per block in no fixed order by both forms (and by two runs of the
same form), so they are compared to ATOL_SUM.  A whole training step adds the atomics of head_bwd / emb_bwd, whose
order differs from run to run; its losses, gradients and updated variables are compared to ATOL_SUM of their largest
element after every tensor the backward consumes (logits, offsets, their gradients, the operand planes) has been
found byte-identical."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from multiverse_b200 import ops, synthetic
from multiverse_b200.pred_models import _soft_labels

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS, T_OBS, T_PRED = 128, 8, 12                 # the training micro-batch
GRIDS = [(18, 32), (9, 16)]                    # the published scene 36x64, strides 2,4
GRID_IDS = ["%dx%d" % g for g in GRIDS]
VIDEO_H, VIDEO_W = 1080, 1920
MODES = list(range(1, 8))
ATOL_SUM = 1e-5        # relative: sums whose order of fp32 atomic additions varies (measured up to 1.2e-6 on an H100)


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import _lib, build
  build.build()
  _lib.load()
  return torch.device("cuda", 0)


def centres(h, w):
  hg, wg = VIDEO_H * 1.0 / h, VIDEO_W * 1.0 / w
  return np.stack(np.meshgrid((np.arange(w) + 0.5) * wg, (np.arange(h) + 0.5) * hg), axis=-1)     # [h,w,2] (x,y)


def points(n, t, seed):
  """fp64 [n,t,2] frame pixels; the first rows sit in the corners and on the edges of the frame."""
  rng = np.random.default_rng(seed)
  p = rng.uniform([0.0, 0.0], [VIDEO_W, VIDEO_H], size=(n, t, 2))
  p[0], p[1], p[2], p[3] = [0.0, 0.0], [VIDEO_W, VIDEO_H], [VIDEO_W - 0.5, 0.5], [0.5, VIDEO_H - 0.5]
  return p


def label_cells(tn, h, w, seed, negative=True):
  """int32 [Tp,N] label cells: random, every corner and edge midpoint, and (soft maps) negative labels, which the
  host's numpy indexing counts from the end."""
  rng = np.random.default_rng(seed)
  lab = rng.integers(0, h * w, size=tn).astype(np.int32)
  edge = [0, w - 1, (h - 1) * w, h * w - 1, w // 2, (h // 2) * w, (h // 2) * w + w - 1, (h - 1) * w + w // 2]
  lab[0, :len(edge)] = edge
  lab[1, :len(edge)] = edge[::-1]
  if negative:
    lab[2, :4] = [-1, -w, -h * w, -(h * w) // 2]
  return lab


def g(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel(a, b):
  return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def same_bytes(a, b):
  return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                    b.contiguous().view(torch.uint8))


# --------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("comp", [True, False], ids=["comp", "plain"])
@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_traj_to_planes_equals_nhwc_to_planes(dev, grid, comp):
  h, w = grid
  obs, c = points(NS, T_OBS, 1), centres(h, w)
  cpad = ops.cell_cpad(2)
  for t in range(T_OBS):
    dense = g((obs[:, t, None, None, :] - c[None]).astype(np.float32), dev)      # [NS,h,w,2]
    a = ops.alloc_xh(NS, h, w, cpad, ops.PLANES_BF16X2, dev)
    b = ops.alloc_xh(NS, h, w, cpad, ops.PLANES_BF16X2, dev)
    a.fill_(-7.0); b.fill_(-7.0)                 # what neither writes must stay
    ops.nhwc_to_planes(dense, a, 0, h, w, comp=comp)
    ops.traj_to_planes(g(obs, dev), t, g(c, dev), b, h, w, comp=comp)
    torch.cuda.synchronize()
    assert same_bytes(a, b), t


def dense_targets(pred, c):
  """fp32 [Tp,N,HW,2]: the host's grid_pred_regress, transposed as the training step reads it."""
  n, tp = pred.shape[:2]
  return (pred[:, :, None, None, :] - c[None, None]).astype(np.float32).transpose(1, 0, 2, 3, 4).reshape(tp, n, -1, 2)


def offsets_near(tgt, seed):
  """Predicted offsets around the targets: both branches of the Huber loss."""
  rng = np.random.default_rng(seed)
  return (tgt + rng.normal(0.0, 1.5, size=tgt.shape)).astype(np.float32)


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_huber_traj_equals_dense(dev, grid):
  h, w = grid
  pred, c = points(NS, T_PRED, 2), centres(h, w)
  tgt = dense_targets(pred, c)
  reg = g(offsets_near(tgt, 3), dev)
  da, db = torch.empty_like(reg), torch.empty_like(reg)
  la, lb = torch.zeros(2, device=dev), torch.zeros(2, device=dev)
  ops.loss_fwd_bwd(None, None, None, 0.0, reg, g(tgt, dev), da, 0.2, la)
  ops.huber_traj_fwd_bwd(reg, g(pred, dev), g(c, dev), db, 0.2, lb)
  torch.cuda.synchronize()
  assert same_bytes(da, db)
  assert float(lb[0]) == 0.0 and rel(lb[1:], la[1:]) < ATOL_SUM


def soft_maps(lab, h, w, mode):
  """[Tp,N,HW] fp32: pred_models._soft_labels of every label cell."""
  tp, n = lab.shape
  return _soft_labels(lab, h, w, mode).reshape(tp, n, h * w)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_soft_ce_label_equals_dense_maps(dev, grid, mode):
  h, w = grid
  lab = label_cells((T_PRED, NS), h, w, 4)
  logits = g(np.random.default_rng(5).normal(0, 3, size=(T_PRED, NS, h * w)).astype(np.float32), dev)
  da, db = torch.empty_like(logits), torch.empty_like(logits)
  la, lb = torch.zeros(2, device=dev), torch.zeros(2, device=dev)
  ops.soft_ce_fwd_bwd(logits, g(soft_maps(lab, h, w, mode), dev), da, 1.0, la)
  ops.soft_ce_label_fwd_bwd(logits, g(lab, dev), mode, h, w, db, 1.0, lb)
  torch.cuda.synchronize()
  assert same_bytes(da, db)
  assert float(lb[1]) == 0.0 and rel(lb[:1], la[:1]) < ATOL_SUM


@pytest.mark.parametrize("mode", [0] + MODES)
@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_fg_count_and_masked_huber_equal_dense(dev, grid, mode):
  """mode 0: sparse labels (the label cell of each row; out-of-range labels have no foreground); 1-7: soft maps."""
  h, w = grid
  pred, c = points(NS, T_PRED, 6), centres(h, w)
  lab = label_cells((T_PRED, NS), h, w, 7, negative=bool(mode))
  if not mode:
    lab[3, :5] = [-1, h * w, h * w + 9, -h * w, 1 << 30]
  tgt = dense_targets(pred, c)
  reg = g(offsets_near(tgt, 8), dev)
  lab_d = g(lab, dev)
  dense_lab = g(soft_maps(lab, h, w, mode), dev) if mode else lab_d
  ka, kb = torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.float64, device=dev)
  ops.fg_count(dense_lab, h * w, ka)
  ops.fg_count_label(lab_d, mode, h, w, kb)
  torch.cuda.synchronize()
  assert float(ka) > 0 and same_bytes(ka, kb)
  zero = torch.zeros(1, dtype=torch.float64, device=dev)
  for count_a, count_b in ((ka, kb), (zero, zero)):         # K = 0: zero loss and gradient (div_no_nan)
    da, db = torch.full_like(reg, 5.0), torch.full_like(reg, 5.0)
    la, lb = torch.zeros(2, device=dev), torch.zeros(2, device=dev)
    ops.masked_huber_fwd_bwd(reg, g(tgt, dev), da, dense_lab, count_a, 0.1, la)
    ops.masked_huber_traj_fwd_bwd(reg, g(pred, dev), g(c, dev), db, lab_d, mode, h, w, count_b, 0.1, lb)
    torch.cuda.synchronize()
    assert same_bytes(da, db)
    if count_a is zero:
      assert float(la[1]) == 0.0 and float(lb[1]) == 0.0 and not bool(db.any())
    else:
      assert rel(lb[1:], la[1:]) < ATOL_SUM


def test_sparse_labels_without_foreground(dev):
  """K = 0 from the labels themselves: no label cell lies in the grid."""
  h, w = GRIDS[1]
  lab = g(np.full((T_PRED, NS), h * w, dtype=np.int32), dev)
  ka, kb = torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.float64, device=dev)
  ops.fg_count(lab, h * w, ka)
  ops.fg_count_label(lab, 0, h, w, kb)
  assert float(ka) == 0.0 and float(kb) == 0.0


# --------------------------------------------------------------------------- whole training steps
def engine_tensors(eng, cfg, n):
  """Every tensor the backward consumes, per used scale (engine buffers of the last micro-batch, cloned)."""
  out = {}
  for i, _ in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      continue
    for key in ("logits", "offs", "dlogits", "doffs"):
      out[(key, i)] = eng._store[(key, i, n)][0].clone()
    for key in ("xh_er", "xh_dr", "xh_dc"):
      for t, x in enumerate(eng._store[(key, i, n)]):
        out[(key, i, t)] = x.clone()
  return out


def state_of(eng, losses):
  return dict(losses=torch.as_tensor(np.asarray(losses, dtype=np.float64)),
              grad=eng.flat_grad.clone(), params=torch.cat([eng.params[k].reshape(-1) for k in eng.names]).clone())


def check_equal(dense, traj, tag):
  ta, tb = dense["tensors"], traj["tensors"]
  assert set(ta) == set(tb)
  for k in ta:
    assert same_bytes(ta[k], tb[k]), (tag, k)
  for k in ("losses", "grad", "params"):
    e = rel(traj[k], dense[k])
    assert e < ATOL_SUM, (tag, k, e)
  print("%s: %d consumed tensors byte-identical; losses/gradients/variables relative differences %s" % (
      tag, len(ta), ["%.2e" % rel(traj[k], dense[k]) for k in ("losses", "grad", "params")]))


FLAG_SETS = {
    # code/train.py's defaults with its multi-future flags: scene 36x64, strides 2,4,8, emb 128, no scene encoder
    "train_py_multifuture": (dict(scene_h=36, scene_w=64, scene_grid_strides=[2, 4, 8], use_grids=[True, True, True],
                                  emb_size=128, use_scene_enc=False, grid_reg_loss_weight=0.1),
                             dict(use_soft_grid_class=True, soft_grid=1, mask_grid_regression=True,
                                  train_w_onehot=False, init_lr=0.2)),
    # TRAINING.md: scene 36x64, strides 2,4, both grids, --train_w_onehot, loss weights 1.0 / 0.2, --init_lr 0.3
    "training_md": (dict(scene_h=36, scene_w=64, scene_grid_strides=[2, 4], use_grids=[True, True],
                         grid_reg_loss_weight=0.2),
                    dict(use_soft_grid_class=False, soft_grid=1, mask_grid_regression=False, train_w_onehot=True,
                         init_lr=0.3)),
}


def dropin_model(monkeypatch, n, over, flags):
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  tf.reset_default_graph()
  cfg = synthetic.make_config(batch_size=n, is_train=True, grid_loss_weight=1.0, wd=0.001, clip_gradient_norm=10.0,
                              **over)
  args = types.SimpleNamespace(**vars(cfg))
  args.modelname = "m"; args.use_gt_grid = False; args.use_teacher_forcing = False
  args.optimizer = "adadelta"; args.emb_lr = 1.0; args.learning_rate_decay = 0.95
  args.num_epoch_per_decay = 2.0; args.train_num_examples = 100; args.use_cosine_lr = False
  for k, v in flags.items():
    setattr(args, k, v)
  w = synthetic.make_weights(cfg, 11)
  f = synthetic.make_feeds(cfg, n, 11, with_pred=True)
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  ns, t = len(cfg.scene_grids), cfg.obs_len
  pred_cls = []
  for j, (h, ww) in enumerate(cfg.scene_grids):    # label cells in the corners and on the edges of every grid
    lab = np.array(f["grid_pred_labels"][j])
    lab[:2] = label_cells((2, T_PRED), h, ww, 13, negative=False)
    pred_cls.append(lab)
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(ns)]) for i in range(n)],
              pred_grid_class=[np.stack([pred_cls[j][i] for j in range(ns)]) for i in range(n)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None],
              obs_traj=list(f["traj64"][:, :t]), pred_traj=list(f["traj64"][:, t:]))
  for j in range(ns):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  shared = {"grid_center_%d" % j: c for j, c in enumerate(synthetic.grid_centers(cfg))}
  return tf, pred_models, model, args, cfg, types.SimpleNamespace(data=data, shared=shared)


@pytest.mark.parametrize("flagset", sorted(FLAG_SETS))
def test_trainer_step_from_trajectories_equals_dense(dev, monkeypatch, flagset):
  """One Trainer.step on trajectory feeds against the same step on the reference's dense feed dict, from the same
  weights and optimizer state."""
  over, flags = FLAG_SETS[flagset]
  n = 8
  tf, pred_models, model, args, cfg, batch = dropin_model(monkeypatch, n, over, flags)
  dense_fd = model.get_feed_dict(batch, is_train=True)
  traj_fd = model.get_feed_dict(batch, is_train=True, train_traj=True)
  used = [j for j in range(len(cfg.scene_grids)) if cfg.use_grids[j]]
  assert all(model.grid_obs_regress[j] in dense_fd for j in used)
  # the trajectory feed dict holds no dense offset, target or label map
  assert model.obs_traj in traj_fd and model.pred_traj in traj_fd
  for j in used:
    assert model.grid_obs_regress[j] not in traj_fd and model.grid_pred_regress[j] not in traj_fd
    lab = traj_fd[model.grid_pred_labels_T[j]]
    assert lab.dtype == np.int32 and lab.shape == (n, cfg.pred_len)
  assert max(np.asarray(v).nbytes for v in traj_fd.values() if isinstance(v, np.ndarray)
             and v is not traj_fd[model.scene_feat]) < 64 * 1024
  trainer = pred_models.Trainer(model, args)
  eng = model._ensure_engine()
  start = {k: v.clone() for k, v in eng.params.items()}
  fetches = [model.loss, trainer.train_op, model.wd_loss, model.pred_grid_loss]
  runs = {}
  with tf.Session() as sess:
    for name, fd in (("dense", dense_fd), ("traj", traj_fd)):
      for k in eng.names:
        eng.params[k].copy_(start[k]); eng.acc[k].zero_(); eng.acc_upd[k].zero_()
      eng._repack()
      model.global_step.value = np.asarray(0, dtype="int32")
      if name == "traj":                          # the step's device feeds: no dense tensor goes to the device
        feeds = model._device_feeds(fd, train_traj=True)
        assert all(a is None for a in feeds["grid_obs_regress"]) and "traj" in feeds
      loss, _, wd_loss, pgl = sess.run(fetches, fd)
      torch.cuda.synchronize()
      runs[name] = state_of(eng, [loss, wd_loss] + list(pgl))
      runs[name]["tensors"] = engine_tensors(eng, cfg, n)
      assert int(sess.run(model.global_step)) == 1
  check_equal(runs["dense"], runs["traj"], flagset)


def test_micro_batched_step_from_trajectories_equals_dense(dev):
  """TrainEngine.train_step over 256 rows in micro-batches of 128 on 18x32 + 9x16 with soft labels (mode 7) and the
  masked regression: the foreground count of the whole batch, the chunked trajectory feeds and every micro-batch's
  consumed tensors equal the dense feeds'."""
  from multiverse_b200.train_engine import TrainEngine
  n, mb, mode = 2 * NS, NS, 7
  cfg = synthetic.make_config(batch_size=mb, is_train=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                              clip_gradient_norm=10.0, scene_h=36, scene_w=64, scene_grid_strides=[2, 4],
                              use_grids=[True, True])
  cfg.mask_grid_regression, cfg.train_w_onehot = True, False
  w = synthetic.make_weights(cfg, 17)
  f = synthetic.make_feeds(cfg, n, 17, with_pred=True)
  labels = [np.ascontiguousarray(label_cells((T_PRED, n), h, ww, 19 + j).T) for j, (h, ww) in
            enumerate(cfg.scene_grids)]                                                       # [N,Tp]
  base = dict(scene_feat=g(f["scene_feat"], dev), obs_scene=g(f["obs_scene"], dev),
              grid_obs_labels=[g(a, dev) for a in f["grid_obs_labels"]])
  dense = dict(base, grid_obs_regress=[g(a, dev) for a in f["grid_obs_regress"]],
               grid_pred_regress=[g(a, dev) for a in f["grid_pred_regress"]],
               grid_pred_labels=[g(_soft_labels(a, h, ww, mode), dev) for a, (h, ww) in zip(labels, cfg.scene_grids)])
  traj = dict(base, grid_obs_regress=[None, None], grid_pred_regress=[None, None],
              grid_pred_labels=[g(a, dev) for a in labels],
              traj=dict(obs=g(f["traj64"][:, :cfg.obs_len], dev), pred=g(f["traj64"][:, cfg.obs_len:], dev),
                        centers=[g(c, dev) for c in synthetic.grid_centers(cfg)], soft_grid=mode))
  runs = {}
  for name, feeds in (("dense", dense), ("traj", traj)):
    eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev)
    K = eng.fg_counts(feeds)
    losses, _ = eng.train_step(feeds, 0.2, None, micro_batch=mb)
    torch.cuda.synchronize()
    runs[name] = state_of(eng, losses.cpu().numpy())
    runs[name]["tensors"] = engine_tensors(eng, cfg, mb)
    runs[name]["tensors"][("K",)] = K
    del eng
  check_equal(runs["dense"], runs["traj"], "micro-batch 128 of 256, soft_grid 7 + mask")
