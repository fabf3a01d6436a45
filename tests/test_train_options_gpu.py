# coding=utf-8
"""The training options of code/train.py:85-92 that the training step supports beyond the published command:
soft grid-class labels (--use_soft_grid_class --soft_grid k), the masked regression loss (--mask_grid_regression) and
the logits-fed class decoder (training without --train_w_onehot, the train.py default).

Kernels, element by element at the training micro-batch (128 trajectories on 36x18 and 18x9), against plain fp64
torch on the device (the reference functions of test_train_atsize_gpu.py):
  - soft_ce_fwd_bwd for the label maps of all seven modes, label cells in the corners, on the edges and inside, so
    the row sums of the maps differ;
  - fg_count + masked_huber_fwd_bwd with sparse and soft foregrounds, |e| on both sides of 1, a micro-batch divided
    by the count of its whole batch, and K = 0;
  - head_class_fwd_dense: the embedded logits map as the next step's x planes, halo rows and the h block untouched;
  - emb_bwd on a dense one-channel input, d_in accumulating over 12 steps.
The whole model: TrainEngine.loss_and_grads_chunked on 256 trajectories in micro-batches of 128 against the fp64
truth of tests/train_options_ref.py for every option, at the bars of test_train_atsize_gpu.py; chunked equals
unchunked for soft labels + mask (128 trajectories in micro-batches of 64).  The drop-in: train.py-shaped arguments
with each flag run Trainer.step; on the inputs of every reference-execution golden (tests/golden/refexec_train_*.npz,
and refexec_native.npz with TRAINING.md's arguments: scene 36x64, both scales, loss weights 1.0 / 0.2, init_lr 0.3)
one Trainer.step equals the unmodified reference Model + Trainer in losses, clipped gradients and updated variables;
the combinations that stay unimplemented raise."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import cases
import train_options_ref as TO
from test_kernels_atsize_gpu import halo_rows, inner, rel, to_halo
from test_train_atsize_gpu import (E, FRAMES, FTOL, GRIDS, GTOL, LTOL, MARGIN, NS, PTOL, SENTINEL, T_PRED, WM_SEED,
                                   gen, head_inputs, on, ref_emb, ref_head, ref_onehot, shared_frame_feeds, vjp,
                                   wm_configs)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_train_options as G  # noqa: E402  (the golden cases and their inputs)


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def edge_cells(h, w):
  """Corners, edge midpoints and interior cells: the soft maps are clipped differently at each."""
  return [0, w - 1, (h - 1) * w, h * w - 1, w // 2, (h // 2) * w, (h // 2) * w + w - 1, (h - 1) * w + w // 2,
          1, w + 1, (h // 2) * w + w // 2]


def soft_maps(cls, h, w, mode):
  from multiverse_b200.pred_models import _soft_labels
  return _soft_labels(cls, h, w, mode)


def ref_soft_ce(logits, y):
  """Mean over rows of softmax_cross_entropy_with_logits(labels=y, logits)."""
  lg = logits.reshape(-1, logits.shape[-1])
  return (-(y.reshape(lg.shape) * torch.log_softmax(lg, -1)).sum(-1)).mean()


def ref_masked_huber(pred, target, fg, k):
  """Huber over the gathered foreground rows of pred / target [cells, 2], summed / (2k)."""
  a = (pred.reshape(-1, 2)[fg] - target.reshape(-1, 2)[fg]).abs()
  return torch.where(a <= 1.0, 0.5 * a * a, a - 0.5).sum() / (2 * k) if k else pred.sum() * 0.0


# --------------------------------------------------------------------------- loss kernels
@pytest.mark.gpu
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_soft_ce_every_mode(dev, grid):
  """soft_ce_fwd_bwd on [12, 128, V] logits against the maps of modes 1-7 (whose sums are 1.8 / 1.08 / ... inside
  and less where the kernel is clipped); the gradient is sum(y) softmax - y, not softmax - y."""
  from multiverse_b200 import ops
  h, w = grid
  v = h * w
  g = gen(dev, 500 + h)
  lg = torch.randn((T_PRED, NS, v), generator=g, device=dev) * 3
  rng = np.random.default_rng(h)
  cls = rng.integers(0, v, size=(NS, T_PRED))
  cells = edge_cells(h, w)
  cls[:len(cells), 0] = cells
  cls[0, :len(cells)] = cells
  cw = 0.5
  one = torch.ones((), dtype=torch.float64, device=dev)
  errs = {}
  for mode in range(1, 8):
    y = on(dev, soft_maps(cls, h, w, mode)).reshape(NS, T_PRED, v).transpose(0, 1).contiguous()
    sums = y.sum(-1)
    assert float(sums.max() - sums.min()) > 0.04, "no row whose label mass differs"
    ce, (dce,) = vjp(lambda a: ref_soft_ce(a, y.double()) * cw, [lg], one)
    dl = torch.full_like(lg, SENTINEL)
    out = torch.zeros(2, device=dev)
    ops.soft_ce_fwd_bwd(lg, y, dl, cw, out)
    errs["loss %d" % mode] = abs(float(out[0]) - float(ce)) / abs(float(ce))
    errs["dlogits %d" % mode] = rel(dl, dce)
    assert float(out[1]) == 0.0
  print("soft CE %dx%d: %s" % (h, w, " ".join("%s %.1e" % kv for kv in errs.items())))
  for k, err in errs.items():
    assert err < FTOL, (k, err)


@pytest.mark.gpu
@pytest.mark.parametrize("labels", ["sparse", "soft"])
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_masked_huber(dev, grid, labels):
  """fg_count over a batch of 2 x 128 rows, masked_huber_fwd_bwd on each half divided by that count (what a
  micro-batch of loss_and_grads_chunked does), against the gather of the whole batch; then K = 0."""
  from multiverse_b200 import ops
  h, w = grid
  v = h * w
  g = gen(dev, 520 + h + len(labels))
  n = 2 * NS
  tgt = torch.randn((T_PRED, n, v, 2), generator=g, device=dev) * 200
  pr = tgt + torch.randn((T_PRED, n, v, 2), generator=g, device=dev) * 1.5
  rng = np.random.default_rng(h + len(labels))
  cls = rng.integers(0, v, size=(n, T_PRED))
  cls[:len(edge_cells(h, w)), 0] = edge_cells(h, w)
  if labels == "soft":
    lab = on(dev, soft_maps(cls, h, w, 7)).reshape(n, T_PRED, v).transpose(0, 1).contiguous()
    fg = (lab > 0).reshape(-1)
  else:
    lab = on(dev, cls.T.astype(np.int32))
    fg = torch.nn.functional.one_hot(lab.long(), v).reshape(-1) > 0
  K = torch.zeros(1, dtype=torch.float64, device=dev)
  ops.fg_count(lab, v, K)
  k = int(fg.sum())
  assert float(K) == k
  e = (pr - tgt).abs().reshape(-1, 2)[fg]
  assert float((e < 1).float().mean()) > 0.3 and float((e > 1).float().mean()) > 0.3
  rw = 0.1
  one = torch.ones((), dtype=torch.float64, device=dev)
  hb, (dhb,) = vjp(lambda a: ref_masked_huber(a, tgt.double(), fg, k) * rw, [pr], one)
  out = torch.zeros(2, device=dev)
  dp = torch.full_like(pr, SENTINEL)
  for half in (slice(0, NS), slice(NS, n)):
    p_h, t_h, d_h = pr[:, half].contiguous(), tgt[:, half].contiguous(), torch.full_like(pr[:, half], SENTINEL)
    ops.masked_huber_fwd_bwd(p_h, t_h, d_h, lab[:, half].contiguous(), K, rw, out)
    dp[:, half] = d_h
  errs = {"loss": abs(float(out[1]) - float(hb)) / float(hb), "doffsets": rel(dp, dhb)}
  print("masked Huber %s %dx%d, K = %d: %s" % (labels, h, w, k, errs))
  assert float(out[0]) == 0.0
  assert bool((dp.reshape(-1, 2)[~fg] == 0).all()), "gradient off the foreground"
  for name, err in errs.items():
    assert err < FTOL, (name, err)
  # K = 0: an empty foreground gives a zero loss and gradient (div_no_nan), not NaN
  empty = torch.zeros_like(lab) if labels == "soft" else torch.full_like(lab, -1)
  K0 = torch.zeros(1, dtype=torch.float64, device=dev)
  ops.fg_count(empty, v, K0)
  assert float(K0) == 0.0
  out0 = torch.zeros(2, device=dev)
  d0 = torch.full_like(pr, SENTINEL)
  ops.masked_huber_fwd_bwd(pr, tgt, d0, empty, K0, rw, out0)
  assert float(out0[1]) == 0.0 and bool((d0 == 0).all())


# --------------------------------------------------------------------------- logits feedback
@pytest.mark.gpu
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_head_dense_feedback(dev, grid):
  """head_class_fwd_dense: logits and arg-max as head_class_fwd, and tanh(conv3x3(logits, We) + be) as the next
  step's bf16 x 2 planes; the halo rows and the h block of the planes keep their sentinel."""
  from multiverse_b200 import ops
  h, w = grid
  d = head_inputs(dev, h, w, 540 + h)
  h32 = to_halo(d["h"][0])
  cpad = ops.cell_cpad(E)
  logits = torch.empty((NS, h * w), device=dev)
  ids = torch.empty((NS,), dtype=torch.int32, device=dev)
  xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
  xh.fill_(SENTINEL)
  ops.head_class_fwd_dense(h32, d["Wo1"], logits, ids, d["We1"], d["be"], xh, h, w, NS, planes=2)
  ref = ref_head(d["h"][0].double(), d["Wo1"].double())[..., 0]
  assert torch.equal(ids.long(), logits.argmax(-1))
  emb = ref_emb(logits.double().view(NS, h, w, 1), d["We1"].double(), d["be"].double())
  vals, _ = ops.operand_values(xh)
  errs = {"logits": rel(logits, ref), "logits emb planes": rel(inner(vals, NS, h, w)[..., :E], emb)}
  emb_ref = ref_emb(ref.view(NS, h, w, 1), d["We1"].double(), d["be"].double())
  errs["emb vs fp64 logits"] = rel(inner(vals, NS, h, w)[..., :E], emb_ref)
  print("dense-feedback head %dx%d: %s" % (h, w, errs))
  v = xh.view(2, NS, h + 1, w + 1, cpad)
  assert bool((v[:, :, h] == SENTINEL).all()) and bool((v[:, :, :, w] == SENTINEL).all()), "a halo row was written"
  assert bool((v[:, :, :h, :w, E:] == SENTINEL).all()), "channels beyond the x block were written"
  assert errs["logits"] < FTOL
  assert errs["logits emb planes"] < PTOL and errs["emb vs fp64 logits"] < PTOL


@pytest.mark.gpu
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_emb_backward_dense_one_channel(dev, grid):
  """emb_bwd with P_out = 1 and a dense input (the logits map fed back): 12 launches accumulating into dWe / dbe,
  d_in added to what the loss left in dlogits."""
  from multiverse_b200 import ops
  h, w = grid
  hw = h * w
  g = gen(dev, 560 + h)
  We = torch.randn((3, 3, 1, E), generator=g, device=dev) * 0.5
  be = torch.randn((E,), generator=g, device=dev) * 0.2
  cpad = ops.cell_cpad(E)
  dWe, dbe = torch.zeros_like(We), torch.zeros_like(be)
  dWe_ref, dbe_ref = torch.zeros_like(We, dtype=torch.float64), torch.zeros_like(be, dtype=torch.float64)
  worst = 0.0
  for _ in range(T_PRED):
    dxh = torch.randn((halo_rows(NS, h, w), cpad), generator=g, device=dev)
    dx = inner(dxh, NS, h, w)[..., :E]
    in_map = torch.randn((NS, hw), generator=g, device=dev) * 3
    din = torch.randn((NS, hw), generator=g, device=dev)
    din0 = din.clone()
    ops.emb_bwd(dxh, None, in_map, We, be, dWe, dbe, din, True, h, w, NS)
    _, (gx, gW, gb) = vjp(ref_emb, [in_map.view(NS, h, w, 1), We, be], dx)
    worst = max(worst, rel(din.double() - din0.double(), gx.reshape(NS, hw)))
    dWe_ref += gW
    dbe_ref += gb
  errs = {"dWe": rel(dWe, dWe_ref), "dbe": rel(dbe, dbe_ref), "d_in (worst step)": worst}
  print("emb_bwd dense P_out 1 %dx%d: %s" % (h, w, errs))
  for k, err in errs.items():
    assert err < FTOL, (k, err)


# --------------------------------------------------------------------------- whole model
OPTIONS = {               # soft grid mode (0: sparse labels), mask, one-hot feedback
    "soft4": (4, False, True),
    "soft7_mask": (7, True, True),
    "sparse_mask": (0, True, True),
    "logits_fed": (0, False, False),
    "logits_fed_soft1_mask": (1, True, False),
}


def option_feeds(cfg, n, mode):
  f = shared_frame_feeds(cfg, n, FRAMES, WM_SEED)
  for i, (h, w) in enumerate(cfg.scene_grids):
    cls = f["grid_pred_labels"][i]
    cells = edge_cells(h, w)
    cls[:len(cells), 0] = cells
    cls[1, :len(cells)] = cells[::-1]
    if mode:
      f["grid_pred_labels"][i] = soft_maps(cls, h, w, mode)
  return f


def engine_feeds(dev, f):
  feeds = dict(scene_feat=on(dev, f["scene_feat"]), obs_scene=on(dev, f["obs_scene"]))
  for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    feeds[k] = [on(dev, a) for a in f[k]]
  return feeds


@pytest.mark.gpu
@pytest.mark.parametrize("option", sorted(OPTIONS))
def test_whole_model_with_option(dev, option):
  """loss_and_grads_chunked on 256 trajectories in micro-batches of 128 against the fp64 truth over chunks of 16 (the
  masked Huber of every chunk divided by the K of all 256), every gradient to 2e-4.  With one-hot feedback the
  arg-max margin precondition of test_whole_model_gradient_at_micro_batch applies; the logits-fed decoder has no
  arg-max in training."""
  from multiverse_b200.train_engine import TrainEngine
  from multiverse_b200 import synthetic
  mode, mask, onehot = OPTIONS[option]
  n, mb, chunk = 256, NS, 16
  cfg, rcfg = wm_configs(n, chunk)
  cfg.mask_grid_regression, cfg.train_w_onehot = mask, onehot
  w = synthetic.make_weights(cfg, WM_SEED)
  f = option_feeds(cfg, n, mode)
  K = TO.fg_counts(cfg, f) if mask else None
  grads = {k: np.zeros(v.shape) for k, v in w.items()}
  losses = np.zeros(4)
  logits = [[], []]
  for lo in range(0, n, chunk):
    sl = slice(lo, lo + chunk)
    part = dict(scene_feat=f["scene_feat"], obs_scene=f["obs_scene"][sl])
    for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
      part[k] = [a[sl] for a in f[k]]
    _, l, _, gr, lg = TO.loss_and_grads(rcfg, w, part, soft=bool(mode), mask=mask, onehot=onehot, device=dev,
                                        loss_scale=chunk / n, fg_count=K, return_logits=True)
    losses += np.array(l)
    for k in grads:
      grads[k] += gr[k]
    for i in range(2):
      logits[i].append(lg[i])
  for k in grads:
    if k.endswith("/W"):
      grads[k] -= (n // chunk) * cfg.wd * w[k]
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  got, _ = eng.loss_and_grads_chunked(engine_feeds(dev, f), mb)
  torch.cuda.synchronize()
  for i, (h, ww) in enumerate(cfg.scene_grids):
    ref = np.concatenate(logits[i]).reshape(n, T_PRED, h * ww)
    mine = eng.last_logits[i].cpu().numpy().transpose(1, 0, 2)
    err = rel(mine, ref[n - mb:])
    if onehot:
      srt = np.sort(ref, -1)
      gap = (srt[..., -1] - srt[..., -2]).min() / np.abs(ref).max()
      assert err * 4 < MARGIN and gap > MARGIN, (err, gap)
    print("%s scale %d: logit error of the last micro-batch %.2e" % (option, i, err))
  got = got.cpu().numpy()
  worst = {k: rel(eng.grads[k], grads[k]) for k in sorted(grads)}
  print("%s: losses %s vs %s, worst gradient errors %s" % (option, got, losses,
                                                           sorted(worst.items(), key=lambda kv: -kv[1])[:3]))
  assert np.abs(got - losses).max() < LTOL * np.abs(losses).max(), (got, losses)
  del eng
  torch.cuda.empty_cache()
  bad = {k: v for k, v in worst.items() if v > GTOL}
  assert not bad, bad


@pytest.mark.gpu
def test_chunked_equals_unchunked_soft_mask(dev):
  """Soft labels + mask: the K of the whole batch makes micro-batches of 64 sum to the batch of 128 at once, though
  the two halves have different foreground counts."""
  from multiverse_b200.train_engine import TrainEngine
  from multiverse_b200 import synthetic
  n, mb = NS, NS // 2             # the activation store of a whole batch of 256 at once does not fit beside the others
  cfg, _ = wm_configs(n, 16)
  cfg.mask_grid_regression = True
  w = synthetic.make_weights(cfg, WM_SEED)
  f = option_feeds(cfg, n, 7)
  halves = [TO.fg_counts(cfg, {"grid_pred_labels": [a[s] for a in f["grid_pred_labels"]]})
            for s in (slice(0, mb), slice(mb, n))]
  assert halves[0] != halves[1], halves
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = engine_feeds(dev, f)
  l_full, _ = eng.loss_and_grads(feeds)
  g_full = eng.flat_grad.clone()
  l_mb, _ = eng.loss_and_grads_chunked(feeds, mb)
  err_l = float((l_full - l_mb).abs().max()) / float(l_full.abs().max())
  err_g = float((g_full - eng.flat_grad).abs().max()) / float(g_full.abs().max())
  print("chunked vs unchunked, soft 7 + mask, %d trajectories in micro-batches of %d: losses %.1e, gradients %.1e"
        % (n, mb, err_l, err_g))
  assert err_l < 1e-5 and err_g < 2e-5


# --------------------------------------------------------------------------- drop-in
def _dropin_model(monkeypatch, w=None, f=None, n=4, over=None, **flags):
  """The drop-in Model of code/train.py's arguments (+ flags; `over`: model-shape and loss-weight arguments) on
  weights w and feeds f (synthetic ones by default), and a batch of f as the reference's pred_utils hands it to
  Trainer.step."""
  from multiverse_b200 import synthetic
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "pred_models", "multiverse_b200.pred_models"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  import pred_models
  tf.reset_default_graph()
  conf = dict(batch_size=n, use_grids=[False, True], grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001)
  conf.update(over or {})
  cfg = synthetic.make_config(is_train=True, clip_gradient_norm=10.0, **conf)
  args = types.SimpleNamespace(**vars(cfg))            # code/train.py's defaults for the multi-future flags
  args.modelname = "m"; args.use_gt_grid = False; args.use_teacher_forcing = False; args.train_w_onehot = False
  args.use_soft_grid_class = False; args.soft_grid = 1; args.mask_grid_regression = False
  args.optimizer = "adadelta"; args.init_lr = 0.2; args.emb_lr = 1.0; args.learning_rate_decay = 0.95
  args.num_epoch_per_decay = 2.0; args.train_num_examples = 100; args.use_cosine_lr = False
  for k, v in flags.items():
    setattr(args, k, v)
  w = synthetic.make_weights(cfg, 5) if w is None else w
  f = synthetic.make_feeds(cfg, n, 5, with_pred=True) if f is None else f
  model = pred_models.get_model(args, gpuid=0)
  tf.global_variables_initializer().run()
  for v in tf.global_variables():
    if v.name.split(":")[0] in w:
      v.assign(w[v.name.split(":")[0]])
  data = dict(obs_grid_class=[np.stack([f["grid_obs_labels"][j][i] for j in range(2)]) for i in range(n)],
              pred_grid_class=[np.stack([f["grid_pred_labels"][j][i] for j in range(2)]) for i in range(n)],
              batch_scene_feat=f["scene_feat"], batch_obs_scene=f["obs_scene"][:, :, None])
  for j in range(2):
    data["obs_grid_target_all_%d" % j] = list(f["grid_obs_regress"][j])
    data["pred_grid_target_all_%d" % j] = list(f["grid_pred_regress"][j])
  return tf, pred_models, model, args, cfg, w, f, (tuple(range(n)), types.SimpleNamespace(data=data))


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [{}, dict(use_soft_grid_class=True, soft_grid=7), dict(mask_grid_regression=True),
                                   dict(train_w_onehot=True, use_soft_grid_class=True, soft_grid=4,
                                        mask_grid_regression=True)],
                         ids=["train_py_defaults", "soft7", "mask", "onehot_soft4_mask"])
def test_dropin_trainer_step(dev, monkeypatch, flags):
  """Trainer.step through the shim Session with code/train.py's flags: losses against the fp64 truth."""
  from oracle import multiverse_ref as R
  tf, pred_models, model, args, cfg, w, f, batch = _dropin_model(monkeypatch, **flags)
  rcfg = R.default_config(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, batch_size=4,
                          use_grids=[False, True])
  rf = dict(f)
  if args.use_soft_grid_class:
    rf["grid_pred_labels"] = [soft_maps(a, h, ww, args.soft_grid) for a, (h, ww) in zip(f["grid_pred_labels"],
                                                                                          cfg.scene_grids)]
  tot, losses, wd, _ = TO.loss_and_grads(rcfg, w, rf, soft=args.use_soft_grid_class, mask=args.mask_grid_regression,
                                         onehot=args.train_w_onehot)
  with tf.Session() as sess:
    trainer = pred_models.Trainer(model, args)
    loss, _, wd_loss, pgl = trainer.step(sess, batch)
    assert abs(loss - tot) < 1e-4 * abs(tot) and abs(wd_loss - wd) < 1e-5 * wd
    assert np.abs(np.array(pgl) - np.array(losses)).max() < 1e-4 * max(losses)
    assert int(sess.run(model.global_step)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(use_teacher_forcing=True), dict(keep_prob=0.7), dict(use_single_decoder=True),
                                   dict(adv_train=True), dict(multiview_train=True),
                                   dict(train_w_onehot=True, use_soft_grid_class=True, adv_train=False,
                                        multiview_train=False)],
                         ids=["teacher_forcing", "dropout", "single_decoder", "adv_train", "multiview_train",
                              "soft_with_simaug_model"])
def test_dropin_still_refuses(dev, monkeypatch, flags):
  """Teacher forcing, dropout and the single decoder stay unimplemented, and so do the new options with SimAug's
  augmentations (and soft labels with SimAug's model, which ignores them): the training step refuses loudly before
  it reads the feeds (SimAug's feeds need more than this batch carries), never a silent run."""
  _, _, model, _, _, _, _, _ = _dropin_model(monkeypatch, **flags)
  with pytest.raises(NotImplementedError):
    model._train_step({})


# --------------------------------------------------------------------------- drop-in against the reference's execution
@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(G.CASES))
def test_dropin_trainer_step_equals_reference_execution(dev, monkeypatch, case):
  """One Trainer.step through the drop-in (get_feed_dict builds the soft maps from the batch's cell labels, the engine
  trains, the shim Session returns the fetches) on the inputs of tests/golden/refexec_train_<case>.npz - what the
  unmodified reference Model + Trainer computed on them: the losses (1e-4), the clipped gradient of every variable
  (2e-4 of its largest element, as the whole-model tests) and the variables after the Adadelta step.  The update
  g sqrt(eps) / sqrt(0.05 g^2 + eps) has slope <= 1 in g, so a variable may differ from the reference's by at most
  lr x the gradient bar plus fp32 rounding of the weight."""
  from oracle import multiverse_ref as R
  mode, mask, onehot = G.CASES[case]
  cfg = R.default_config(**G.OVER)
  w, f = R.make_weights(cfg, G.SEED), G.edge_labels(cfg, R.make_inputs(cfg, G.SEED))   # cell labels, as a batch has
  got = np.load(os.path.join(ROOT, "tests", "golden", "refexec_train_%s.npz" % case))
  tf, pred_models, model, args, _, _, _, batch = _dropin_model(
      monkeypatch, w=w, f=f, n=cfg.batch_size, use_soft_grid_class=bool(mode), soft_grid=mode or 1,
      mask_grid_regression=mask, train_w_onehot=onehot)
  check_step_against_reference_execution(case, tf, pred_models, model, args, batch, w, got, "")


def check_step_against_reference_execution(tag, tf, pred_models, model, args, batch, w, got, prefix):
  """One Trainer.step of the drop-in model against a reference-execution golden (keys under `prefix`): the losses,
  the clipped gradients and the variables after the Adadelta step, at the learning rate of the arguments."""
  with tf.Session() as sess:
    loss, _, wd_loss, pgl = pred_models.Trainer(model, args).step(sess, batch)
    assert int(sess.run(model.global_step)) == 1
  got = {k[len(prefix):]: got[k] for k in got.files if k.startswith(prefix)}
  assert abs(loss - float(got["loss"])) <= LTOL * abs(float(got["loss"]))
  assert abs(wd_loss - float(got["wd_loss"])) <= 1e-5 * float(got["wd_loss"])
  assert len(pgl) == len(got["pred_grid_loss"])
  assert np.abs(np.array(pgl) - got["pred_grid_loss"]).max() <= LTOL * got["pred_grid_loss"].max()
  eng = model._engine
  lr, worst = args.init_lr * args.emb_lr, {}        # the Adadelta rate at step 0
  for k in got["variables"]:
    g = eng.grads[k].double().cpu().numpy() + (args.wd * w[k] if k.endswith("/W") else 0.0)   # + weight decay
    gc = np.clip(g, -10.0, 10.0)
    bar_g = GTOL * float(got["grad_absmax/" + k])
    err_g = np.abs(G.sample(gc) - got["grad/" + k]).max()
    err_w = np.abs(G.sample(eng.params[k].double().cpu().numpy()) - got["updated/" + k]).max()
    bar_w = lr * bar_g + 2.4e-7 * max(np.abs(w[k]).max(), 1e-30)
    worst[k] = (err_g / float(got["grad_absmax/" + k]), err_w)
    assert err_g <= bar_g, (k, err_g, bar_g)
    assert err_w <= bar_w, (k, err_w, bar_w)
  print("%s: loss %.6g vs %.6g (rel %.2e), worst gradient errors %s" % (
      tag, loss, float(got["loss"]), abs(loss - float(got["loss"])) / abs(float(got["loss"])),
      sorted(worst.items(), key=lambda kv: -kv[1][0])[:3]))


@pytest.mark.gpu
def test_dropin_trainer_step_on_the_published_command_equals_reference_execution(dev, monkeypatch):
  """One Trainer.step with TRAINING.md's arguments - scene 36x64, strides 2,4 (grids 18x32 and 9x16), use_grids 1,1,
  --train_w_onehot, loss weights 1.0 / 0.2, --init_lr 0.3 - on the inputs of tests/golden/refexec_native.npz,
  against what the unmodified reference Model + Trainer computed on them, with the checks of
  test_dropin_trainer_step_equals_reference_execution."""
  cfg, w, f = cases.refexec_native_inputs()
  opts = cases.REFEXEC_NATIVE[2]
  assert G.SAMPLE == cases.NATIVE_TRAIN_SAMPLE
  got = np.load(os.path.join(ROOT, "tests", "golden", "refexec_native.npz"))
  over = dict(scene_h=cfg.scene_h, scene_w=cfg.scene_w, scene_grid_strides=[2, 4], use_grids=[True, True],
              grid_loss_weight=opts["grid_loss_weight"], grid_reg_loss_weight=opts["grid_reg_loss_weight"],
              wd=opts["wd"])
  tf, pred_models, model, args, dcfg, _, _, batch = _dropin_model(
      monkeypatch, w=w, f=f, n=cfg.batch_size, over=over, train_w_onehot=opts["train_w_onehot"],
      init_lr=opts["init_lr"])
  assert dcfg.scene_grids == [(18, 32), (9, 16)] and args.init_lr == 0.3 and args.grid_reg_loss_weight == 0.2
  check_step_against_reference_execution("published command 36x64", tf, pred_models, model, args, batch, w, got,
                                         "train/")
