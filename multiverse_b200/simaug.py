# coding=utf-8
"""SimAug's white-box attack on the scene input, on the H100 engine (SURVEY.md section 8 row f-4, first part).

Mirrors ``white_box_attack`` of ``SimAug/code/pred_models.py:60-170`` - same argument meaning, same config
attributes (``adv_epsilon, adv_step_size, adv_num_iter, adv_start_from_clean_prob, adv_use_fgsm, use_mixup,
mixup_alpha, mixup_mix_adv, use_grids, scene_grids``) - with the reference's ``model_func`` + ``tf.gradients(
classification_loss, adv_input)`` replaced by ``TrainEngine.loss_and_grads(dscene_out=...)``: the ordinary BPTT of
this library with the scene CNN's input gradient switched on (``mvb_scene_conv_bwd`` ``din`` of the first
convolution).  The update itself is ``mvb_adv_step`` / ``mvb_mix``.  SimAug's model differs from Multiverse's in one place that matters here: its ``gnn_edge`` (:1213-1226) uses the scene
features only in the beam decoder, so the training tower's graph attention runs over h alone - build the TrainEngine
with ``cfg.gnn_scene_in_greedy = False`` (the drop-in Model does it for configs that carry SimAug's flags).  Pinned
on an execution of the reference file (tests/golden/simaug_multiview.npz and its generating script).
Random draws (start noise, random target
offsets, the Beta mixup weight) come from a numpy Generator - TensorFlow's random streams cannot be reproduced.

``multiview_augmentation`` (:346-541; second part of row f-4) runs the same one-step attack on the batch tiled
over the M camera views - the role of the reference's ``build_tower`` (:544, the forward of the model on given scene
semantics and tiled feeds) is played by ``TrainEngine.loss_and_grads`` on the tiled feed dict - ranks the views by
their per-sample classification loss (``mvb_ce_rows``), picks two per ``config.multiview_exp`` and mixes them.  The
label side of experiment 3 (mixed observed class maps and loss labels, focal weights; :616-638, :1371-1405) lives in
``TrainEngine`` (``feeds["mixup"]``) and is wired up by the drop-in ``Model._simaug_feeds``.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def create_random_target(label, max_class, rng):
  """:66-72: label + uniform{1..max_class-1} modulo max_class - always a WRONG class."""
  off = rng.integers(1, max_class, size=label.shape)
  return ((label.astype(np.int64) + off) % max_class).astype(np.int32)


def scene_input_grad(engine, feeds, target_label, scale_idx):
  """d sum(sparse CE(target)) / d scene_feat up to a positive factor (the attack only uses its sign):
  SimAug/code/pred_models.py:96-115.  feeds: a TrainEngine feed dict whose scene_feat [F,SH,SW,SC] the gradient
  is taken for; target_label int32 [N,Tp] replaces grid_pred_labels of the attacked scale."""
  f = dict(feeds)
  f["grid_pred_labels"] = list(feeds["grid_pred_labels"])
  f["grid_pred_labels"][scale_idx] = target_label
  g = torch.zeros_like(feeds["scene_feat"], dtype=torch.float32)
  engine.loss_and_grads(f, dscene_out=g, cls_weight=1.0, reg_weight=0.0)
  return g


def white_box_attack(engine, feeds, label, config, rng=None, norm_feat=False):
  """SimAug/code/pred_models.py:60-170.  `feeds["scene_feat"]` is the clean input feature (one frame per (n,t)
  row like the reference's [N*T_obs,SH,SW,SC], or unique frames + obs_scene indices: the gradient then sums over
  the rows that share a frame).  label: numpy int [N,T_pred] of the attacked scale.  Returns (adv_final fp32 tensor
  shaped like scene_feat, target_label numpy int32 [N,T_pred])."""
  rng = rng or np.random.default_rng()
  assert not norm_feat, "norm_feat (softmax of the start point) is not implemented"
  scale_idx = list(config.use_grids).index(True)                      # :128
  h, w = config.scene_grids[scale_idx]
  dev = engine.device
  x = feeds["scene_feat"].float().contiguous()
  target_label = create_random_target(np.asarray(label), int(h * w), rng)      # :132-133
  tl = torch.from_numpy(target_label).to(dev)
  eps = float(config.adv_epsilon)

  def get_start_adv():                                                # :75-89
    if config.adv_start_from_clean_prob >= 1.0:
      return x.clone()
    noise = torch.from_numpy(rng.uniform(-eps, eps, size=tuple(x.shape)).astype(np.float32)).to(dev)
    if config.adv_start_from_clean_prob > 0:
      noise = noise * float(rng.uniform() > config.adv_start_from_clean_prob)
    return x + noise

  def one_step_attack(adv):                                           # :91-124
    g = scene_input_grad(engine, dict(feeds, scene_feat=adv), tl, scale_idx)
    out = torch.empty_like(adv)
    ops.adv_step(x, adv, g, out, eps, eps if config.adv_use_fgsm else float(config.adv_step_size))
    return out

  adv = one_step_attack(get_start_adv())
  if not config.adv_use_fgsm:                                          # PGD: adv_num_iter steps in all (:145-155)
    for _ in range(int(config.adv_num_iter) - 1):
      adv = one_step_attack(adv)
  if getattr(config, "use_mixup", False):                             # :157-170
    weight = float(rng.beta(config.mixup_alpha, config.mixup_alpha))
    out = torch.empty_like(adv)
    if getattr(config, "mixup_mix_adv", False):
      assert config.adv_use_fgsm and config.adv_start_from_clean_prob < 1.0
      adv2 = one_step_attack(get_start_adv())
      ops.mix(adv2, adv, out, weight)
    else:
      ops.mix(x, adv, out, weight)
    adv = out
  return adv, target_label


def _tile_views(t, m):
  """[N, ...] -> [N*M, ...]: every sample repeated M times in a row (tf.tile on a new axis 1 + reshape, :404-431)."""
  return t.unsqueeze(1).expand((t.shape[0], m) + tuple(t.shape[1:])).reshape((t.shape[0] * m,) + tuple(t.shape[1:])).contiguous()


def multiview_augmentation(engine, feeds, config, rng=None):
  """SimAug/code/pred_models.py:346-541.  feeds: a TrainEngine feed dict of N samples (scene_feat [F,SH,SW,SC] +
  obs_scene [N,T]: the reference's per-row features are scene_feat[obs_scene]) with two more entries:
    grid_pred_labels_extra[i] int [N,M,Tp]  labels of the M other views (self.grid_pred_labels_T_extra): the attack
                                            targets of the M tiled copies of every sample;
    obs_scene_extra int [N,M,T]             frame indices of the other views (multiview_exp == 3 only).
  config: adv_epsilon, adv_start_from_clean_prob, multiview_max_num, multiview_exp (1 top-2 loss, 4 bottom-2,
  2 two random views, 3 top adversarial + another view's clean features), multiview_use_adv_for_loss,
  multiview_random, fl_gamma, mixup_alpha, multiview_max_weight_for_first, use_grids, scene_grids.
  Returns (adv_final fp32 [N*T,SH,SW,SC] - the scene semantics the training tower is then fed with, one frame per
  (sample, step) row -, info) with info = dict(beta_weight, adv_loss [N,M] tensor, loss_indices [N,M],
  selected_extra_indices / focal_loss_weight for exp 3)."""
  rng = rng or np.random.default_rng()
  dev = engine.device
  m = int(config.multiview_max_num)
  scale_idx = list(config.use_grids).index(True)                      # :348
  eps = float(config.adv_epsilon)
  obs_scene = feeds["obs_scene"].long()
  n, t_obs = obs_scene.shape
  clean = feeds["scene_feat"].float()[obs_scene]                      # [N,T,SH,SW,SC]  (embedding_lookup)
  feat_shape = tuple(clean.shape[2:])
  tiled = _tile_views(clean, m).reshape((n * m * t_obs,) + feat_shape)        # [N*M*T, SH,SW,SC]  (:399-407)
  # the tiled feed dict (:409-431): one private frame per (sample, view, step) row
  tf = dict(obs_scene=torch.arange(n * m * t_obs, device=dev, dtype=torch.int32).reshape(n * m, t_obs))
  for key in ("grid_obs_labels", "grid_obs_regress", "grid_pred_regress"):
    tf[key] = [None if a is None else _tile_views(a, m) for a in feeds[key]]
  extra = torch.as_tensor(np.asarray(feeds["grid_pred_labels_extra"][scale_idx]), device=dev).to(torch.int32)
  target = extra.reshape(n * m, -1).contiguous()                      # [N*M,Tp]  (:433-435)
  tf["grid_pred_labels"] = [None if a is None else _tile_views(a.to(torch.int32), m) for a in feeds["grid_pred_labels"]]
  tf["grid_pred_labels"][scale_idx] = target

  def get_start_adv(x):                                               # :350-365
    if config.adv_start_from_clean_prob >= 1.0:
      return x
    noise = torch.from_numpy(rng.uniform(-eps, eps, size=tuple(x.shape)).astype(np.float32)).to(dev)
    if config.adv_start_from_clean_prob > 0:
      noise = noise * float(rng.uniform() > config.adv_start_from_clean_prob)
    return x + noise

  def one_step_attack(x):                                             # :367-397
    start = get_start_adv(x).contiguous()
    g = torch.zeros_like(start)
    engine.loss_and_grads(dict(tf, scene_feat=start), dscene_out=g, cls_weight=1.0, reg_weight=0.0)
    logits = engine.last_logits[scale_idx]                            # [Tp, N*M, HW]
    per_row = ops.ce_rows(logits, target.t().contiguous())            # [Tp, N*M]
    loss = per_row.mean(0)                                            # reduce_mean over the predicted steps (:396)
    adv = torch.empty_like(start)
    ops.adv_step(start, start, g, adv, eps, eps)                      # FGSM around the start point (:384-392)
    return adv, loss

  adv_out, adv_loss = one_step_attack(tiled)
  info = {}
  rows = torch.arange(n, device=dev)
  view6 = lambda a: a.reshape((n, m, t_obs) + feat_shape)
  pick = lambda a, idx: view6(a)[rows, idx.long()].reshape((n * t_obs,) + feat_shape).contiguous()   # gather_at_second_dim
  exp = int(config.multiview_exp)
  if exp == 3 and getattr(config, "multiview_use_adv_for_loss", False):      # :463-470
    _, adv_loss = one_step_attack(adv_out)
  adv_loss = adv_loss.reshape(n, m)
  # tf.nn.top_k(sorted=True): descending, the lower index first among equals
  loss_val, loss_idx = torch.sort(adv_loss, dim=1, descending=True, stable=True)
  if exp == 1:                                                        # :439-444
    feat1, feat2 = pick(adv_out, loss_idx[:, 0]), pick(adv_out, loss_idx[:, 1])
  elif exp == 4:                                                      # :445-450
    feat1, feat2 = pick(adv_out, loss_idx[:, m - 1]), pick(adv_out, loss_idx[:, m - 2])
  elif exp == 2:                                                      # :451-462  two different views, uniformly
    r1 = torch.from_numpy(rng.integers(0, m, size=n)).to(dev)
    r2 = (r1 + torch.from_numpy(rng.integers(1, m, size=n)).to(dev)) % m
    feat1, feat2 = pick(adv_out, r1), pick(adv_out, r2)
    info["random_views"] = (r1, r2)
  elif exp == 3:                                                      # :463-496
    info["focal_loss_weight"] = (1.0 - torch.exp(-loss_val[:, 0])) ** float(config.fl_gamma)
    feat1 = pick(adv_out, loss_idx[:, 0])
    sel = loss_idx[:, 0]
    if getattr(config, "multiview_random", False):
      sel = torch.from_numpy(rng.integers(0, m, size=n)).to(dev)
    other = torch.as_tensor(np.asarray(feeds["obs_scene_extra"]), device=dev).long()        # [N,M,T]
    feat2 = feeds["scene_feat"].float()[other[rows, sel.long()]].reshape((n * t_obs,) + feat_shape).contiguous()
    info["selected_extra_indices"] = sel
  else:
    raise ValueError("Please set experiment number (multiview_exp in 1..4)")          # :497-499
  weight = float(rng.beta(config.mixup_alpha, config.mixup_alpha))    # :503-508
  if getattr(config, "multiview_max_weight_for_first", False):
    weight = max(weight, 1.0 - weight)
  out = torch.empty_like(feat1)
  ops.mix(feat1, feat2, out, weight)                                  # :511
  info.update(beta_weight=weight, adv_loss=adv_loss, loss_indices=loss_idx)
  return out, info
