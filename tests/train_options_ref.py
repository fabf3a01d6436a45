# coding=utf-8
"""fp64 torch truth for the training options of code/train.py:85-92 that change Model.build_loss and the
training-mode class decoder, built on the oracle's torch restatement (oracle/multiverse_ref_torch.py):

  soft     --use_soft_grid_class: grid_pred_labels[i] are [N,Tp,h,w,1] label maps and the classification loss is
           softmax_cross_entropy_with_logits against them (code/pred_models.py:986-989);
  mask     --mask_grid_regression: Huber over the cells whose label is > 0 only, gathered as tf.where + tf.gather do
           and averaged over the 2K gathered elements (:999-1018), 0 when K = 0 (div_no_nan);
  onehot   False without --train_w_onehot: the class decoder feeds back its logits map (:285, :426-435).

Test infrastructure; tests/test_train_options_cpu.py pins it to executions of the unmodified reference."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import multiverse_ref as R
from oracle import multiverse_ref_torch as RT


def forward(cfg, w, feeds, dtype, device=None, onehot=True):
  """Greedy training-mode forward (RT._forward without beam search and mixup), the class decoder fed
  one_hot(argmax) (onehot) or its logits."""
  n = cfg.batch_size
  scene_feat = torch.from_numpy(np.asarray(feeds["scene_feat"])).to(device=device, dtype=dtype)
  obs_scene = torch.from_numpy(np.asarray(feeds["obs_scene"])).to(scene_feat.device).long()
  x = scene_feat[obs_scene.reshape(-1)]
  convs = []
  for i in range(len(cfg.scene_grid_strides)):
    x = torch.tanh(RT.conv2d_same(x, w["person_pred/scene_conv%d/W" % (i + 1)], 2)
                   + w["person_pred/scene_conv%d/b" % (i + 1)])
    convs.append(x.reshape((n, -1) + tuple(x.shape[1:])))
  cls, reg = [], []
  for i, (h, ww) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      cls.append(None); reg.append(None)
      continue
    sw = R.scale_weights(w, i)
    labels = torch.from_numpy(np.asarray(feeds["grid_obs_labels"][i])).to(device).long()
    obs_cls = F.one_hot(labels, h * ww).to(dtype).reshape(n, -1, h, ww, 1)
    obs_reg = torch.from_numpy(np.asarray(feeds["grid_obs_regress"][i])).to(device=device, dtype=dtype)
    mask = RT.neighbour_mask(h, ww, dtype, device)
    enc = RT.encoder(convs[i] * obs_cls, sw.enc_class[0], sw.enc_class[1], cfg.enc_hidden_size, device)
    enc_r = RT.encoder(obs_reg, sw.enc_reg[0], sw.enc_reg[1], cfg.enc_hidden_size, device)
    sm = convs[i].mean(1) if getattr(cfg, "gnn_scene_in_greedy", True) else None
    cls.append(RT.decoder_greedy(obs_cls[:, -1], enc, cfg.pred_len, sw.dec_class, sw.emb_class, sw.head_class, sm,
                                 mask, cfg.use_gnn, onehot))
    reg.append(RT.decoder_greedy(obs_reg[:, -1], enc_r, cfg.pred_len, sw.dec_reg, sw.emb_reg, sw.head_reg, None,
                                 None, False, False))
  return cls, reg


def foreground(labels, hw):
  """Flat foreground mask [N*Tp*HW] of the masked regression loss: label > 0 of the maps, or one_hot of the cells."""
  if labels.dim() > 2:
    return labels.reshape(-1) > 0
  return F.one_hot(labels.long().reshape(-1), hw).reshape(-1) > 0


def fg_counts(cfg, feeds):
  """K per scale (0 for an unused one), as TrainEngine.fg_counts."""
  out = []
  for i, (h, ww) in enumerate(cfg.scene_grids):
    out.append(int(foreground(torch.from_numpy(np.asarray(feeds["grid_pred_labels"][i])), h * ww).sum())
               if cfg.use_grids[i] else 0)
  return out


def loss_and_grads(cfg, weights, feeds, soft=False, mask=False, onehot=True, dtype=torch.float64, device="cpu",
                   loss_scale=1.0, fg_count=None, return_logits=False):
  """(total, [cls_0, reg_0, ...], wd, {name: grad} as numpy[, logits per scale]) of Model.build_loss under the
  options, by autograd.  loss_scale weights the losses of this batch inside a larger one, except the masked Huber
  when fg_count (K of the larger batch, per scale) is given: that one is already divided by the whole batch's K."""
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=dtype).requires_grad_(True)
       for k, v in weights.items()}
  cls_out, reg_out = forward(cfg, w, feeds, dtype, device, onehot)
  losses = []
  for i, (h, ww) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      continue
    hw = h * ww
    logits = cls_out[i].reshape(-1, hw)
    lab = torch.from_numpy(np.asarray(feeds["grid_pred_labels"][i])).to(device)
    if soft:
      y = lab.to(dtype).reshape(-1, hw)
      cls = (-(y * F.log_softmax(logits, dim=1)).sum(1)).mean()
    else:
      cls = F.cross_entropy(logits, lab.long().reshape(-1))
    pred = reg_out[i].reshape(-1, 2)
    tgt = torch.from_numpy(np.asarray(feeds["grid_pred_regress"][i])).to(device=device, dtype=dtype).reshape(-1, 2)
    reg_scale = loss_scale
    if mask:
      fg = torch.nonzero(foreground(lab, hw))[:, 0]          # tf.where(labels > 0)[:, 0]
      a = (pred[fg] - tgt[fg]).abs()                           # tf.gather of both
      terms = torch.where(a <= 1.0, 0.5 * a * a, a - 0.5)
      k = fg.numel() if fg_count is None else fg_count[i]
      if fg_count is not None:
        reg_scale = 1.0
      reg = terms.sum() / (2 * k) if k > 0 else terms.sum() * 0.0
    else:
      reg = F.huber_loss(pred, tgt, delta=1.0)
    losses += [cls * cfg.grid_loss_weight * loss_scale, reg * cfg.grid_reg_loss_weight * reg_scale]
  wd = sum(cfg.wd * 0.5 * (v * v).sum() for k, v in w.items() if k.endswith("/W"))
  total = sum(losses) + wd
  total.backward()
  grads = {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in w.items()}
  res = (float(total.detach()), [float(l.detach()) for l in losses], float(wd.detach()), grads)
  if return_logits:
    res += ([None if c is None else c.detach().cpu().numpy() for c in cls_out],)
  return res
