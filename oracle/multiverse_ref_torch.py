# coding=utf-8
"""torch-CPU fp32 restatement of the reference forward pass, used ONLY as the timed CPU baseline
(bench.py ``cpu_baseline`` / ``--impl reference``) and as an independent cross-check of
``oracle/multiverse_ref.py`` in tests.  TEST INFRASTRUCTURE - never imported by multiverse_b200.

Pinned like multiverse_ref.py (to which tests/test_oracle_cpu.py ties it): on the execution of the
unmodified reference graph code over the eager TF-1.15 stand-in of oracle/tf1_eager.  TensorFlow 1.15
itself cannot run here, so "the reference's own CPU path" as a timed baseline is this restatement of
code/pred_models.py with the same op decomposition TF uses
(conv2d -> oneDNN convolution, dense [HW,HW] graph attention via batched matmul, full sort for
the diverse-beam rank), running on all host threads.  ``loss_and_grads`` also runs on a CUDA device (fp64, the
convolutions as im2col matmuls): the truth of the at-size whole-model gradient test.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import multiverse_ref as R


def conv2d_same(x, w, stride=1):
  """tf.nn.conv2d(..., "SAME") on NHWC tensors / HWIO filters (code/pred_models.py:1363).  CUDA tensors go through
  an im2col matmul: fp64 convolutions have no fast cuDNN algorithm, fp64 GEMMs run on the tensor cores."""
  n, h, wd, c = x.shape
  kh, kw = w.shape[0], w.shape[1]
  oh, pt, pb = R.same_pad(h, kh, stride)
  ow, pl, pr = R.same_pad(wd, kw, stride)
  if x.is_cuda:
    p = F.pad(x, (0, 0, pl, pr, pt, pb))
    cols = torch.cat([p[:, dy:dy + stride * (oh - 1) + 1:stride, dx:dx + stride * (ow - 1) + 1:stride]
                      for dy in range(kh) for dx in range(kw)], -1)
    return (cols.reshape(-1, kh * kw * c) @ w.reshape(kh * kw * c, -1)).reshape(n, oh, ow, -1)
  xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
  y = F.conv2d(xn.contiguous(), w.permute(3, 2, 0, 1).contiguous(), stride=stride)
  return y.permute(0, 2, 3, 1)


def convlstm_cell(x, c, h, kernel, biases, forget_bias=1.0):
  """ConvLSTMCell.call (TF 1.15), code/pred_models.py:189-202,:236-249."""
  g = conv2d_same(torch.cat([x, h], dim=-1), kernel) + biases
  gi, gj, gf, go = torch.split(g, g.shape[-1] // 4, dim=-1)
  new_c = torch.sigmoid(gf + forget_bias) * c + torch.sigmoid(gi) * torch.tanh(gj)
  return new_c, torch.tanh(new_c) * torch.sigmoid(go)


def neighbour_mask(h, w, dtype=torch.float32, device=None):
  eye = torch.eye(h * w, dtype=dtype, device=device).reshape(h * w, h, w, 1)
  return conv2d_same(eye, torch.ones(3, 3, 1, 1, dtype=dtype, device=device)).reshape(h * w, h * w)


def gnn_dense(hs, scene_mean, mask):
  """gnn_edge + gnn_mask_edge(exp_mask) + gnn_node + residual, code/pred_models.py:808-909,:378."""
  n, h, w, d = hs.shape
  feats = hs.reshape(n, h * w, d)
  if scene_mean is not None:
    feats = torch.cat([feats, scene_mean.reshape(n, h * w, -1)], dim=-1)
  fn = feats * torch.rsqrt(torch.clamp((feats * feats).sum(-1, keepdim=True), min=1e-12))
  edge = torch.bmm(fn, fn.transpose(1, 2)) + (1.0 - mask)[None] * -1e30
  a = torch.softmax(edge, dim=-1)
  return hs + torch.bmm(a, hs.reshape(n, h * w, d)).reshape(n, h, w, d)


def grid_emb(x, W, b):
  return torch.tanh(conv2d_same(x, W) + b)


def encoder(inputs, kernel, biases, ch, device=None):
  n, t, h, w, _ = inputs.shape
  c = torch.zeros(n, h, w, ch, dtype=inputs.dtype, device=device)
  hs = torch.zeros(n, h, w, ch, dtype=inputs.dtype, device=device)
  for s in range(t):
    c, hs = convlstm_cell(inputs[:, s], c, hs, kernel, biases)
  return c, hs


def one_hot_map(ids, h, w, dtype=torch.float32, device=None):
  ids = ids if device is None else ids.to(device)
  return F.one_hot(ids.long(), h * w).to(dtype).reshape(-1, h, w, 1)


def decoder_greedy(first, state, tp, cell_w, emb_w, head_w, scene_mean, mask, use_gnn, onehot):
  """Model.grid_decoder at inference, code/pred_models.py:311-471."""
  c, h = state
  n, hh, ww, p = first.shape
  inp, outs = first, []
  for _ in range(tp):
    h_in = gnn_dense(h, scene_mean, mask) if use_gnn else h
    c, h = convlstm_cell(grid_emb(inp, *emb_w), c, h_in, *cell_w)
    o = conv2d_same(h, head_w)
    outs.append(o)
    inp = one_hot_map(o.reshape(n, -1).argmax(1), hh, ww, o.dtype) if onehot else o
  return torch.stack(outs, 1)


def decoder_beam(first, state, tp, b, cell_w, emb_w, head_w, scene_mean, mask, diverse, gamma,
                 fix_num_timestep, margins=None):
  """Model.grid_decoder_beam_search, code/pred_models.py:474-806 (diverse rank through a full
  sort, as add_div_penalty :1197-1223 does)."""
  c0, h0 = state
  n, hh, ww, _ = h0.shape
  v = hh * ww
  rep = lambda t: t.repeat_interleave(b, dim=0)
  c, h, inp, sm = rep(c0), rep(h0), rep(first), rep(scene_mean)
  score = torch.zeros(n, b, dtype=h0.dtype)
  ids_l, par_l, log_l = [], [], []

  def step(inp, c, h):
    return convlstm_cell(grid_emb(inp, *emb_w), c, gnn_dense(h, sm, mask), *cell_w)

  c, h = step(inp, c, h)
  for time in range(1, tp + 1):
    logits = conv2d_same(h, head_w).reshape(n, b, v)
    lp = torch.log_softmax(logits, -1) + score[:, :, None]
    if diverse:
      order = torch.argsort(lp, dim=-1, descending=True, stable=True)
      rank = torch.empty_like(order)
      rank.scatter_(-1, order, torch.arange(v).expand_as(order))
      lp = lp + math.log(gamma) * rank.to(lp.dtype)
    cand = lp.reshape(n, b * v) if time > 1 else lp[:, 0]
    sc, idx = torch.topk(cand, b, dim=-1, sorted=True)
    if margins is not None:      # [smallest gap between consecutive selected candidates, gap to the best unselected one]
      top = torch.topk(cand, b + 1, dim=-1, sorted=True).values
      margins.append(torch.stack([(top[:, :-2] - top[:, 1:-1]).min(-1).values, top[:, -2] - top[:, -1]], -1))
    if time <= fix_num_timestep:
      sc = torch.zeros_like(sc)
    ids, par = idx % v, idx // v
    ids_l.append(ids); par_l.append(par); log_l.append(logits)
    score = sc
    flat = (par + (torch.arange(n) * b)[:, None]).reshape(-1)
    c, h = c[flat], h[flat]
    inp = one_hot_map(ids.reshape(-1), hh, ww, h0.dtype)
    if time == tp:
      break
    c, h = step(inp, c, h)
  parents = torch.arange(b)[None].repeat(n, 1)
  rows = torch.arange(n)[:, None]
  out_ids = torch.zeros(n, b, tp, dtype=torch.long)
  out_logits = torch.zeros(n, b, tp, v, dtype=h0.dtype)
  for tau in range(tp - 1, -1, -1):
    out_ids[:, :, tau] = ids_l[tau][rows, parents]
    out_logits[:, :, tau] = log_l[tau][rows, parents]
    parents = par_l[tau][rows, parents]
  return out_logits, out_ids, score


@torch.no_grad()
def forward(cfg, weights, feeds):
  """Model.build_forward at inference (code/pred_models.py:123-308), fp32, torch CPU."""
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).float() for k, v in weights.items()}
  out = _forward(cfg, w, feeds, torch.float32)
  return {k: ([t.numpy() if torch.is_tensor(t) else t for t in v] if isinstance(v, list) else v)
          for k, v in out.items()}


def scene_input_grad(cfg, weights, feeds, target_labels, scale_idx, dtype=torch.float64, per_sample=False):
  """Truth for SimAug's attack gradient (SimAug/code/pred_models.py:96-115): d sum(sparse CE(logits, target)) /
  d scene_feat through the train-mode forward, by torch autograd.  per_sample=True also returns the per-sample mean
  over the predicted steps of that cross entropy [N] - what multiview_augmentation ranks the views by (:394-397)."""
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dtype) for k, v in weights.items()}
  f = dict(feeds)
  sf = torch.from_numpy(np.ascontiguousarray(feeds["scene_feat"])).to(dtype).requires_grad_(True)
  f["scene_feat"] = sf
  out = _forward(cfg, w, f, dtype)
  h, ww = cfg.scene_grids[scale_idx]
  logits = out["grid_pred_decoded"][scale_idx].reshape(-1, h * ww)
  rows = F.cross_entropy(logits, torch.from_numpy(np.asarray(target_labels)).long().reshape(-1), reduction="none")
  rows.sum().backward()
  if per_sample:
    n = np.asarray(target_labels).shape[0]
    return sf.grad.numpy(), rows.detach().reshape(n, -1).mean(1).numpy()
  return sf.grad.numpy()


def loss_and_grads(cfg, weights, feeds, dtype=torch.float64, device="cpu", return_logits=False):
  """Training objective of Model.build_loss (code/pred_models.py:961-1040) on the greedy
  train-mode forward (train_w_onehot: the class decoder is fed one_hot(argmax), :285) and its
  gradients w.r.t. every trainable variable by torch autograd - the truth for the hand-written
  backward kernels.  Returns (total, [cls_0, reg_0, cls_1, ...], wd_loss, {name: grad}), computed on `device`
  (gradients returned as numpy arrays); with return_logits, also the decoded class logits of every scale
  (numpy [N, Tp, h, w, 1], an empty list for an unused scale) as a fifth element."""
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=dtype).requires_grad_(True)
       for k, v in weights.items()}
  out = _forward(cfg, w, feeds, dtype, device)
  losses = []
  n = cfg.batch_size
  for i, (h, ww) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      continue
    logits = out["grid_pred_decoded"][i].reshape(-1, h * ww)
    labels = torch.from_numpy(feeds["grid_pred_labels"][i]).to(device).long().reshape(-1)
    mixup = feeds.get("mixup")
    if mixup is None:
      cls = F.cross_entropy(logits, labels) * cfg.grid_loss_weight        # :991-995, :1024
    else:
      # SimAug multiview_exp 3 (SimAug/code/pred_models.py:1371-1405): softmax CE against the mixed labels, per-row
      # focal weights under double_weighting, then the mean
      beta = torch.tensor(np.float32(mixup["beta"])).to(device=device, dtype=dtype)
      l2 = torch.from_numpy(np.asarray(mixup["pred_labels2"][i])).to(device).long().reshape(-1)
      soft = F.one_hot(labels, h * ww).to(dtype) * beta + F.one_hot(l2, h * ww).to(dtype) * (1 - beta)
      rows = -(soft * F.log_softmax(logits, dim=1)).sum(1)
      if mixup.get("focal") is not None:
        fw = torch.from_numpy(np.asarray(mixup["focal"])).to(device=device, dtype=dtype)
        rows = rows * fw[:, None].expand(n, cfg.pred_len).reshape(-1)
      cls = rows.mean() * cfg.grid_loss_weight
    tgt = torch.from_numpy(feeds["grid_pred_regress"][i]).to(device=device, dtype=dtype)
    reg = F.huber_loss(out["grid_pred_reg_decoded"][i], tgt, delta=1.0) * cfg.grid_reg_loss_weight
    losses += [cls, reg]
  # wd_cost(".*/W", wd): wd * l2_loss(p) = wd * sum(p^2)/2 for variables whose name ends in /W
  wd = sum(cfg.wd * 0.5 * (v * v).sum() for k, v in w.items() if k.endswith("/W"))
  total = sum(losses) + wd
  total.backward()
  grads = {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in w.items()}
  if return_logits:
    logits = [d.detach().cpu().numpy() if torch.is_tensor(d) else d for d in out["grid_pred_decoded"]]
    return float(total), [float(l) for l in losses], float(wd), grads, logits
  return float(total), [float(l) for l in losses], float(wd), grads


def _forward(cfg, w, feeds, dtype, device=None):
  n = cfg.batch_size
  scene_feat = feeds["scene_feat"] if torch.is_tensor(feeds["scene_feat"]) else torch.from_numpy(feeds["scene_feat"]).to(dtype)
  scene_feat = scene_feat if device is None else scene_feat.to(device)
  obs_scene = torch.from_numpy(feeds["obs_scene"]).to(scene_feat.device).long()
  x = scene_feat[obs_scene.reshape(-1)]              # embedding_lookup, :148-152
  convs = []
  for i in range(len(cfg.scene_grid_strides)):
    x = torch.tanh(conv2d_same(x, w["person_pred/scene_conv%d/W" % (i + 1)], 2)
                   + w["person_pred/scene_conv%d/b" % (i + 1)])
    convs.append(x.reshape((n, -1) + tuple(x.shape[1:])))
  out = dict(grid_pred_decoded=[], grid_pred_reg_decoded=[], beam_outputs=None)
  for i, (h, ww) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      out["grid_pred_decoded"].append([]); out["grid_pred_reg_decoded"].append([])
      continue
    sw = R.scale_weights(w, i)
    labels = torch.from_numpy(feeds["grid_obs_labels"][i]).to(device).long()
    onehot = F.one_hot(labels, h * ww).to(dtype).reshape(n, -1, h, ww, 1)
    mixup = feeds.get("mixup")
    if mixup is not None:      # SimAug multiview_exp 3 (SimAug/code/pred_models.py:616-635): mixed observed class maps
      beta = torch.tensor(np.float32(mixup["beta"])).to(device=device, dtype=dtype)
      other = F.one_hot(torch.from_numpy(np.asarray(mixup["obs_labels2"][i])).to(device).long(), h * ww).to(dtype)
      onehot = beta * onehot + other.reshape(n, -1, h, ww, 1) * (1 - beta)
    obs_reg = torch.from_numpy(feeds["grid_obs_regress"][i]).to(device=device, dtype=dtype)
    mask = neighbour_mask(h, ww, dtype, device)
    enc = encoder(convs[i] * onehot, sw.enc_class[0], sw.enc_class[1], cfg.enc_hidden_size, device)
    enc_r = encoder(obs_reg, sw.enc_reg[0], sw.enc_reg[1], cfg.enc_hidden_size, device)
    scene_mean = convs[i].mean(1)
    if cfg.use_beam_search:
      margins = []
      lg, ids, sc = decoder_beam(onehot[:, -1], enc, cfg.pred_len, cfg.beam_size, sw.dec_class,
                                 sw.emb_class, sw.head_class, scene_mean, mask, cfg.diverse_beam,
                                 cfg.diverse_gamma, cfg.fix_num_timestep, margins)
      out["beam_margins"] = torch.stack(margins, 1).numpy()      # [N, Tp, 2]: test infrastructure (near-tie masks)
      out["beam_outputs"] = [lg.numpy(), ids.numpy().astype(np.int32), sc.numpy()]   # no_grad only
      dec = lg[:, 0].reshape(n, cfg.pred_len, h, ww, 1)
    else:
      # SimAug/code/pred_models.py:1213-1226 concatenates the scene features to the node features only under
      # `if tile_to_beam:` - in SimAug's model the greedy decoder's attention sees h alone (cfg.gnn_scene_in_greedy
      # False); the Multiverse file (code/pred_models.py:824-838) always uses them
      sm_greedy = scene_mean if getattr(cfg, "gnn_scene_in_greedy", True) else None
      dec = decoder_greedy(onehot[:, -1], enc, cfg.pred_len, sw.dec_class, sw.emb_class,
                           sw.head_class, sm_greedy, mask, cfg.use_gnn, True)
    reg = decoder_greedy(obs_reg[:, -1], enc_r, cfg.pred_len, sw.dec_reg, sw.emb_reg, sw.head_reg,
                         None, None, False, False)
    out["grid_pred_decoded"].append(dec)
    out["grid_pred_reg_decoded"].append(reg)
  return out
