# coding=utf-8
"""Training step of the Multiverse ConvRNN (code/pred_models.py: Model.build_loss :961-1040 and
Trainer :1636-1742) as a sequence of libmultiverse_b200 kernel launches: train-mode forward
(train_w_onehot, no teacher forcing - the published configuration) that keeps every step's
operands, loss, hand-written BPTT, element-wise clip + Adadelta, and - across ranks - ONE NCCL
all-reduce of the flat fp32 gradient buffer (SURVEY.md §8e): sum, scale by 1/G inside the
optimizer kernel, then clip, which reproduces the single-GPU batch semantics because every loss
is a mean over equal shards.

Three training options of code/train.py:85-92 change the step: soft grid-class label maps
(--use_soft_grid_class, feeds["grid_pred_labels"][i] fp32 [N,Tp,h,w,1]), the regression loss masked to the cells
whose label is > 0 (--mask_grid_regression, divided by the foreground count K of the whole batch - a device scalar,
all-reduced across ranks) and the class decoder fed its own logits map instead of one_hot(argmax) (no
--train_w_onehot, the train.py default; gradient flows through that feedback).

Per cell step the backward is  lstm_gates_bwd -> cell_dgrad (wgmma) -> cell_wgrad_direct (wgmma,
MN-major operands read straight from the stored planes);  around it: head_bwd, emb_bwd, gnn_bwd, enc_class_input_bwd, scene_*_bwd.
Without use_scene_enc the class encoder's input is embedded by emb_onehot_fwd and its gradient goes through emb_bwd into
the one grid_emb variable every scale and step shares (code/pred_models.py:218-229); there is no scene CNN.
"""
from __future__ import annotations

import math

import torch

from . import ops
from .engine import ENC_EMB, ConvRNNEngine, P_, _names

HID = ops.HIDDEN


class _CellGrad(object):
  """Packed fp32 accumulators of one ConvLSTM cell's weight gradient."""

  def __init__(self, packed, dev):
    self.dwp = torch.zeros((ops.wgrad_slabs(packed.cpad), 4 * HID, 9 * packed.cpad), dtype=torch.float32,
                           device=dev)
    self.dbp = torch.zeros((4 * HID,), dtype=torch.float32, device=dev)

  def zero(self):
    self.dwp.zero_()
    self.dbp.zero_()


class TrainEngine(ConvRNNEngine):
  """ConvRNNEngine + loss + backward + optimizer.  `params` (fp32 device tensors under the TF
  variable names) are the master weights; packed bf16 operand planes are refreshed after every
  update."""
  ALLOW_F16F8 = False

  def __init__(self, cfg, weights, device=None, planes=ops.PLANES_BF16X2):
    super(TrainEngine, self).__init__(cfg, weights, device, planes)
    assert not cfg.use_beam_search, "beam search is inference-only (code/pred_models.py:261)"
    dev = self.device
    self.params = {k: (v if torch.is_tensor(v) else torch.as_tensor(v)).detach().to(dev).float().contiguous()
                   for k, v in weights.items()}
    self.names = sorted(self.params)
    sizes = [self.params[k].numel() for k in self.names]
    self.flat_grad = torch.zeros((sum(sizes),), dtype=torch.float32, device=dev)
    self.grads, off = {}, 0
    for k, n in zip(self.names, sizes):
      self.grads[k] = self.flat_grad[off:off + n].view(self.params[k].shape)
      off += n
    self.acc = {k: torch.zeros_like(v) for k, v in self.params.items()}
    self.acc_upd = {k: torch.zeros_like(v) for k, v in self.params.items()}
    self._repack()
    self._store = {}

  # ------------------------------------------------------------------ weights
  def _repack(self):
    self.set_weights(self.params)
    for i, sw in enumerate(self.scales):
      if sw is None:
        continue
      nm = _names(i)
      for key in ("enc_class", "enc_reg", "dec_class", "dec_reg"):
        ops.pack_dgrad(getattr(sw, key), self.params[nm[key][0]])

  # ------------------------------------------------------------------ storage
  def _steps(self, tag, count, maker):
    lst = self._store.get(tag)
    if lst is None or len(lst) != count:
      lst = [maker() for _ in range(count)]
      self._store[tag] = lst
    return lst

  def _one(self, tag, maker):
    return self._steps(tag, 1, maker)[0]

  # ------------------------------------------------------------------ forward with storage
  def _forward_scale(self, i, feeds, convs, means):
    cfg, dev, P = self.cfg, self.device, self.planes
    h, w = cfg.scene_grids[i]
    sw = self.scales[i]
    T, Tp = cfg.obs_len, cfg.pred_len
    labels_t = feeds["grid_obs_labels"][i].to(torch.int32).t().contiguous()
    obs_scene_t = feeds["obs_scene"].to(torch.int32).t().contiguous()
    tr = feeds.get("traj")
    obs_reg_t = None if tr is not None else feeds["grid_obs_regress"][i].float().transpose(0, 1).contiguous()
    n = labels_t.shape[1]
    mix = feeds.get("mixup")
    labels2_t = mix["obs_labels2"][i].to(torch.int32).t().contiguous() if mix is not None else None
    R = ops.halo_rows(n, h, w)
    st = lambda tag, cnt: self._steps((tag, i, n), cnt, lambda: ops.alloc_state(n, h, w, dev))
    gt = lambda tag, cnt: self._steps((tag, i, n), cnt, lambda: torch.zeros((R, 4 * HID), device=dev))
    xs = lambda tag, cnt, cpad: self._steps((tag, i, n), cnt, lambda: ops.alloc_xh(n, h, w, cpad, P, dev))
    S = dict(n=n, h=h, w=w, labels_t=labels_t, obs_scene_t=obs_scene_t)
    # ---- class encoder
    xh = xs("xh_ec", T, sw.enc_class.cpad); c = st("c_ec", T); g = gt("g_ec", T)
    h32_last = self._one(("h32_ec", i, n), lambda: ops.alloc_state(n, h, w, dev))
    xh_dc = xs("xh_dc", Tp, sw.dec_class.cpad)
    assert sw.enc_emb is None or mix is None, "SimAug's mixup perturbs the scene input, which this model does not have"
    for t in range(T):
      if sw.enc_emb is None:
        xh[t][:, :, :sw.enc_class.cxp].zero_()
      if t == 0:
        xh[0][:, :, sw.enc_class.cxp:].zero_()
      if sw.enc_emb is not None:    # tanh(conv3x3(one_hot(label_t)) + b) into every valid cell of the x block
        ops.emb_onehot_fwd(labels_t[t], *sw.enc_emb, xh[t], h, w)
      elif mix is None:
        ops.enc_class_input(convs[i], obs_scene_t[t], labels_t[t], None, xh[t], h, w)
      else:          # SimAug multiview_exp 3: the observed class map is a mix of two views' one-hot maps
        ops.enc_class_input_mix(convs[i], obs_scene_t[t], labels_t[t], labels2_t[t], mix["beta"], xh[t], h, w)
      last = t == T - 1
      nxt = xh[t + 1] if not last else (None if cfg.use_gnn else xh_dc[0])
      ops.cell_fwd_train(xh[t], sw.enc_class, None if t == 0 else c[t - 1], c[t],
                         h32_last if last else None, nxt, g[t], h, w, n)
    S.update(xh_ec=xh, c_ec=c, g_ec=g, h32_ec=h32_last)
    # ---- class decoder (greedy, one-hot feedback: no gradient through the arg-max; without train_w_onehot the
    # embedded logits map is fed back, :426-435, and the gradient flows through it)
    dense_fb = not getattr(cfg, "train_w_onehot", True)
    assert not (dense_fb and mix is not None), "the logits-fed decoder is not combined with SimAug's mixup"
    head = ops.head_class_fwd_dense if dense_fb else ops.head_class_fwd
    c = st("c_dc", Tp); g = gt("g_dc", Tp); h32 = st("h32_dc", Tp)
    logits = self._one(("logits", i, n), lambda: torch.empty((Tp, n, h * w), device=dev))
    ids = self._one(("ids", i, n), lambda: torch.empty((Tp, n), dtype=torch.int32, device=dev))
    We, be = sw.emb_class
    first_ids = labels_t[-1].contiguous()
    first_map = We_pad = None
    if mix is None:
      ops.emb_onehot_fwd(first_ids, We, be, xh_dc[0], h, w)
    else:
      # the decoder's first input is the MIXED last observed class map (obs_grid_class[:, -1], :690): a two-cell
      # dense map, embedded by the dense-input kernel with the class embedding padded to two input channels
      beta = float(mix["beta"])
      first_map = torch.zeros((n, h * w, 2), dtype=torch.float32, device=dev)
      rows = torch.arange(n, device=dev)
      first_map[:, :, 0].index_put_((rows, first_ids.long()), torch.full((n,), beta, device=dev), accumulate=True)
      first_map[:, :, 0].index_put_((rows, labels2_t[-1].long()), torch.full((n,), 1.0 - beta, device=dev,
                                                                                dtype=torch.float32), accumulate=True)
      We_pad = torch.cat([We, torch.zeros_like(We)], dim=2).contiguous()
      ops.emb_dense_fwd(first_map, We_pad, be, xh_dc[0], h, w)
    for t in range(Tp):
      h_prev = h32_last if t == 0 else h32[t - 1]
      c_prev = S["c_ec"][T - 1] if t == 0 else c[t - 1]
      if cfg.use_gnn:
        ops.gnn_attend_fwd(h_prev, means[i] if self.gnn_scene_in_greedy else None, xh_dc[t], h, w, n)
      last = t == Tp - 1
      ops.cell_fwd_train(xh_dc[t], sw.dec_class, c_prev, c[t], h32[t],
                         None if (cfg.use_gnn or last) else xh_dc[t + 1], g[t], h, w, n)
      head(h32[t], sw.head_class, logits[t], ids[t], None if last else We, None if last else be,
           None if last else xh_dc[t + 1], h, w, n, planes=P)
    S.update(xh_dc=xh_dc, c_dc=c, g_dc=g, h32_dc=h32, logits=logits, ids=ids, first_ids=first_ids,
             first_map=first_map, We_pad=We_pad, labels2_t=labels2_t, mix=mix, dense_fb=dense_fb)
    # ---- regression encoder
    xh = xs("xh_er", T, sw.enc_reg.cpad); c = st("c_er", T); g = gt("g_er", T)
    xh_dr = xs("xh_dr", Tp, sw.dec_reg.cpad)
    xh[0][:, :, sw.enc_reg.cxp:].zero_()
    for t in range(T):
      if tr is None:
        ops.nhwc_to_planes(obs_reg_t[t], xh[t], 0, h, w, comp=sw.enc_reg.comp)
      else:
        ops.traj_to_planes(tr["obs"], t, tr["centers"][i], xh[t], h, w, comp=sw.enc_reg.comp)
      last = t == T - 1
      ops.cell_fwd_train(xh[t], sw.enc_reg, None if t == 0 else c[t - 1], c[t], None,
                         xh_dr[0] if last else xh[t + 1], g[t], h, w, n)
    S.update(xh_er=xh, c_er=c, g_er=g)
    # ---- regression decoder (dense feedback: gradient flows through head -> emb)
    c = st("c_dr", Tp); g = gt("g_dr", Tp); h32 = st("h32_dr", Tp)
    offs = self._one(("offs", i, n), lambda: torch.empty((Tp, n, h * w, 2), device=dev))
    We, be = sw.emb_reg
    if tr is None:
      obs_last = obs_reg_t[-1].reshape(n, h * w, 2)
    else:
      # the last observed offsets [n,HW,2]: the decoder's first input, and what emb_bwd reads for its weight gradient
      obs_last = self._one(("obs_last", i, n), lambda: torch.empty((n, h * w, 2), device=dev))
      scratch = self._one(("obs_last_cell", i, n), lambda: torch.empty((n,), dtype=torch.int32, device=dev))
      vh, vw = getattr(cfg, "video_h", 1080), getattr(cfg, "video_w", 1920)
      ops.traj_to_grid(tr["obs"][:, -1].contiguous(), tr["centers"][i], vh * 1.0 / h, vw * 1.0 / w, scratch, obs_last,
                       h, w)
    ops.emb_dense_fwd(obs_last, We, be, xh_dr[0], h, w)
    for t in range(Tp):
      c_prev = S["c_er"][T - 1] if t == 0 else c[t - 1]
      last = t == Tp - 1
      ops.cell_fwd_train(xh_dr[t], sw.dec_reg, c_prev, c[t], h32[t], None if last else xh_dr[t + 1],
                         g[t], h, w, n)
      ops.head_reg_fwd(h32[t], sw.head_reg, offs[t], None if last else We, None if last else be,
                       None if last else xh_dr[t + 1], h, w, n, planes=P)
    S.update(xh_dr=xh_dr, c_dr=c, g_dr=g, h32_dr=h32, offs=offs, obs_last=obs_last)
    return S

  # ------------------------------------------------------------------ backward helpers
  def _cell_bwd(self, S, i, packed, cg, xh, gates, c_prev, c_new, dh, dc, need_dxh=True, need_dx=True):
    """One BPTT step of a cell: returns (dxh [R,cpad] fp32 or None, dc_prev)."""
    n, h, w = S["n"], S["h"], S["w"]
    dev, P = self.device, self.planes
    R = ops.halo_rows(n, h, w)
    dg = self._one(("dg", i, n), lambda: torch.zeros((P, R, 4 * HID), dtype=torch.bfloat16, device=dev))
    dc_prev = self._steps(("dc_pp", i, n), 2, lambda: ops.alloc_state(n, h, w, dev))
    out_dc = dc_prev[0] if dc is not dc_prev[0] else dc_prev[1]
    ops.lstm_gates_bwd(gates, c_prev, c_new, dh, dc, dg, out_dc, cg.dbp, h, w, n)
    dxh = None
    if need_dxh:
      dxh = self._one(("dxh", i, n, packed.cpad), lambda: torch.zeros((R, packed.cpad), device=dev))
      ops.cell_dgrad(dg, packed.wd, dxh, h, w, n, need_dx=need_dx)
    ops.cell_wgrad_direct(dg, xh, cg.dwp, h, w, n)     # MN-major operands: no transposed copies
    return dxh, out_dc

  def _backward_scale(self, i, S, feeds, convs, means, dconv, loss_out, cw, rw, fg=None):
    cfg, dev = self.cfg, self.device
    n, h, w = S["n"], S["h"], S["w"]
    sw = self.scales[i]
    nm = _names(i)
    T, Tp = cfg.obs_len, cfg.pred_len
    G = self.grads
    cgr = {k: self._one(("cg", i, k), lambda k=k: _CellGrad(getattr(sw, k), dev))
           for k in ("enc_class", "enc_reg", "dec_class", "dec_reg")}
    for v in cgr.values():
      v.zero()
    dh = self._one(("dh", i, n), lambda: ops.alloc_state(n, h, w, dev))
    # ---- losses and their gradients (Model.build_loss :988-1027)
    lab_in = feeds["grid_pred_labels"][i]
    tr = feeds.get("traj")         # trajectory feeds: targets and label maps are computed in the loss kernels
    soft = tr is None and lab_in.dim() > 2                                         # [N,Tp,h,w,1] label maps
    if soft:
      lab = lab_in.float().reshape(n, Tp, h * w).transpose(0, 1).contiguous()   # [Tp,N,HW]
    else:
      lab = lab_in.to(torch.int32).t().contiguous()                              # [Tp,N]
    tgt = None if tr is not None else \
        feeds["grid_pred_regress"][i].float().transpose(0, 1).reshape(Tp, n, h * w, 2).contiguous()
    dlogits = self._one(("dlogits", i, n), lambda: torch.empty_like(S["logits"]))
    doffs = self._one(("doffs", i, n), lambda: torch.empty_like(S["offs"]))
    mix = S["mix"]
    assert mix is None or not (soft or fg is not None), "soft labels / masked regression with SimAug's mixup"
    assert mix is None or tr is None, "SimAug's mixup keeps the dense feeds"
    if tr is not None:
      mode, pred, centers = tr["soft_grid"], tr["pred"], tr["centers"][i]
      if mode:
        ops.soft_ce_label_fwd_bwd(S["logits"], lab, mode, h, w, dlogits, cw, loss_out)
      else:
        ops.loss_fwd_bwd(S["logits"], lab, dlogits, cw, None, None, None, 0.0, loss_out)
      if fg is not None:
        ops.masked_huber_traj_fwd_bwd(S["offs"], pred, centers, doffs, lab, mode, h, w, fg[0], fg[1], loss_out)
      else:
        ops.huber_traj_fwd_bwd(S["offs"], pred, centers, doffs, rw, loss_out)
    elif mix is None and not soft and fg is None:
      ops.loss_fwd_bwd(S["logits"], lab, dlogits, cw, S["offs"], tgt, doffs, rw, loss_out)
    elif mix is None:
      if soft:
        ops.soft_ce_fwd_bwd(S["logits"], lab, dlogits, cw, loss_out)
      else:
        ops.loss_fwd_bwd(S["logits"], lab, dlogits, cw, None, None, None, 0.0, loss_out)
      if fg is not None:                    # (fg count [1] fp64, weight): mean over the foreground of the whole batch
        ops.masked_huber_fwd_bwd(S["offs"], tgt, doffs, lab, fg[0], fg[1], loss_out)
      else:
        ops.loss_fwd_bwd(None, None, None, 0.0, S["offs"], tgt, doffs, rw, loss_out)
    else:
      # mixed labels (SimAug/code/pred_models.py:1371-1405): softmax CE against beta one_hot(l1) + (1-beta) one_hot(l2)
      # = beta CE(l1) + (1-beta) CE(l2), optionally times the per-sample focal weight (double_weighting)
      beta = float(mix["beta"])
      lab2 = mix["pred_labels2"][i].to(torch.int32).t().contiguous()             # [Tp,N]
      focal = mix.get("focal")
      rowl = beta * ops.ce_rows(S["logits"], lab) + (1.0 - beta) * ops.ce_rows(S["logits"], lab2)
      if focal is not None:
        rowl = rowl * focal.float()[None, :]
      loss_out[0] += rowl.mean() * cw
      scratch = torch.zeros(2, dtype=torch.float32, device=dev)
      dl2 = self._one(("dlogits2", i, n), lambda: torch.empty_like(S["logits"]))
      ops.loss_fwd_bwd(S["logits"], lab, dlogits, cw * beta, None, None, None, 0.0, scratch)
      ops.loss_fwd_bwd(S["logits"], lab2, dl2, cw * (1.0 - beta), None, None, None, 0.0, scratch)
      dlogits += dl2
      if focal is not None:
        dlogits *= focal.float()[None, :, None]
      ops.loss_fwd_bwd(None, None, None, 0.0, S["offs"], tgt, doffs, rw, loss_out)
    # ---- class decoder
    dsm = None
    if self.scene_enc:
      dsm = self._one(("dsm", i, n), lambda: torch.zeros_like(means[i]))
      dsm.zero_()
    work = self._one(("gnnwork", i, n), lambda: torch.empty((19 * n * h * w,), device=dev))
    We, be = sw.emb_class
    dc = None
    for t in range(Tp - 1, -1, -1):
      ops.head_bwd(S["h32_dc"][t], dlogits[t], sw.head_class, G[nm["head_class"]], dh, t < Tp - 1, h, w, n)
      c_prev = S["c_ec"][T - 1] if t == 0 else S["c_dc"][t - 1]
      dxh, dc = self._cell_bwd(S, i, sw.dec_class, cgr["dec_class"], S["xh_dc"][t], S["g_dc"][t], c_prev,
                               S["c_dc"][t], dh, dc)
      ids_prev = S["first_ids"] if t == 0 else S["ids"][t - 1]
      if t == 0 and mix is not None:       # the mixed two-cell first input: dense path, padded embedding
        dWe_pad = torch.zeros_like(S["We_pad"])
        ops.emb_bwd(dxh, None, S["first_map"], S["We_pad"], be, dWe_pad, G[nm["emb_class"][1]], None, False, h, w, n)
        G[nm["emb_class"][0]] += dWe_pad[:, :, :1]
      elif t > 0 and S["dense_fb"]:         # input = logits[t-1]: its gradient joins dlogits[t-1] before head_bwd reads it
        ops.emb_bwd(dxh, None, S["logits"][t - 1], We, be, G[nm["emb_class"][0]], G[nm["emb_class"][1]],
                    dlogits[t - 1], True, h, w, n)
      else:
        ops.emb_bwd(dxh, ids_prev, None, We, be, G[nm["emb_class"][0]], G[nm["emb_class"][1]], None, False, h, w, n)
      gout = dxh[:, sw.dec_class.cxp:].contiguous()
      if cfg.use_gnn:
        h_prev = S["h32_ec"] if t == 0 else S["h32_dc"][t - 1]
        if self.gnn_scene_in_greedy:
          ops.gnn_bwd(h_prev, means[i], gout, work, dh, False, dsm, h, w, n)
        else:
          ops.gnn_bwd(h_prev, None, gout, work, dh, False, None, h, w, n)
      else:
        dh.copy_(gout)
    # ---- class encoder
    for t in range(T - 1, -1, -1):
      dxh, dc = self._cell_bwd(S, i, sw.enc_class, cgr["enc_class"], S["xh_ec"][t], S["g_ec"][t],
                               None if t == 0 else S["c_ec"][t - 1], S["c_ec"][t], dh, dc)
      if sw.enc_emb is not None:    # summed over steps and scales (the kernel adds into the shared gradient)
        ops.emb_bwd(dxh, S["labels_t"][t], None, *sw.enc_emb, G[ENC_EMB[0]], G[ENC_EMB[1]], None, False, h, w, n)
      elif mix is None:
        ops.enc_class_input_bwd(dxh, S["obs_scene_t"][t], S["labels_t"][t], dconv[i], h, w)
      else:
        ops.enc_class_input_mix_bwd(dxh, S["obs_scene_t"][t], S["labels_t"][t], S["labels2_t"][t], mix["beta"],
                                    dconv[i], h, w)
      if t > 0:
        dh.copy_(dxh[:, sw.enc_class.cxp:])
    if self.gnn_scene_in_greedy:
      ops.scene_time_mean_bwd(dsm, feeds["obs_scene"].to(torch.int32).contiguous(), dconv[i])
    # ---- regression decoder
    We, be = sw.emb_reg
    dc = None
    for t in range(Tp - 1, -1, -1):
      ops.head_bwd(S["h32_dr"][t], doffs[t], sw.head_reg, G[nm["head_reg"]], dh, t < Tp - 1, h, w, n)
      c_prev = S["c_er"][T - 1] if t == 0 else S["c_dr"][t - 1]
      dxh, dc = self._cell_bwd(S, i, sw.dec_reg, cgr["dec_reg"], S["xh_dr"][t], S["g_dr"][t], c_prev,
                               S["c_dr"][t], dh, dc)
      in_map = S["obs_last"] if t == 0 else S["offs"][t - 1]
      ops.emb_bwd(dxh, None, in_map, We, be, G[nm["emb_reg"][0]], G[nm["emb_reg"][1]],
                  None if t == 0 else doffs[t - 1], True, h, w, n)
      dh.copy_(dxh[:, sw.dec_reg.cxp:])
    # ---- regression encoder (its input is data: only the h path is propagated)
    for t in range(T - 1, -1, -1):
      dxh, dc = self._cell_bwd(S, i, sw.enc_reg, cgr["enc_reg"], S["xh_er"][t], S["g_er"][t],
                               None if t == 0 else S["c_er"][t - 1], S["c_er"][t], dh, dc, need_dxh=t > 0,
                               need_dx=False)
      if t > 0:
        dh.copy_(dxh[:, sw.enc_reg.cxp:])
    # ---- packed accumulators -> gradients of the TF variables
    for key in ("enc_class", "enc_reg", "dec_class", "dec_reg"):
      pk = getattr(sw, key)
      ops.unpack_cell_wgrad(cgr[key].dwp, cgr[key].dbp, G[nm[key][0]], G[nm[key][1]], pk.cx, comp=pk.comp,
                            accumulate=True)

  # ------------------------------------------------------------------ public
  def fg_counts(self, feeds):
    """Foreground size K of the masked regression loss per scale (fp64 [scales] on the device, no host sync): the
    cells whose label is > 0 of the soft maps, or the in-range label cells of sparse labels.  With trajectory feeds
    the soft maps are those of the label cells under feeds["traj"]["soft_grid"]."""
    cfg = self.cfg
    K = torch.zeros((len(cfg.scene_grids),), dtype=torch.float64, device=self.device)
    tr = feeds.get("traj")
    for i, (h, w) in enumerate(cfg.scene_grids):
      if cfg.use_grids[i]:
        lab = feeds["grid_pred_labels"][i]
        if tr is not None and tr["soft_grid"]:
          ops.fg_count_label(lab.to(torch.int32).contiguous(), tr["soft_grid"], h, w, K[i:i + 1])
          continue
        lab = lab.float().contiguous() if lab.dim() > 2 else lab.to(torch.int32).contiguous()
        ops.fg_count(lab, h * w, K[i:i + 1])
    return K

  def loss_and_grads(self, feeds, loss_scale=1.0, zero=True, dscene_out=None, cls_weight=None, reg_weight=None,
                     fg_count=None):
    """Forward + loss + backward.  feeds additionally needs grid_pred_labels[i] int32 [N,Tp] and
    grid_pred_regress[i] fp32 [N,Tp,h,w,2] - or, instead of grid_obs_regress and grid_pred_regress, the trajectory
    feeds feeds["traj"] = dict(obs fp64 [N,T,2], pred fp64 [N,Tp,2], centers [scale] fp64 [h,w,2] (None for an unused
    scale), soft_grid: the --soft_grid mode of the label maps, 0 for sparse labels) with int32 label cells in
    grid_pred_labels: the offsets, targets and label maps are then computed by the kernels that read them, bit-identical
    to the dense feeds float32(trajectory - centre) and pred_models._soft_labels.  Returns (losses fp32 tensor [2*scales] on device in
    the reference's order cls_0, reg_0, cls_1, ..., wd_loss tensor); gradients are ADDED into
    self.grads (TF variable names; zeroed first unless zero=False), WITHOUT the weight-decay term
    (added by the optimizer).  loss_scale weights this call's batch inside a larger one
    (micro-batching: n_chunk / N, every loss being a batch mean).
    dscene_out (fp32 [F,SH,SW,SC], zeroed by the caller): receives d loss / d scene_feat - the input gradient of
    SimAug's white-box attack (SURVEY.md section 8 row f-4); cls_weight / reg_weight override the config's loss
    weights for this call (the attack differentiates the classification loss alone).
    feeds["mixup"] (optional; SimAug multiview_exp 3, SimAug/code/pred_models.py:616-638, :1371-1405) =
    dict(beta, obs_labels2[i] int [N,T], pred_labels2[i] int [N,Tp], focal fp32 [N] or None): the observed class
    maps (encoder input and the decoder's first input) and the loss labels become beta * view 1 + (1 - beta) * view 2,
    the per-sample classification losses are weighted by `focal`.
    grid_pred_labels[i] may be fp32 label maps [N,Tp,h,w,1] (--use_soft_grid_class).  Under cfg.mask_grid_regression
    the regression loss is divided by fg_count[i] (fg_counts of the whole batch this call is part of; loss_scale then
    does not apply to it), or by this call's own count when fg_count is None."""
    cfg, dev = self.cfg, self.device
    cls_w = cfg.grid_loss_weight if cls_weight is None else cls_weight
    reg_w = cfg.grid_reg_loss_weight if reg_weight is None else reg_weight
    if zero:
      self.flat_grad.zero_()
    obs_scene = feeds["obs_scene"].to(torch.int32).contiguous()
    scene_feat = feeds["scene_feat"].float().contiguous()
    convs, means = self.scene_cnn(scene_feat, obs_scene)
    used = [i for i in range(len(cfg.scene_grids)) if cfg.use_grids[i]]
    loss_out = torch.zeros((len(cfg.scene_grids), 2), dtype=torch.float32, device=dev)
    dconv = [None if c is None else torch.zeros_like(c) for c in convs]
    assert dscene_out is None or self.scene_enc, "the scene-input gradient needs a model that encodes the scene"
    fg = None
    mask = getattr(cfg, "mask_grid_regression", False)
    assert fg_count is None or mask, "fg_count is the denominator of the masked regression loss (mask_grid_regression)"
    if mask:
      if fg_count is None:
        fg_count, fg_w = self.fg_counts(feeds), reg_w * loss_scale
      else:
        fg_w = reg_w
    self.last_logits = {}      # scale -> class logits [Tp,N,HW] of this call's train-mode forward (engine buffers)
    for i in used:
      S = self._forward_scale(i, feeds, convs, means)
      self.last_logits[i] = S["logits"]
      if fg_count is not None:
        fg = (fg_count[i:i + 1], fg_w)
      self._backward_scale(i, S, feeds, convs, means, dconv, loss_out[i],
                           cls_w * loss_scale, reg_w * loss_scale, fg)
    # scene CNN backward: conv_k -> conv_{k-1} chain (code/pred_models.py:155-165)
    ins = [scene_feat] + convs[:-1]
    for k in range(len(self.scene_w) - 1, -1, -1):
      W, _ = self.scene_w[k]
      ops.scene_conv_bwd(ins[k], W, convs[k], dconv[k], self.grads[P_ + "scene_conv%d/W" % (k + 1)],
                         self.grads[P_ + "scene_conv%d/b" % (k + 1)], dconv[k - 1] if k > 0 else dscene_out)
    wd = sum(0.5 * cfg.wd * (self.params[k] * self.params[k]).sum() for k in self.names if k.endswith("/W"))
    return loss_out[used].reshape(-1), wd

  def apply_gradients(self, lr, world=1):
    """Element-wise clip (+-clip_gradient_norm, :1700-1705) + Adadelta (:1672), weight decay on the
    variables named .../W (:1033), gradients pre-scaled by 1/world after an all-reduce SUM."""
    cfg = self.cfg
    clip = getattr(cfg, "clip_gradient_norm", None) or 0.0
    opt = getattr(cfg, "optimizer", "adadelta")
    if opt != "adadelta" and not getattr(self, "_opt_slots_ready", False):
      if opt == "rmsprop":                      # TF initialises the RMSProp mean-square slot to ones
        for k in self.names:
          self.acc[k].fill_(1.0)
      self._opt_steps, self._opt_slots_ready = 0, True
    if opt == "adam":
      self._opt_steps += 1
      t = self._opt_steps
      lr = lr * math.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t)
    for k in self.names:
      wd = cfg.wd if k.endswith("/W") else 0.0
      if opt == "adadelta":                     # tf.train.AdadeltaOptimizer(lr): rho 0.95, eps 1e-8
        ops.clip_adadelta(self.params[k], self.grads[k], self.acc[k], self.acc_upd[k], lr, clip, wd, 1.0 / world)
      elif opt == "momentum":                   # MomentumOptimizer(lr, momentum=0.9), :1668
        ops.clip_update(self.params[k], self.grads[k], self.acc[k], self.acc_upd[k], 1, lr, 0.9, 0.0, 0.0, clip, wd, 1.0 / world)
      elif opt == "adam":                       # AdamOptimizer(lr): beta1 .9, beta2 .999, eps 1e-8, :1675
        ops.clip_update(self.params[k], self.grads[k], self.acc[k], self.acc_upd[k], 2, lr, 0.9, 0.999, 1e-8, clip, wd, 1.0 / world)
      elif opt == "rmsprop":                    # RMSPropOptimizer(lr): decay .9, momentum 0, eps 1e-10, :1678
        ops.clip_update(self.params[k], self.grads[k], self.acc[k], self.acc_upd[k], 3, lr, 0.9, 0.0, 1e-10, clip, wd, 1.0 / world)
      else:
        raise ValueError("Optimizer not implemented: %r" % (opt,))      # :1681
    self._repack()

  def loss_and_grads_chunked(self, feeds, micro_batch, fg_count=None):
    """loss_and_grads over a batch larger than the activation store allows: gradient
    accumulation over contiguous chunks (identical result - every loss is a batch mean; the masked regression loss,
    whose foreground differs per chunk, divides every chunk by the foreground count of the whole batch)."""
    n = feeds["obs_scene"].shape[0]
    if fg_count is None and getattr(self.cfg, "mask_grid_regression", False):
      fg_count = self.fg_counts(feeds)
    if not micro_batch or n <= micro_batch:
      return self.loss_and_grads(feeds, fg_count=fg_count)
    assert n % micro_batch == 0, "batch must be a multiple of the micro batch"
    total, wd = None, None
    for lo in range(0, n, micro_batch):
      sl = slice(lo, lo + micro_batch)
      uniq, inv = torch.unique(feeds["obs_scene"][sl], return_inverse=True)
      part = dict(scene_feat=feeds["scene_feat"][uniq.long()].contiguous(), obs_scene=inv.to(torch.int32))
      for key in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
        part[key] = [None if a is None else a[sl] for a in feeds[key]]
      if feeds.get("traj") is not None:
        part["traj"] = dict(feeds["traj"], obs=feeds["traj"]["obs"][sl], pred=feeds["traj"]["pred"][sl])
      if feeds.get("mixup") is not None:
        mx = feeds["mixup"]
        part["mixup"] = dict(beta=mx["beta"], obs_labels2=[None if a is None else a[sl] for a in mx["obs_labels2"]],
                             pred_labels2=[None if a is None else a[sl] for a in mx["pred_labels2"]],
                             focal=None if mx.get("focal") is None else mx["focal"][sl])
      losses, wd = self.loss_and_grads(part, loss_scale=micro_batch / float(n), zero=(lo == 0), fg_count=fg_count)
      total = losses if total is None else total + losses
    return total, wd

  def train_step(self, feeds, lr, dist=None, micro_batch=0):
    world = 1
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
      world = dist.get_world_size()
    fg_count = None
    if getattr(self.cfg, "mask_grid_regression", False):
      fg_count = self.fg_counts(feeds)
      if world > 1:
        # the gradients are summed over ranks and scaled by 1/world: dividing by K_all / world makes that sum the
        # mean over the foreground of the global batch
        dist.all_reduce(fg_count)
        fg_count /= world
    losses, wd = self.loss_and_grads_chunked(feeds, micro_batch, fg_count)
    if world > 1:
      ev = getattr(self, "allreduce_events", None)   # bench.py: CUDA events around the collective
      if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
      dist.all_reduce(self.flat_grad)                # the one collective of the path
      if ev is not None:
        e1.record()
        ev.append((e0, e1))
      dist.all_reduce(losses)
      losses = losses / world
    self.apply_gradients(lr, world)
    return losses, wd
