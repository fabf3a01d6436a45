# coding=utf-8
"""fp64 truth for models built without --use_scene_enc, on the oracle's pieces (oracle/multiverse_ref.py and its torch
restatement).  Without scene encoding code/pred_models.py creates no scene CNN (:146-165), feeds the class encoder
grid_emb(one_hot(label_t)) = tanh(conv3x3(one_hot) + b) through the variable person_pred/grid_emb that every scale
shares (:218-229, conv2d's AUTO_REUSE :1339), and its graph attention sees h alone (:824-838).

Test infrastructure; tests/test_no_scene_enc_cpu.py pins it to executions of the unmodified reference
(tests/golden/make_golden_no_scene_enc.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import multiverse_ref as R
from oracle import multiverse_ref_torch as RT

ENC_EMB = ("person_pred/grid_emb/W", "person_pred/grid_emb/b")

# name: (oracle.default_config overrides, seed); every case has use_scene_enc off
ROLLOUTS = {
    # test.py: greedy decode of both scales with graph attention
    "greedy_two_scale": (dict(batch_size=3, use_gnn=True), 71),
    # multifuture_inference.py --use_gnn: K = 20 diverse beam on 36x18 (60 beam rows: the CTA-pair cell kernel)
    "beam_k20_gnn": (dict(batch_size=3, use_grids=[True, False], use_beam_search=True, beam_size=20,
                          diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=True), 72),
    # test.py --use_beam_search without --use_gnn: K = 5 plain beam on 18x9.  Without scene features the logits of
    # cells far from the trajectory nearly tie, so selections near a tie are common: seeds 73-82 and 84-89 put some
    # selection of the fp64 reference within 2e-4 of a tie; 83 is the first that clears it
    "beam_k5_nognn": (dict(batch_size=2, use_grids=[False, True], use_beam_search=True, beam_size=5,
                           diverse_beam=False, fix_num_timestep=0, use_gnn=False), 83),
}
# TRAINING.md's arguments without --use_scene: scene 36x64 (grids 18x32 and 9x16), loss weights 1.0 / 0.2, wd 0.001,
# init_lr 0.3, clip 10, Adadelta
TRAIN = (dict(batch_size=2, scene_h=36, scene_w=64, use_gnn=True, grid_loss_weight=1.0, grid_reg_loss_weight=0.2,
              wd=0.001, init_lr=0.3, clip_gradient_norm=10.0, optimizer="adadelta"), 75)


def config(**over):
  return R.default_config(**dict(over, use_scene_enc=False))


def forward(cfg, weights, feeds, dtype=np.float64, return_intermediates=False):
  """R.forward (Model.build_forward at inference) without scene encoding."""
  assert not cfg.use_scene_enc
  weights = R.cast_tree(weights, dtype)
  feeds = R.cast_tree(feeds, dtype)
  n = cfg.batch_size
  res = dict(grid_pred_decoded=[], grid_pred_reg_decoded=[], beam_outputs=None, inter=[])
  for i, (h, w) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      res["grid_pred_decoded"].append([])
      res["grid_pred_reg_decoded"].append([])
      res["inter"].append(None)
      continue
    sw = R.scale_weights(weights, i)
    obs_onehot = R.one_hot(feeds["grid_obs_labels"][i], h * w, dtype).reshape(n, -1, h, w, 1)    # :174-175
    emb = R.grid_emb(obs_onehot.reshape(-1, h, w, 1), weights[ENC_EMB[0]], weights[ENC_EMB[1]])  # :221-225
    enc_state = R.encoder(emb.reshape(n, -1, h, w, cfg.emb_size), sw.enc_class[0], sw.enc_class[1],
                          cfg.enc_hidden_size)
    obs_reg = feeds["grid_obs_regress"][i]
    enc_reg_state = R.encoder(obs_reg, sw.enc_reg[0], sw.enc_reg[1], cfg.enc_hidden_size)
    if cfg.use_beam_search:
      best, logits, ids, logprobs = R.grid_decoder_beam_search(
          obs_onehot[:, -1], enc_state, cfg.pred_len, cfg.beam_size, sw.dec_class, sw.emb_class, sw.head_class,
          scene_mean=None, use_gnn=cfg.use_gnn, diverse_beam=cfg.diverse_beam, diverse_gamma=cfg.diverse_gamma,
          fix_num_timestep=cfg.fix_num_timestep)
      res["beam_outputs"] = [logits, ids, logprobs]
      dec = best
    else:
      dec, _ = R.grid_decoder(obs_onehot[:, -1], enc_state, cfg.pred_len, sw.dec_class, sw.emb_class, sw.head_class,
                              scene_mean=None, use_gnn=cfg.use_gnn, input_onehot=True)
    reg, _ = R.grid_decoder(obs_reg[:, -1], enc_reg_state, cfg.pred_len, sw.dec_reg, sw.emb_reg, sw.head_reg,
                            use_gnn=False, input_onehot=False)
    res["grid_pred_decoded"].append(dec)
    res["grid_pred_reg_decoded"].append(reg)
    res["inter"].append(dict(enc_state=enc_state, enc_reg_state=enc_reg_state, obs_onehot=obs_onehot)
                        if return_intermediates else None)
  return res


def decoder_greedy_fed(first, state, cell_w, emb_w, head_w, mask, use_gnn, ids):
  """RT.decoder_greedy with one_hot(ids[:, t]) fed back instead of one_hot(argmax): the class decoder on a given
  arg-max path (no gradient flows through the arg-max, so the loss along that path is the training objective)."""
  c, h = state
  n, hh, ww, _ = first.shape
  inp, outs = first, []
  for t in range(ids.shape[1]):
    h_in = RT.gnn_dense(h, None, mask) if use_gnn else h
    c, h = RT.convlstm_cell(RT.grid_emb(inp, *emb_w), c, h_in, *cell_w)
    outs.append(RT.conv2d_same(h, head_w))
    inp = RT.one_hot_map(ids[:, t], hh, ww, h.dtype)
  return torch.stack(outs, 1)


def loss_and_grads(cfg, weights, feeds, dtype=torch.float64, device="cpu", return_logits=False, fed_ids=None):
  """(total, [cls_0, reg_0, ...], wd, {name: grad} as numpy[, logits per scale]) of Model.build_loss on the greedy
  train-mode forward (train_w_onehot) without scene encoding, by torch autograd.  fed_ids[i] int [N,Tp]: the class
  decoder of scale i follows that arg-max path (decoder_greedy_fed)."""
  assert not cfg.use_scene_enc
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=dtype).requires_grad_(True)
       for k, v in weights.items()}
  n = cfg.batch_size
  losses, logits_out = [], []
  for i, (h, ww) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      logits_out.append([])
      continue
    sw = R.scale_weights(w, i)
    labels = torch.from_numpy(np.asarray(feeds["grid_obs_labels"][i])).to(device).long()
    obs_cls = F.one_hot(labels, h * ww).to(dtype).reshape(n, -1, h, ww, 1)
    emb = RT.grid_emb(obs_cls.reshape(-1, h, ww, 1), w[ENC_EMB[0]], w[ENC_EMB[1]]).reshape(n, -1, h, ww, cfg.emb_size)
    obs_reg = torch.from_numpy(np.asarray(feeds["grid_obs_regress"][i])).to(device=device, dtype=dtype)
    mask = RT.neighbour_mask(h, ww, dtype, device)
    enc = RT.encoder(emb, sw.enc_class[0], sw.enc_class[1], cfg.enc_hidden_size, device)
    enc_r = RT.encoder(obs_reg, sw.enc_reg[0], sw.enc_reg[1], cfg.enc_hidden_size, device)
    if fed_ids is None:
      cls = RT.decoder_greedy(obs_cls[:, -1], enc, cfg.pred_len, sw.dec_class, sw.emb_class, sw.head_class, None, mask,
                              cfg.use_gnn, True)
    else:
      cls = decoder_greedy_fed(obs_cls[:, -1], enc, sw.dec_class, sw.emb_class, sw.head_class, mask, cfg.use_gnn,
                               torch.as_tensor(np.asarray(fed_ids[i])).to(device).long())
    reg = RT.decoder_greedy(obs_reg[:, -1], enc_r, cfg.pred_len, sw.dec_reg, sw.emb_reg, sw.head_reg, None, None,
                            False, False)
    lab = torch.from_numpy(np.asarray(feeds["grid_pred_labels"][i])).to(device).long().reshape(-1)
    tgt = torch.from_numpy(np.asarray(feeds["grid_pred_regress"][i])).to(device=device, dtype=dtype)
    losses += [F.cross_entropy(cls.reshape(-1, h * ww), lab) * cfg.grid_loss_weight,
               F.huber_loss(reg, tgt, delta=1.0) * cfg.grid_reg_loss_weight]
    logits_out.append(cls.detach().cpu().numpy())
  wd = sum(cfg.wd * 0.5 * (v * v).sum() for k, v in w.items() if k.endswith("/W"))     # wd_cost(".*/W"), :1033
  total = sum(losses) + wd
  total.backward()
  grads = {k: (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in w.items()}
  res = (float(total.detach()), [float(l.detach()) for l in losses], float(wd.detach()), grads)
  if return_logits:
    res += (logits_out,)
  return res


def beam_replay(cfg, weights, feeds, i, step_ids, step_par, dtype=torch.float64, device="cpu"):
  """The beam decoder of scale i without scene features (RT.decoder_beam's steps, scene_mean None) with its
  selections given: the cells step_ids[t] and parent beams step_par[t] [N,K] of every step, e.g. an engine's trace.
  Returns the logits [Tp,N,K,V] that every live beam row computes along those selections.  Without scene features far
  cells' log-probabilities nearly tie inside a row, and the diverse penalty (log gamma x rank in the row) turns a swap
  of two such siblings into other selections: a comparison along the engine's own selections stays well posed."""
  w = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=dtype) for k, v in weights.items()}
  n, b = cfg.batch_size, cfg.beam_size
  h, ww = cfg.scene_grids[i]
  sw = R.scale_weights(w, i)
  labels = torch.from_numpy(np.asarray(feeds["grid_obs_labels"][i])).to(device).long()
  obs_cls = F.one_hot(labels, h * ww).to(dtype).reshape(n, -1, h, ww, 1)
  emb = RT.grid_emb(obs_cls.reshape(-1, h, ww, 1), w[ENC_EMB[0]], w[ENC_EMB[1]]).reshape(n, -1, h, ww, cfg.emb_size)
  c, hs = RT.encoder(emb, sw.enc_class[0], sw.enc_class[1], cfg.enc_hidden_size, device)
  mask = RT.neighbour_mask(h, ww, dtype, device) if cfg.use_gnn else None

  def step(inp, c, hs):
    h_in = RT.gnn_dense(hs, None, mask) if cfg.use_gnn else hs
    return RT.convlstm_cell(RT.grid_emb(inp, *sw.emb_class), c, h_in, *sw.dec_class)

  c, hs = step(obs_cls[:, -1], c, hs)                     # time 0: the K beams of a sample are identical
  c, hs = c.repeat_interleave(b, 0), hs.repeat_interleave(b, 0)
  base = torch.arange(n, device=device)[:, None] * b
  out = []
  for t in range(len(step_ids)):
    out.append(RT.conv2d_same(hs, sw.head_class).reshape(n, b, -1))
    flat = (torch.as_tensor(np.asarray(step_par[t])).to(device).long() + base).reshape(-1)
    c, hs = c[flat], hs[flat]
    if t == len(step_ids) - 1:
      break
    inp = RT.one_hot_map(torch.as_tensor(np.asarray(step_ids[t])).reshape(-1), h, ww, dtype, device)
    c, hs = step(inp, c, hs)
  return torch.stack(out).cpu().numpy()
