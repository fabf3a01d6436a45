# coding=utf-8
"""fp64 truths of the decoders of one grid scale on the oracle's pieces (oracle/multiverse_ref_torch.py), on any torch
device: the class decoder's beam replayed along given selections (an engine's trace), the fp64 beam search itself with
its per-step trace and selection margins, the greedy class decoder along given arg-max ids, and the regression decoder.
Test infrastructure; tests/test_beam_truth_cpu.py ties beam_replay to RT.decoder_beam."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import multiverse_ref as R
from oracle import multiverse_ref_torch as RT

DT = torch.float64


def _weights(weights, device):
  return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=DT) for k, v in weights.items()}


def class_inputs(cfg, weights, feeds, i, device):
  """(scale weights, first input one_hot(last observed cell) [N,h,w,1], encoder state (c, h), scene mean [N,h,w,64] or
  None without scene encoding, attention mask or None without use_gnn) of the class decoder of scale i."""
  import no_scene_enc_ref as NS
  w = _weights(weights, device)
  n = cfg.batch_size
  h, ww = cfg.scene_grids[i]
  sw = R.scale_weights(w, i)
  labels = torch.from_numpy(np.asarray(feeds["grid_obs_labels"][i])).to(device).long()
  obs = F.one_hot(labels, h * ww).to(DT).reshape(n, -1, h, ww, 1)
  if cfg.use_scene_enc:
    x = torch.from_numpy(feeds["scene_feat"]).to(device=device, dtype=DT)[
        torch.from_numpy(feeds["obs_scene"]).long().reshape(-1).to(device)]
    for j in range(i + 1):
      x = torch.tanh(RT.conv2d_same(x, w["person_pred/scene_conv%d/W" % (j + 1)], 2)
                     + w["person_pred/scene_conv%d/b" % (j + 1)])
    conv = x.reshape((n, -1) + tuple(x.shape[1:]))
    enc_in, sm = conv * obs, conv.mean(1)
  else:
    enc_in = RT.grid_emb(obs.reshape(-1, h, ww, 1), w[NS.ENC_EMB[0]], w[NS.ENC_EMB[1]]).reshape(n, -1, h, ww,
                                                                                               cfg.emb_size)
    sm = None
  state = RT.encoder(enc_in, sw.enc_class[0], sw.enc_class[1], cfg.enc_hidden_size, device)
  mask = RT.neighbour_mask(h, ww, DT, device) if cfg.use_gnn else None
  return sw, obs[:, -1], state, sm, mask


def beam_replay(cfg, weights, feeds, i, step_ids, step_par, device):
  """The fp64 truth of the beam decoder of scale i (RT.decoder_beam's steps) with its selections given: the cells
  step_ids[t] and parent beams step_par[t] [N,K] of every step, e.g. an engine's trace.  Returns the logits [Tp,N,K,V]
  every live beam row computes along those selections.  Without scene encoding: no_scene_enc_ref.beam_replay."""
  import no_scene_enc_ref as NS
  if not cfg.use_scene_enc:
    return NS.beam_replay(cfg, weights, feeds, i, step_ids, step_par, device=device)
  n, b = cfg.batch_size, cfg.beam_size
  h, ww = cfg.scene_grids[i]
  sw, first, (c, hs), sm, mask = class_inputs(cfg, weights, feeds, i, device)

  def step(inp, c, hs, sm):
    h_in = RT.gnn_dense(hs, sm, mask) if cfg.use_gnn else hs
    return RT.convlstm_cell(RT.grid_emb(inp, *sw.emb_class), c, h_in, *sw.dec_class)

  c, hs = step(first, c, hs, sm)                          # time 0: the K beams of a sample are identical
  c, hs, sm = c.repeat_interleave(b, 0), hs.repeat_interleave(b, 0), sm.repeat_interleave(b, 0)
  base = torch.arange(n, device=device)[:, None] * b
  out = []
  for t in range(len(step_ids)):
    out.append(RT.conv2d_same(hs, sw.head_class).reshape(n, b, -1))
    flat = (torch.as_tensor(np.asarray(step_par[t])).to(device).long() + base).reshape(-1)
    c, hs = c[flat], hs[flat]
    if t == len(step_ids) - 1:
      break
    inp = RT.one_hot_map(torch.as_tensor(np.asarray(step_ids[t])).reshape(-1), h, ww, DT, device)
    c, hs = step(inp, c, hs, sm)
  return torch.stack(out).cpu().numpy()


def beam_search(cfg, weights, feeds, i, tp, device):
  """RT.decoder_beam of scale i for tp steps (with graph attention): (trace dict of numpy ids / parents [Tp,N,K] and
  logits [Tp,N,K,V] of every step, margins [Tp,N,3], back-traced (logits [N,K,Tp,V], ids [N,K,Tp], scores [N,K])).
  The margins of a step: the smallest gap between consecutive selected candidates, the gap to the best unselected
  one, and (diverse beam) the smallest gap between consecutive logits among the K + 1 largest of a row the selection
  reads.  The diverse penalty (log gamma x rank in the row) puts |log gamma| between the candidates of one row, so the
  first two stay wide when two cells of a row tie; which of them gets the lower rank, and with it the selection, is
  decided by their logits (an entry of rank K or more is never selected)."""
  assert cfg.use_gnn, "RT.decoder_beam attends at every step"
  sw, first, state, sm, mask = class_inputs(cfg, weights, feeds, i, device)
  margins, trace = [], []
  with torch.no_grad():
    lg, ids, sc = RT.decoder_beam(first, state, tp, cfg.beam_size, sw.dec_class, sw.emb_class, sw.head_class, sm,
                                  mask, cfg.diverse_beam, cfg.diverse_gamma, cfg.fix_num_timestep, margins, trace)
  np_ = lambda t: t.cpu().numpy()
  k = cfg.beam_size
  rank_gap = []
  for time, (_, _, x) in enumerate(trace):
    top = torch.topk(x[:, :1] if time == 0 else x, k + 1, dim=-1).values       # time 1 reads beam 0's row only
    rank_gap.append((top[..., :-1] - top[..., 1:]).amin((-2, -1)) if cfg.diverse_beam else
                    torch.full(top.shape[:1], math.inf, dtype=DT, device=top.device))
  margins = torch.cat([torch.stack(margins), torch.stack(rank_gap)[..., None]], -1)
  tr = dict(ids=np.stack([np_(a) for a, _, _ in trace]), parents=np.stack([np_(p) for _, p, _ in trace]),
            logits=np.stack([np_(x) for _, _, x in trace]))
  return tr, np_(margins), (np_(lg), np_(ids), np_(sc))


def greedy_replay(cfg, weights, feeds, i, ids, device):
  """The greedy class decoder of scale i (RT.decoder_greedy, test.py's) fed one_hot(ids[:, t]) after step t instead of
  its own arg-max: logits [N,Tp,V] along the given ids [N,Tp]."""
  n = cfg.batch_size
  h, ww = cfg.scene_grids[i]
  sw, inp, (c, hs), sm, mask = class_inputs(cfg, weights, feeds, i, device)
  sm = sm if getattr(cfg, "gnn_scene_in_greedy", True) else None
  ids = torch.as_tensor(np.asarray(ids)).to(device).long()
  outs = []
  for t in range(ids.shape[1]):
    h_in = RT.gnn_dense(hs, sm, mask) if cfg.use_gnn else hs
    c, hs = RT.convlstm_cell(RT.grid_emb(inp, *sw.emb_class), c, h_in, *sw.dec_class)
    outs.append(RT.conv2d_same(hs, sw.head_class).reshape(n, -1))
    inp = RT.one_hot_map(ids[:, t], h, ww, DT, device)
  return torch.stack(outs, 1).cpu().numpy()


def reg_truth(cfg, weights, obs_regress, i, tp, device):
  """The regression decoder of scale i (RT.decoder_greedy with onehot=False: its raw 2-channel output fed back) on
  the regression encoder's state of the observed offsets obs_regress [N,T,h,w,2]: offsets [N,Tp,h,w,2].  It does not
  depend on the class decoder's selections."""
  sw = R.scale_weights(_weights(weights, device), i)
  obs = torch.from_numpy(np.asarray(obs_regress)).to(device=device, dtype=DT)
  enc = RT.encoder(obs, sw.enc_reg[0], sw.enc_reg[1], cfg.enc_hidden_size, device)
  reg = RT.decoder_greedy(obs[:, -1], enc, tp, sw.dec_reg, sw.emb_reg, sw.head_reg, None, None, False, False)
  return reg.cpu().numpy()


def backtrace(ids, parents, logits, length):
  """The beam outputs of a per-step trace (ids / parents [T,N,K], logits [T,N,K,V]) as a rollout of `length` steps
  returns them: ids [N,K,length] and logits [N,K,length,V], each beam's row followed back from its slot at the last
  step (RT.decoder_beam's back-trace)."""
  _, n, b = ids.shape[:3]
  out_ids = np.zeros((n, b, length), ids.dtype)
  out_lg = np.zeros((n, b, length) + logits.shape[3:], logits.dtype)
  rows = np.arange(n)[:, None]
  par = np.tile(np.arange(b), (n, 1))
  for t in range(length - 1, -1, -1):
    out_ids[:, :, t] = ids[t][rows, par]
    out_lg[:, :, t] = logits[t][rows, par]
    par = parents[t][rows, par]
  return out_ids, out_lg


def beam_scores(cfg, truth, eng_logits, ids, par, lp_scale):
  """fp64 log-probabilities [K] after the last of T selections of one sample, along its selections ids / par [T,K]:
  sum over the steps after fix_num_timestep of log_softmax(truth[t][parent])[id] + log(gamma) x rank(id in that row).
  truth / eng_logits [T,K,V]: the fp64 replay and the engine's logits.  The rank is the truth's; where the truth puts
  another cell of the row within twice the engine's logit error of the selected one (plus the rounding of fp32
  log-probabilities of magnitude lp_scale), the rank is ambiguous at fp32 and the engine's is taken if it lies in the
  admissible range.  Returns (scores, number of ambiguous ranks, ranks outside the admissible range)."""
  lg = math.log(cfg.diverse_gamma) if cfg.diverse_beam else 0.0
  k = ids.shape[1]
  score = np.zeros(k)
  amb = bad = 0
  for t in range(len(ids)):
    p = par[t] if t > 0 else np.zeros(k, np.int64)          # the first selection reads beam 0's row
    rows, erows = truth[t][p], eng_logits[t][p].astype(np.float64)
    x = rows[np.arange(k), ids[t]][:, None]
    tol = 2 * np.abs(eng_logits[t] - truth[t]).max() + 2.5e-7 * (lp_scale + 30.0)
    r_lo, r_hi = (rows > x + tol).sum(-1), (rows >= x - tol).sum(-1) - 1
    ex = erows[np.arange(k), ids[t]][:, None]
    cols = np.arange(rows.shape[1])[None]
    r_eng = ((erows > ex) | ((erows == ex) & (cols < ids[t][:, None]))).sum(-1)
    amb += int((r_lo != r_hi).sum())
    bad += int(((r_eng < r_lo) | (r_eng > r_hi)).sum())
    rank = np.where(r_lo == r_hi, r_lo, np.clip(r_eng, r_lo, r_hi))
    m = rows.max(-1)
    lsm = rows[np.arange(k), ids[t]] - m - np.log(np.exp(rows - m[:, None]).sum(-1))
    new = score[p] + lsm + lg * rank
    score = np.zeros(k) if t + 1 <= cfg.fix_num_timestep else new
  return score, amb, bad
