# coding=utf-8
"""Goldens of the beam decoder without graph attention (tests/cases_ablation.py): the unmodified reference
code/pred_models.py executed on the eager TF-1.15 stand-in of oracle/tf1_eager, with use_gnn off.  Before writing, the
script asserts that the oracle (oracle/multiverse_ref.py) reproduces that execution to 1e-12 with identical ids.
Each file holds
  - what the reference execution returned, fp64, for the CPU pin (tests/test_beam_no_gnn_cpu.py): the variable names,
    strided samples (cases.sample) of the class / offset maps and beam logits, the beam ids and log-probabilities;
  - the rollout-golden fields the GPU tests compare against (as tests/golden/make_golden.py writes them);
  - beam_lg_max / beam_lg_mean [N, K, Tp]: per-beam statistics of the beam logits;
  - beam_margins [Tp, N, 2]: per step and sample, the smallest gap between consecutive selected candidates and the gap
    between the K-th selected and the best unselected candidate (how far the selection is from a tie).

The at-size golden (cases_ablation.ROLLOUTS_NO_GNN_ATSIZE, tests/golden/atsize_beam_k20_nognn_n16.npz) holds reduced
statistics of the fp64 numpy oracle alone (about 5 minutes on 8 cores).

    python tests/golden/make_golden_ablation.py [name ...]   (the reference repository is needed for the rollout
                                                              goldens; MVB_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import cases_ablation  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def beam_margins(cfg, w, f, i):
  """[Tp, N, 2] selection margins of the oracle's beam search on scale i."""
  r = R.forward(cfg, w, f, np.float64, return_intermediates=True)
  sw = R.scale_weights(R.cast_tree(w, np.float64), i)
  h, ww = cfg.scene_grids[i]
  obs = R.one_hot(f["grid_obs_labels"][i], h * ww, np.float64).reshape(cfg.batch_size, -1, h, ww, 1)
  inter = r["inter"][i]
  *_, tr = R.grid_decoder_beam_search(obs[:, -1], inter["enc_state"], cfg.pred_len, cfg.beam_size, sw.dec_class,
                                      sw.emb_class, sw.head_class, scene_mean=inter["scene_mean"], use_gnn=cfg.use_gnn,
                                      diverse_beam=cfg.diverse_beam, diverse_gamma=cfg.diverse_gamma,
                                      fix_num_timestep=cfg.fix_num_timestep, return_trace=True)
  return margins_of(cfg, tr)


def margins_of(cfg, tr):
  """[Tp, N, 2] selection margins from the per-step trace of R.grid_decoder_beam_search."""
  n, b = cfg.batch_size, cfg.beam_size
  out = []
  for t, logits in enumerate(tr["logits"]):
    prev = tr["scores"][t - 1] if t else np.zeros((n, b))
    lp = R.log_softmax(logits) + prev[:, :, None]
    if cfg.diverse_beam:
      lp = R.add_div_penalty(lp, cfg.diverse_gamma)
    cand = lp[:, 0] if t == 0 else lp.reshape(n, -1)
    top = -np.sort(-cand, -1)[:, :b + 1]
    out.append(np.stack([(top[:, :-2] - top[:, 1:-1]).min(-1), top[:, -2] - top[:, -1]], -1))
  return np.stack(out)


def golden(name):
  over, seed = cases_ablation.ROLLOUTS_NO_GNN[name]
  cfg = R.default_config(**over)
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  x = X.forward(cfg, w, f)
  r = R.forward(cfg, w, f, np.float64)
  g = dict(source=np.array("reference_exec"), variables=np.array(sorted(x["variables"])),
           checksum=cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"]))
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      continue
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
      assert np.abs(x[k][i] - r[k][i]).max() <= 1e-12 * np.abs(r[k][i]).max(), (name, k, i)
      g["%s_%d" % (k, i)] = cases.sample(x[k][i])
      g["%s_%d_absmax" % (k, i)] = np.float64(np.abs(x[k][i]).max())
    lg = x["grid_pred_decoded"][i]
    g["logits_%d" % i] = lg.astype(np.float32)
    s = np.sort(lg.reshape(lg.shape[0], lg.shape[1], -1), -1)
    g["margin_%d" % i] = s[..., -1] - s[..., -2]
    g["reg_%d" % i] = x["grid_pred_reg_decoded"][i].astype(np.float32)
    g["beam_margins"] = beam_margins(cfg, w, f, i)
  lg, ids, lp = x["beam_outputs"]
  assert np.array_equal(ids, r["beam_outputs"][1]), name
  assert np.abs(lg - r["beam_outputs"][0]).max() <= 1e-12 * np.abs(lg).max(), name
  assert np.abs(lp - r["beam_outputs"][2]).max() < 1e-11, name
  g.update(beam_ids=ids, beam_logprobs=lp, beam_logits=cases.sample(lg), beam_logits_absmax=np.float64(np.abs(lg).max()),
           beam_logits_top3=lg[:, :3].astype(np.float32), beam_lg_max=lg.max(-1), beam_lg_mean=lg.mean(-1))
  return g


def atsize_golden(name):
  """Reduced statistics (cases.rollout_stats) of the fp64 numpy oracle at an at-size shape, plus beam_margins
  [N, Tp, 2] (the layout of tests/golden/atsize_*.npz).  One beam search: the encoders and the offset decoder come from
  a forward of the same model with the greedy class decoder."""
  over, seed = cases_ablation.ROLLOUTS_NO_GNN_ATSIZE[name]
  cfg = R.default_config(**over)
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  i = cfg.use_grids.index(True)
  r = R.forward(R.default_config(**dict(over, use_beam_search=False)), w, f, np.float64, return_intermediates=True)
  sw = R.scale_weights(R.cast_tree(w, np.float64), i)
  h, ww = cfg.scene_grids[i]
  obs = R.one_hot(f["grid_obs_labels"][i], h * ww, np.float64).reshape(cfg.batch_size, -1, h, ww, 1)
  inter = r["inter"][i]
  best, lg, ids, lp, tr = R.grid_decoder_beam_search(
      obs[:, -1], inter["enc_state"], cfg.pred_len, cfg.beam_size, sw.dec_class, sw.emb_class, sw.head_class,
      scene_mean=inter["scene_mean"], use_gnn=cfg.use_gnn, diverse_beam=cfg.diverse_beam,
      diverse_gamma=cfg.diverse_gamma, fix_num_timestep=cfg.fix_num_timestep, return_trace=True)
  res = dict(r, grid_pred_decoded=[best if j == i else d for j, d in enumerate(r["grid_pred_decoded"])],
             beam_outputs=[lg, ids, lp])
  st = cases.rollout_stats(cfg, res)
  st["beam_margins"] = margins_of(cfg, tr).transpose(1, 0, 2)
  st["checksum"] = cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"])
  return st


def main(only=None):
  for name in cases_ablation.ROLLOUTS_NO_GNN_ATSIZE:
    if only and name not in only:
      continue
    path = os.path.join(OUT, "atsize_%s.npz" % name)
    np.savez_compressed(path, **atsize_golden(name))
    print("wrote", path, os.path.getsize(path), "bytes", flush=True)
  assert X.available(), "the reference repository is needed to make these goldens"
  for name in cases_ablation.ROLLOUTS_NO_GNN:
    if only and name not in only:
      continue
    g = golden(name)
    path = os.path.join(OUT, "rollout_%s.npz" % name)
    np.savez_compressed(path, **g)
    print("wrote", path, os.path.getsize(path), "bytes; smallest selection margins (in-beam, boundary): %.1e %.1e"
          % (g["beam_margins"][..., 0].min(), g["beam_margins"][..., 1].min()))


if __name__ == "__main__":
  main(sys.argv[1:])
