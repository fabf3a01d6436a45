# coding=utf-8
"""Goldens of models built without --use_scene_enc (tests/no_scene_enc_ref.py): the unmodified reference
code/pred_models.py executed on the eager TF-1.15 stand-in of oracle/tf1_eager with use_scene_enc off.  Before writing,
the script asserts that the fp64 truth of tests/no_scene_enc_ref.py reproduces that execution (1e-12, identical ids).

  rollout_noscene_<case>.npz  per no_scene_enc_ref.ROLLOUTS case, in the layout of make_golden_ablation.py: the
                              variable names and shapes, strided samples of the outputs (CPU pin) and the rollout fields
                              the GPU tests compare against;
  refexec_train_noscene.npz   one Model + Trainer step at no_scene_enc_ref.TRAIN (TRAINING.md's arguments without
                              --use_scene): losses, every clipped gradient and the variables after Adadelta, sampled
                              as refexec_native.npz.

    python tests/golden/make_golden_no_scene_enc.py [name ...]   (needs the reference repository; MVB_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cases  # noqa: E402
import make_golden_ablation as A  # noqa: E402
import no_scene_enc_ref as NS  # noqa: E402
from multiverse_b200 import synthetic  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def inputs(over, seed):
  """(config, weights, feeds) of a case: weights under the variables the model declares (synthetic.weight_shapes),
  feeds of the oracle (the scene frames are fed, and nothing reads them)."""
  cfg = NS.config(**over)
  return cfg, synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)


def checksum(w, f):
  return cases.checksum(*w.values()) + cases.checksum(f["traj"])


def reference_forward(cfg, w, f):
  """run_reference.forward without the scene convolutions (the model has none)."""
  tf, model, _, _ = X.build(cfg, w, f)
  np_ = lambda t: t.numpy() if hasattr(t, "numpy") else t
  assert not hasattr(model, "scene_convs")
  out = dict(grid_pred_decoded=[np_(t) for t in model.grid_pred_decoded],
             grid_pred_reg_decoded=[np_(t) for t in model.grid_pred_reg_decoded], beam_outputs=None,
             variables={v.op.name: tuple(int(d) for d in v.shape) for v in tf.global_variables()})
  if model.beam_outputs is not None:
    out["beam_outputs"] = [np_(t) for t in model.beam_outputs]
  return out


def beam_margins(cfg, w, f, i):
  """([Tp, N, 2] selection margins, per-step trace) of the fp64 beam search on scale i."""
  inter = NS.forward(cfg, w, f, np.float64, return_intermediates=True)["inter"][i]
  sw = R.scale_weights(R.cast_tree(w, np.float64), i)
  *_, tr = R.grid_decoder_beam_search(inter["obs_onehot"][:, -1], inter["enc_state"], cfg.pred_len, cfg.beam_size,
                                      sw.dec_class, sw.emb_class, sw.head_class, scene_mean=None, use_gnn=cfg.use_gnn,
                                      diverse_beam=cfg.diverse_beam, diverse_gamma=cfg.diverse_gamma,
                                      fix_num_timestep=cfg.fix_num_timestep, return_trace=True)
  return A.margins_of(cfg, tr), tr


def golden(name):
  cfg, w, f = inputs(*NS.ROLLOUTS[name])
  x = reference_forward(cfg, w, f)
  r = NS.forward(cfg, w, f, np.float64)
  names = sorted(x["variables"])
  g = dict(source=np.array("reference_exec"), variables=np.array(names),
           variable_shapes=np.array([str(x["variables"][k]) for k in names]), checksum=checksum(w, f))
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
    if cfg.use_beam_search:
      g["beam_margins"] = beam_margins(cfg, w, f, i)[0]
  if cfg.use_beam_search:
    lg, ids, lp = x["beam_outputs"]
    assert np.array_equal(ids, r["beam_outputs"][1]), name
    assert np.abs(lg - r["beam_outputs"][0]).max() <= 1e-12 * np.abs(lg).max(), name
    assert np.abs(lp - r["beam_outputs"][2]).max() < 1e-11, name
    g.update(beam_ids=ids, beam_logprobs=lp, beam_logits=cases.sample(lg),
             beam_logits_absmax=np.float64(np.abs(lg).max()), beam_logits_top3=lg[:, :3].astype(np.float32),
             beam_lg_max=lg.max(-1), beam_lg_mean=lg.mean(-1))
  return g


def train_golden():
  over, seed = NS.TRAIN
  cfg, w, f = inputs(over, seed)
  kw = {k: over[k] for k in ("grid_loss_weight", "grid_reg_loss_weight", "wd", "init_lr", "clip_gradient_norm",
                             "optimizer")}
  got = X.train_step(cfg, w, f, train_w_onehot=True, **kw)
  tot, losses, wd, grads = NS.loss_and_grads(cfg, w, f)
  assert abs(tot - got["loss"]) <= 1e-12 * abs(tot) and abs(wd - got["wd_loss"]) <= 1e-12 * wd
  assert np.abs(np.array(losses) - got["pred_grid_loss"]).max() <= 1e-12 * max(losses)
  assert set(got["grads"]) == set(grads) == set(w)
  for k, gr in grads.items():
    gc = np.clip(gr, -10.0, 10.0)        # element-wise clip of the Trainer (:1700-1705)
    assert np.abs(gc - got["grads"][k]).max() <= 1e-12 * max(np.abs(gc).max(), 1e-30), k
  g = dict(source=np.array("reference_exec"), loss=np.float64(got["loss"]), wd_loss=np.float64(got["wd_loss"]),
           pred_grid_loss=np.asarray(got["pred_grid_loss"], np.float64), global_step=np.int64(got["global_step"]),
           variables=np.array(sorted(got["grads"])), checksum=checksum(w, f))
  for k in got["grads"]:
    g["grad/" + k] = cases.sample(got["grads"][k], cases.NATIVE_TRAIN_SAMPLE)
    g["grad_absmax/" + k] = np.float64(np.abs(got["grads"][k]).max())
    g["updated/" + k] = cases.sample(got["updated"][k], cases.NATIVE_TRAIN_SAMPLE)
  return g


def main(only=None):
  want = lambda name: not only or name in only
  assert X.available(), "the reference repository is needed to make these goldens"
  for name in NS.ROLLOUTS:
    if want(name):
      path = os.path.join(OUT, "rollout_noscene_%s.npz" % name)
      np.savez_compressed(path, **golden(name))
      print("wrote", path, os.path.getsize(path), "bytes", flush=True)
  if want("train"):
    path = os.path.join(OUT, "refexec_train_noscene.npz")
    np.savez_compressed(path, **train_golden())
    print("wrote", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
  main(sys.argv[1:])
