# coding=utf-8
"""Goldens of models built with --emb_size above 64 (tests/emb_size_cases.py): the unmodified reference
code/pred_models.py executed on the eager TF-1.15 stand-in of oracle/tf1_eager.  Before writing, the script asserts
that the fp64 oracle (oracle/multiverse_ref.py with scene encoding, tests/no_scene_enc_ref.py without) reproduces that
execution to 1e-12 with identical ids, and for the training steps that the fp64 autograd truth
(oracle/multiverse_ref_torch.py / tests/no_scene_enc_ref.py) reproduces the reference's loss and clipped gradients.

  rollout_emb_<case>.npz   per ROLLOUTS case, in the layout of make_golden_ablation.py;
  refexec_train_emb_<case>.npz   per TRAIN case, in the layout of make_golden_no_scene_enc.py's training golden.

    python tests/golden/make_golden_emb_size.py [name ...]   (needs the reference repository; MVB_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cases  # noqa: E402
import emb_size_cases as EC  # noqa: E402
import make_golden_ablation as A  # noqa: E402
import make_golden_no_scene_enc as G  # noqa: E402
import no_scene_enc_ref as NS  # noqa: E402
from multiverse_b200 import synthetic  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle import multiverse_ref_torch as RT  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def inputs(over, seed):
  """(config, weights, feeds, checksum): weights under the variables the model declares (synthetic.weight_shapes)."""
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  return cfg, w, f, cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"])


def truth(cfg, w, f):
  return R.forward(cfg, w, f, np.float64) if cfg.use_scene_enc else NS.forward(cfg, w, f, np.float64)


def golden(name):
  cfg, w, f, ck = inputs(*EC.ROLLOUTS[name])
  x = X.forward(cfg, w, f) if cfg.use_scene_enc else G.reference_forward(cfg, w, f)
  r = truth(cfg, w, f)
  g = dict(source=np.array("reference_exec"), variables=np.array(sorted(x["variables"])), checksum=ck)
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
      g["beam_margins"] = A.beam_margins(cfg, w, f, i)
  if cfg.use_beam_search:
    lg, ids, lp = x["beam_outputs"]
    assert np.array_equal(ids, r["beam_outputs"][1]), name
    assert np.abs(lg - r["beam_outputs"][0]).max() <= 1e-12 * np.abs(lg).max(), name
    assert np.abs(lp - r["beam_outputs"][2]).max() < 1e-11, name
    g.update(beam_ids=ids, beam_logprobs=lp, beam_logits=cases.sample(lg),
             beam_logits_absmax=np.float64(np.abs(lg).max()), beam_logits_top3=lg[:, :3].astype(np.float32))
  return g


def train_truth(cfg, w, f):
  """(total, losses, wd, grads) of the fp64 autograd truth."""
  if cfg.use_scene_enc:
    return RT.loss_and_grads(cfg, w, f)
  return NS.loss_and_grads(cfg, w, f)


def train_golden(name):
  over, seed = EC.TRAIN[name]
  cfg, w, f, ck = inputs(dict(over, **{k: v for k, v in EC.TRAIN_ARGS.items() if k != "optimizer"}), seed)
  got = X.train_step(cfg, w, f, train_w_onehot=True, **EC.TRAIN_ARGS)
  tot, losses, wd, grads = train_truth(cfg, w, f)
  assert abs(tot - got["loss"]) <= 1e-12 * abs(tot) and abs(wd - got["wd_loss"]) <= 1e-12 * wd, name
  assert np.abs(np.array(losses) - got["pred_grid_loss"]).max() <= 1e-12 * max(losses), name
  assert set(got["grads"]) == set(grads) == set(w), name
  for k, gr in grads.items():
    gc = np.clip(gr, -10.0, 10.0)        # element-wise clip of the Trainer (:1700-1705)
    assert np.abs(gc - got["grads"][k]).max() <= 1e-12 * max(np.abs(gc).max(), 1e-30), (name, k)
  g = dict(source=np.array("reference_exec"), loss=np.float64(got["loss"]), wd_loss=np.float64(got["wd_loss"]),
           pred_grid_loss=np.asarray(got["pred_grid_loss"], np.float64), global_step=np.int64(got["global_step"]),
           variables=np.array(sorted(got["grads"])), checksum=ck)
  for k in got["grads"]:
    g["grad/" + k] = cases.sample(got["grads"][k], cases.NATIVE_TRAIN_SAMPLE)
    g["grad_absmax/" + k] = np.float64(np.abs(got["grads"][k]).max())
    g["updated/" + k] = cases.sample(got["updated"][k], cases.NATIVE_TRAIN_SAMPLE)
  return g


def main(only=None):
  want = lambda name: not only or name in only
  assert X.available(), "the reference repository is needed to make these goldens"
  for name in EC.ROLLOUTS:
    if want(name):
      path = os.path.join(OUT, "rollout_emb_%s.npz" % name)
      np.savez_compressed(path, **golden(name))
      print("wrote", path, os.path.getsize(path), "bytes", flush=True)
  for name in EC.TRAIN:
    if want("train_" + name):
      path = os.path.join(OUT, "refexec_train_emb_%s.npz" % name)
      np.savez_compressed(path, **train_golden(name))
      print("wrote", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
  main(sys.argv[1:])
