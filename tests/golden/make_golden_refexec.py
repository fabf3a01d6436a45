# coding=utf-8
"""Golden vectors of the reference's own graph code, EXECUTED: the unmodified code/pred_models.py and
SimAug/code/pred_models.py of the reference repository on the eager TF-1.15 stand-in (oracle/tf1_eager).  The tests
regenerate the inputs from the seeds in cases.REFEXEC_* and hold the oracle to these outputs
(tests/test_reference_exec_cpu.py, tests/test_simaug_reference_cpu.py).  Large arrays are stored as a strided sample
(cases.sample); everything is fp64 except where a test's bar allows fp32.

  python tests/golden/make_golden_refexec.py          (needs the reference repository; MVB_REFERENCE_ROOT)
  python tests/golden/make_golden_refexec.py native   (refexec_native.npz alone)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402
from oracle.tf1_eager import run_simaug as RS  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def forward_golden(name):
  over, seed = cases.REFEXEC_FORWARD[name]
  cfg = R.default_config(**over)
  out = X.forward(cfg, R.make_weights(cfg, seed), R.make_inputs(cfg, seed))
  g = dict(variables=np.array(sorted(out["variables"])))
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      continue
    for key in ("grid_pred_decoded", "grid_pred_reg_decoded", "scene_convs"):
      g["%s_%d" % (key, i)] = cases.sample(out[key][i])
      g["%s_%d_absmax" % (key, i)] = np.float64(np.abs(out[key][i]).max())
  if cfg.use_beam_search:
    lg, ids, lp = out["beam_outputs"]
    g.update(beam_logits=cases.sample(lg), beam_logits_absmax=np.float64(np.abs(lg).max()), beam_ids=ids,
             beam_logprobs=lp)
  return g


def train_golden():
  over, seed, kw = cases.REFEXEC_TRAIN
  cfg = R.default_config(**over)
  w, f = R.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  got = X.train_step(cfg, w, f, **kw)
  g = dict(loss=np.float64(got["loss"]), wd_loss=np.float64(got["wd_loss"]),
           pred_grid_loss=np.asarray(got["pred_grid_loss"], np.float64), global_step=np.int64(got["global_step"]),
           variables=np.array(sorted(got["grads"])))
  for k in got["grads"]:
    g["grad/" + k] = cases.sample(got["grads"][k])
    g["grad_absmax/" + k] = np.float64(np.abs(got["grads"][k]).max())
    g["updated/" + k] = cases.sample(got["updated"][k])
  return g


def native_golden():
  """refexec_native.npz: the published configuration (cases.REFEXEC_NATIVE: scene 36x64, grids 18x32 and 9x16):
  the greedy two-scale forward (forward/...) and one training step with Trainer's Adadelta at init_lr 0.3
  (train/...; per-variable samples of at most cases.NATIVE_TRAIN_SAMPLE elements)."""
  cfg, w, f = cases.refexec_native_inputs()
  out = X.forward(cfg, w, f)
  g = {"forward/variables": np.array(sorted(out["variables"]))}
  for i in range(len(cfg.scene_grids)):
    for key in ("grid_pred_decoded", "grid_pred_reg_decoded", "scene_convs"):
      g["forward/%s_%d" % (key, i)] = cases.sample(out[key][i])
      g["forward/%s_%d_absmax" % (key, i)] = np.float64(np.abs(out[key][i]).max())
  got = X.train_step(cfg, w, f, **cases.REFEXEC_NATIVE[2])
  g.update({"train/loss": np.float64(got["loss"]), "train/wd_loss": np.float64(got["wd_loss"]),
            "train/pred_grid_loss": np.asarray(got["pred_grid_loss"], np.float64),
            "train/global_step": np.int64(got["global_step"]), "train/variables": np.array(sorted(got["grads"]))})
  for k in got["grads"]:
    g["train/grad/" + k] = cases.sample(got["grads"][k], cases.NATIVE_TRAIN_SAMPLE)
    g["train/grad_absmax/" + k] = np.float64(np.abs(got["grads"][k]).max())
    g["train/updated/" + k] = cases.sample(got["updated"][k], cases.NATIVE_TRAIN_SAMPLE)
  path = os.path.join(GOLD, "refexec_native.npz")
  np.savez_compressed(path, source=np.array("reference_exec"), **g)
  print("refexec_native.npz", os.path.getsize(path), "bytes")


def attack_golden():
  cfg, w, f, extra, spec = cases.simaug_case()
  rcfg = R.default_config(**spec["config"])
  g = {}
  for mode in ("fgsm", "pgd_mixup"):
    off, step, iters, beta = cases.attack_spec(mode, spec, cfg)
    ref = RS.adversarial(rcfg, w, f, spec["eps"], off, fgsm=(mode == "fgsm"), step_size=step, num_iter=iters,
                         mixup_beta=beta)
    g[mode + "/target_label"] = np.asarray(ref["target_label"], np.int64)
    g[mode + "/adv_final"] = cases.sample(ref["adv_final"])
    g[mode + "/losses"] = np.asarray(ref["losses"], np.float64)
  return g


def _handle_key(h):
  return "%s/%s" % (h.name, "-" if h.index is None else h.index)


def pack_batch(data):
  """batch.data -> flat arrays: lists of per-sample arrays stacked under list/<key>, the rest under arr/<key>."""
  out = {}
  for k, v in data.items():
    out[("list/" if isinstance(v, list) else "arr/") + k] = np.stack(v) if isinstance(v, list) else np.asarray(v)
  return out


def feed_goldens():
  """The reference's Model.get_feed_dict (code/pred_models.py:1042-1194) executed on the drop-in Model for batches
  read by the reference's pred_utils, and SimAug's (SimAug/code/pred_models.py:1457-1560) on a multiview batch:
  the batches and the feed dicts, keyed by placeholder name / index."""
  import importlib.util
  import tempfile
  import test_dropin_cpu as T
  sys.path.insert(0, T.DROPIN)
  import tensorflow as tf
  import pred_models as pm
  from multiverse_b200 import synthetic
  sys.path.insert(0, T.REF)
  spec = importlib.util.spec_from_file_location("ref_pred_models", os.path.join(T.REF, "pred_models.py"))
  ref = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(ref)
  import pred_utils
  out = {}
  for ci, kw in enumerate(cases.FEED_CONFIGS):
    tf.reset_default_graph()
    tmp = tempfile.mkdtemp()
    args, cfg = T.make_args(tmp, **kw)
    args.prepropath = tmp
    synthetic.write_npz(os.path.join(tmp, "data_test.npz"), cfg, 5, seed=3)
    data = pred_utils.read_data(args, "test")
    model = pm.get_model(args, gpuid=0)
    g = {}
    for bi, (_, batch) in enumerate(data.get_batches(args.batch_size, full=True, shuffle=False)):
      g.update(("batch%d/%s" % (bi, k), v) for k, v in pack_batch(batch.data).items())
      g.update(("batch%d/shared/%s" % (bi, k), np.asarray(v)) for k, v in batch.shared.items()
               if k.startswith("grid_center_"))
      for is_train in (False, True):
        theirs = ref.Model.get_feed_dict(model, batch, is_train=is_train)
        g.update(("feed%d_%d/%s" % (bi, is_train, _handle_key(h)), np.asarray(v)) for h, v in theirs.items())
    out["refexec_feed_dict_%d.npz" % ci] = g
  # SimAug's multiview feed dict (the module binds `tf` to the drop-in shim; its get_feed_dict uses only numpy)
  spec = importlib.util.spec_from_file_location("ref_simaug_pred_models",
                                                os.path.join(os.path.dirname(T.REF), "SimAug", "code", "pred_models.py"))
  sref = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(sref)
  tf.reset_default_graph()
  model, batch = T.multiview_case(pm, tempfile.mkdtemp())
  theirs = sref.Model.get_feed_dict(model, batch, is_train=True)
  g = {"feed/" + _handle_key(h): np.asarray(v) for h, v in theirs.items()}
  out["refexec_feed_dict_simaug.npz"] = g
  return out


def main():
  assert X.available() and RS.available(), "the reference repository is needed to make these goldens"
  for f, g in feed_goldens().items():
    np.savez_compressed(os.path.join(GOLD, f), source=np.array("reference_exec"), **g)
    print(f, os.path.getsize(os.path.join(GOLD, f)), "bytes")
  out = {}
  for name in cases.REFEXEC_FORWARD:
    out.update(("%s/%s" % (name, k), v) for k, v in forward_golden(name).items())
  np.savez_compressed(os.path.join(GOLD, "refexec_forward.npz"), source=np.array("reference_exec"), **out)
  np.savez_compressed(os.path.join(GOLD, "refexec_train.npz"), source=np.array("reference_exec"), **train_golden())
  np.savez_compressed(os.path.join(GOLD, "refexec_attack.npz"), source=np.array("reference_exec:SimAug"),
                      **attack_golden())
  for f in ("refexec_forward.npz", "refexec_train.npz", "refexec_attack.npz"):
    print(f, os.path.getsize(os.path.join(GOLD, f)), "bytes")
  native_golden()


if __name__ == "__main__":
  if sys.argv[1:] == ["native"]:
    assert X.available(), "the reference repository is needed to make this golden"
    native_golden()
  else:
    main()
