# coding=utf-8
"""Golden output of the reference's single-future evaluation: `pred_utils.evaluate` and `Dataset.get_batches` of both
code/ and SimAug/code/, imported unmodified (their `tensorflow` the drop-in shim), fed by a stub tester that replays
stored decode outputs batch by batch.

The set: 23 trajectories (batches of 5: the last one is padded), scene 12x16 -> grids 6x8 and 3x4, obs 8 / pred 12,
float32 trajectories, ActEV-style keys over the five scenes (0500 only twice), one ground-truth class of -1 (numpy
indexing wraps it).  Cases (single_future_eval_cases): greedy on two scales; beam search (K=3) with use_grids 0,1 (no
seq_ids / obs_list / pred_gt_list: they are written only for j == 0); --use_gt_grid; --per_scene_eval; SimAug with
only_scene 0400, keys in seq_key only, --per_scene_eval (scenes without rows give 0.0); logits with exact ties (the first
maximum wins).  Stored per case: the outputs replayed, the batches get_batches yielded, and the returned dict and the
save_output pickle (pickled, as uint8).

  python tests/golden/make_golden_single_future_eval.py        (needs the reference tree)"""
import importlib.util
import os
import pickle
import sys
import tempfile

import numpy as np

ROOT = os.environ.get("MVB_REFERENCE_ROOT", "/root/reference")
OUT = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(OUT))


def load_pred_utils(code_dir, name):
  spec = importlib.util.spec_from_file_location(name, os.path.join(code_dir, "pred_utils.py"))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


def main():
  sys.path.insert(0, os.path.join(REPO, "multiverse_b200", "dropin"))     # the `tensorflow` shim
  sys.path.insert(0, os.path.dirname(OUT))
  import single_future_eval_cases as C
  mods = {False: load_pred_utils(os.path.join(ROOT, "code"), "_ref_pred_utils"),
          True: load_pred_utils(os.path.join(ROOT, "SimAug", "code"), "_ref_simaug_pred_utils")}
  base = C.make_set()
  store = dict(("set/" + k, v) for k, v in base.items())
  with tempfile.TemporaryDirectory() as tmp:
    for name in C.CASES:
      cfg, simaug = C.case_config(name, os.path.join(tmp, name + ".p"))
      data, shared = C.case_data(base, simaug)
      pu = mods[simaug]
      ds = pu.Dataset(data, "test", shared=shared, config=cfg)
      outs = C.case_outputs(name, cfg, ds.num_examples)
      C.store_outputs(store, name, outs)
      batches = list(ds.get_batches(cfg.batch_size, full=True, shuffle=False))
      it = iter(outs)

      class Tester(object):
        def step(self, sess, evalbatch):
          return next(it)

      p = pu.evaluate(ds, cfg, None, Tester())
      store[name + "/p"] = np.frombuffer(pickle.dumps(p), np.uint8)
      if cfg.save_output is not None:
        with open(cfg.save_output, "rb") as f:
          store[name + "/out_data"] = np.frombuffer(f.read(), np.uint8)
      for b, (idxs, batch) in enumerate(batches):
        store["%s/batch%d/idxs" % (name, b)] = np.array(idxs)
        store["%s/batch%d/original_batch_size" % (name, b)] = np.array(batch.data["original_batch_size"])
        store["%s/batch%d/batch_obs_scene" % (name, b)] = batch.data["batch_obs_scene"]
        store["%s/batch%d/batch_scene_feat" % (name, b)] = batch.data["batch_scene_feat"]
      print(name, p)
  np.savez_compressed(os.path.join(OUT, "single_future_eval.npz"), **store)


if __name__ == "__main__":
  main()
