# coding=utf-8
"""Golden vectors of the reference's own training step under the options of code/train.py:85-92, EXECUTED: the
unmodified code/pred_models.py (Model + Trainer) on the eager TF-1.15 stand-in (oracle/tf1_eager), and its
get_feed_dict's soft label maps.  tests/test_train_options_cpu.py holds tests/train_options_ref.py to them.

  refexec_train_<case>.npz   losses, the clipped gradient of every trainable variable and the variables after one
                             Adadelta train_op (strided samples of at most SAMPLE elements per array)
  refexec_soft_labels.npz    the grid_pred_labels_T feeds of get_feed_dict(is_train=True) for soft_grid 1-7

  python tests/golden/make_golden_train_options.py     (needs the reference repository; MVB_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import multiverse_ref as R  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SAMPLE = 1536            # every golden file stays well under 1 MB
SEED = 10
OVER = dict(batch_size=2, use_grids=[False, True], grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001)
# case -> (soft_grid (0: sparse labels), mask_grid_regression, train_w_onehot)
CASES = {
    "soft4": (4, False, True),
    "soft7_mask": (7, True, True),
    "sparse_mask": (0, True, True),
    "logits_fed": (0, False, False),
    "logits_fed_soft1_mask": (1, True, False),
}


def sample(a):
  flat = np.asarray(a, np.float64).reshape(-1)
  return flat[::max(1, -(-flat.size // SAMPLE))]


def edge_labels(cfg, f):
  """Prediction labels in the corners and on the edges of every used grid (the soft maps are clipped there)."""
  for i, (h, w) in enumerate(cfg.scene_grids):
    cells = [0, w - 1, (h - 1) * w, h * w - 1, w // 2, (h // 2) * w, (h // 2) * w + w - 1, (h - 1) * w + w // 2]
    lab = np.array(f["grid_pred_labels"][i])
    lab[0, :len(cells)] = cells
    lab[1, :len(cells)] = cells[::-1]
    f["grid_pred_labels"][i] = lab
  return f


def soft_maps_reference(cls, h, w, mode):
  """The reference's get_feed_dict loop (code/pred_models.py:1085-1136), verbatim in effect: one ndimage.convolve
  per (sample, step)."""
  from scipy import ndimage
  kern = {1: (0.1, 1.0), 2: (0.01, 1.0), 3: (0.05, 1.0), 4: (0.0125, 0.9), 5: (0.05, 0.6), 6: (0.1, 0.2)}
  if mode == 7:
    k = np.full((5, 5), 0.0625)
    k[1:4, 1:4] = 0.0125
    k[2, 2] = 0.8
  else:
    k = np.full((3, 3), kern[mode][0])
    k[1, 1] = kern[mode][1]
  out = np.zeros(cls.shape + (h, w, 1))
  for n in range(cls.shape[0]):
    for t in range(cls.shape[1]):
      m = np.zeros((h * w,))
      m[cls[n, t]] = 1.0
      out[n, t, :, :, 0] = ndimage.convolve(m.reshape(h, w), k, mode="constant", cval=0.0)
  return out


def case_inputs(name):
  """(cfg, weights, feeds) of a case; the feeds' labels are the soft maps for a soft case."""
  mode = CASES[name][0]
  cfg = R.default_config(**OVER)
  w, f = R.make_weights(cfg, SEED), edge_labels(cfg, R.make_inputs(cfg, SEED))
  if mode:
    f["grid_pred_labels"] = [soft_maps_reference(np.asarray(a), h, ww, mode)      # every scale's placeholder is a map
                             for a, (h, ww) in zip(f["grid_pred_labels"], cfg.scene_grids)]
  return cfg, w, f


def train_golden(name):
  mode, mask, onehot = CASES[name]
  cfg, w, f = case_inputs(name)
  got = X.train_step(cfg, w, f, grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001,
                     use_soft_grid_class=bool(mode), soft_grid=mode, mask_grid_regression=mask, train_w_onehot=onehot)
  g = dict(loss=np.float64(got["loss"]), wd_loss=np.float64(got["wd_loss"]),
           pred_grid_loss=np.asarray(got["pred_grid_loss"], np.float64), variables=np.array(sorted(got["grads"])))
  for k in got["grads"]:
    g["grad/" + k] = sample(got["grads"][k])
    g["grad_absmax/" + k] = np.float64(np.abs(got["grads"][k]).max())
    g["updated/" + k] = sample(got["updated"][k])
  return g


def soft_label_golden():
  """get_feed_dict(is_train=True) of the reference Model, executed on the drop-in Model (as make_golden_refexec's
  feed goldens), for every soft_grid mode on a batch of synthetic trajectories read by the reference's pred_utils."""
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
  g = {}
  for mode in range(1, 8):
    tf.reset_default_graph()
    tmp = tempfile.mkdtemp()
    args, cfg = T.make_args(tmp)
    args.prepropath, args.use_soft_grid_class, args.soft_grid = tmp, True, mode
    synthetic.write_npz(os.path.join(tmp, "data_test.npz"), cfg, 3, seed=5)
    data = pred_utils.read_data(args, "test")
    model = pm.get_model(args, gpuid=0)
    _, batch = next(iter(data.get_batches(args.batch_size, full=True, shuffle=False)))
    theirs = ref.Model.get_feed_dict(model, batch, is_train=True)
    for j, _ in enumerate(cfg.scene_grids):
      g["mode%d/pred_grid_class/%d" % (mode, j)] = np.stack([np.asarray(a)[j] for a in batch.data["pred_grid_class"]])
      g["mode%d/labels/%d" % (mode, j)] = np.asarray(theirs[model.grid_pred_labels_T[j]])
  return g


def main():
  assert X.available(), "the reference repository is needed to make these goldens"
  for name in CASES:
    path = os.path.join(GOLD, "refexec_train_%s.npz" % name)
    np.savez_compressed(path, source=np.array("reference_exec"), **train_golden(name))
    print(path, os.path.getsize(path), "bytes")
  path = os.path.join(GOLD, "refexec_soft_labels.npz")
  np.savez_compressed(path, source=np.array("reference_exec"), **soft_label_golden())
  print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
