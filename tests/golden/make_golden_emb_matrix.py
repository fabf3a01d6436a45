# coding=utf-8
"""Goldens of the --emb_size matrix at embedding widths that are not a multiple of 32 (tests/emb_matrix_cases.py):
the unmodified reference code/pred_models.py executed on the eager TF-1.15 stand-in of oracle/tf1_eager, with the
checks and layouts of make_golden_emb_size.py (the fp64 oracle reproduces the execution to 1e-12 before anything is
written).

  rollout_emb_<case>.npz   per ROLLOUTS case;
  refexec_train_emb_<case>.npz   per TRAIN case.

    python tests/golden/make_golden_emb_matrix.py [name ...]   (needs the reference repository; MVB_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emb_matrix_cases as EM  # noqa: E402
import make_golden_emb_size as ES  # noqa: E402

ES.EC = EM          # make_golden_emb_size's golden() / train_golden() on this file's cases


def main(only=None):
  want = lambda name: not only or name in only
  assert ES.X.available(), "the reference repository is needed to make these goldens"
  for name in EM.ROLLOUTS:
    if want(name):
      path = os.path.join(ES.OUT, "rollout_emb_%s.npz" % name)
      np.savez_compressed(path, **ES.golden(name))
      print("wrote", path, os.path.getsize(path), "bytes", flush=True)
  for name in EM.TRAIN:
    if want("train_" + name):
      path = os.path.join(ES.OUT, "refexec_train_emb_%s.npz" % name)
      np.savez_compressed(path, **ES.train_golden(name))
      print("wrote", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
  main(sys.argv[1:])
