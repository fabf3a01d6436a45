# coding=utf-8
"""SURVEY.md section 8 row f-4, the pin: SimAug's multi-view augmentation as EXECUTED FROM THE REFERENCE'S OWN FILE
(the unmodified SimAug/code/pred_models.py of the reference repository on the eager TF-1.15 stand-in,
oracle/tf1_eager/run_simaug.py), stored in tests/golden/simaug_multiview.npz and tests/golden/refexec_attack.npz,
against the same pipeline written on the oracle (oracle/multiverse_ref_torch.py: autograd input gradient, per-view
losses, selection, mixup, mixed-label objective) - the expectation the GPU tests of multiverse_b200/simaug.py and
TrainEngine's mixup path are held to."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle import multiverse_ref_torch as RT  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "simaug_multiview.npz")
ATTACK = os.path.join(ROOT, "tests", "golden", "refexec_attack.npz")


def oracle_pipeline(exp):
  """multiview_augmentation + the training objective on its output, on the oracle.  Returns what the reference run
  returns."""
  cfg, w, f, extra, spec = cases.simaug_case()
  n, m, eps = spec["n"], spec["m"], spec["eps"]
  t_obs, tp = cfg.obs_len, cfg.pred_len
  tile = lambda a: np.repeat(np.asarray(a), m, axis=0)
  clean = f["scene_feat"].astype(np.float64)[f["obs_scene"]]                  # [N,T,SH,SW,SC]
  tf_ = dict(scene_feat=tile(clean).reshape((n * m * t_obs,) + clean.shape[2:]),
             obs_scene=np.arange(n * m * t_obs, dtype=np.int32).reshape(n * m, t_obs))
  for key in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    tf_[key] = [None if a is None else tile(a) for a in f[key]]
  target = extra["grid_pred_labels_extra"][1].reshape(n * m, tp)
  rcfg_t = R.default_config(**dict(spec["config"], batch_size=n * m))
  g, loss = RT.scene_input_grad(rcfg_t, w, tf_, target, 1, per_sample=True)
  loss = loss.reshape(n, m)
  x = tf_["scene_feat"]
  adv = np.minimum(np.maximum(x - eps * np.sign(g), np.clip(x - eps, -1, 1)), np.clip(x + eps, -1, 1))
  adv = adv.reshape((n, m, t_obs) + clean.shape[2:])
  order = np.argsort(-loss, axis=1, kind="stable")
  rows = np.arange(n)
  beta = max(spec["beta_draw"], 1 - spec["beta_draw"])
  res = dict(beta=beta)
  if exp == 1:
    f1, f2 = adv[rows, order[:, 0]], adv[rows, order[:, 1]]
  elif exp == 4:
    f1, f2 = adv[rows, order[:, m - 1]], adv[rows, order[:, m - 2]]
  else:
    f1 = adv[rows, order[:, 0]]
    f2 = f["scene_feat"].astype(np.float64)[extra["obs_scene_extra"][rows, order[:, 0]]]
    res["selected"] = order[:, 0]
    res["focal"] = (1.0 - np.exp(-np.sort(loss, axis=1)[:, -1])) ** 2.0
  final = (f1 * beta + f2 * (1 - beta)).reshape((n * t_obs,) + clean.shape[2:])
  res["adv_final"] = final
  # the training tower on the augmented features (one private frame per (sample, step) row)
  ft = dict(f, scene_feat=final, obs_scene=np.arange(n * t_obs, dtype=np.int32).reshape(n, t_obs))
  if exp == 3:
    sel = res["selected"]
    ft["mixup"] = dict(beta=beta, obs_labels2=[None, extra["grid_obs_labels_extra"][1][rows, sel]],
                       pred_labels2=[None, extra["grid_pred_labels_extra"][1][rows, sel]], focal=res["focal"])
  rcfg = R.default_config(**spec["config"])
  _, losses, _, grads = RT.loss_and_grads(rcfg, w, ft)
  res["losses"], res["grads"] = losses, grads
  return res


@pytest.mark.parametrize("exp", [1, 4, 3])
def test_reference_execution_matches_golden_and_oracle_pipeline(exp):
  """The oracle's pipeline against the reference execution's augmented features (a strided fp32 sample), mixing
  weight, losses and - experiment 3 - selected views, focal weights and every variable gradient (sampled)."""
  cfg, w, f, extra, spec = cases.simaug_case()
  g = np.load(GOLD)
  assert str(g["source"]).startswith("reference_exec")
  o = oracle_pipeline(exp)
  assert abs(o["beta"] - float(g["exp%d_beta" % exp])) < 1e-12
  d = np.abs(o["adv_final"].reshape(-1)[::cases.ADV_SAMPLE_STRIDE] - g["exp%d_adv_final_sample" % exp])
  # fp64 both, stored as fp32: the sign of an input-gradient entry that is ~0 is the only thing that may differ
  assert (d <= 1e-6).mean() > 0.9999 and d.max() <= 2 * spec["eps"] + 1e-6
  ref_losses = g["exp%d_losses" % exp]
  assert np.abs(np.array(o["losses"]) - ref_losses).max() < 1e-6 * ref_losses.max()
  if exp == 3:
    assert np.array_equal(o["selected"], g["exp3_selected"])
    assert np.abs(o["focal"] - g["exp3_focal"]).max() < 1e-9
    worst = 0.0
    for k, og in o["grads"].items():
      scale = max(float(g["exp3_grad_norms/" + k][2]), 1e-30)          # max |gradient| of the reference run
      samp = np.asarray(og, np.float64).reshape(-1)[::cases.grad_sample_stride(og.size)]
      err = np.abs(samp - g["exp3_grad_sample/" + k]).max() / scale
      worst = max(worst, err)
      assert err <= 1e-6, k
    print("exp 3: oracle vs reference-exec gradients, worst relative error %.2e over %d variables" % (worst, len(o["grads"])))


@pytest.mark.parametrize("mode", ["fgsm", "pgd_mixup"])
def test_white_box_attack_reference_execution_matches_oracle_pipeline(mode):
  """white_box_attack (SimAug/code/pred_models.py:60-170) as executed from the reference file - targeted FGSM, and PGD
  (tf.while_loop, 3 iterations, bounds around the clean input) followed by the mixup with the clean input - against
  the same update rule driven by the oracle's autograd input gradient: what multiverse_b200/simaug.py::
  white_box_attack and mvb_adv_step / mvb_mix implement (GPU: test_simaug_scene_input_gradient_and_attack)."""
  cfg, w, f, extra, spec = cases.simaug_case()
  rcfg = R.default_config(**spec["config"])
  n, eps = spec["n"], spec["eps"]
  off, step, iters, beta = cases.attack_spec(mode, spec, cfg)
  ref = np.load(ATTACK)
  assert str(ref["source"]).startswith("reference_exec")
  hw = 18 * 9
  target = (f["grid_pred_labels"][1].astype(np.int64) + off) % hw                       # create_random_target
  assert np.array_equal(ref[mode + "/target_label"], target) and not (target == f["grid_pred_labels"][1]).any()
  # the oracle's pipeline: one private frame per (sample, step) row, like the reference's [N*T,SH,SW,SC] input
  t_obs = cfg.obs_len
  x = f["scene_feat"].astype(np.float64)[f["obs_scene"]].reshape((n * t_obs,) + f["scene_feat"].shape[1:])
  rows = dict(f, obs_scene=np.arange(n * t_obs, dtype=np.int32).reshape(n, t_obs))
  lo, hi = np.clip(x - eps, -1, 1), np.clip(x + eps, -1, 1)
  adv = x.copy()
  for _ in range(iters):
    gr = RT.scene_input_grad(rcfg, w, dict(rows, scene_feat=adv), target, 1)
    adv = np.minimum(np.maximum(adv - step * np.sign(gr), lo), hi)
  if beta is not None:
    adv = x * beta + adv * (1 - beta)
  d = np.abs(cases.sample(adv) - ref[mode + "/adv_final"])
  print("white_box_attack %s: %.6f of the sampled pixels equal, max diff %.3g" % (mode, (d <= 1e-9).mean(), d.max()))
  assert (d <= 1e-9).mean() > 0.9999 and d.max() <= 2 * eps + 1e-9
  # and the training tower on the attacked features
  _, losses, _, _ = RT.loss_and_grads(rcfg, w, dict(rows, scene_feat=adv))
  assert np.abs(np.array(losses) - ref[mode + "/losses"]).max() < 1e-9 * ref[mode + "/losses"].max()
