# coding=utf-8
"""--emb_size: the configurations the drop-in accepts (every multiple of 8 from 8 to 256, with and without
--use_scene_enc) and the ones it refuses before any kernel runs; the f16f8 operand layout of wide x blocks; the fp64
oracle against the executed reference at wide emb sizes (tests/golden/make_golden_emb_size.py)."""
import os

import numpy as np
import pytest
import torch

import emb_size_cases as EC
from multiverse_b200 import ops, synthetic
from multiverse_b200.pred_models import _engine_config


@pytest.mark.parametrize("scene_enc", [True, False])
@pytest.mark.parametrize("emb", [8, 32, 64, 96, 128, 256])
def test_engine_config_accepts_emb_size(emb, scene_enc):
  cfg = synthetic.make_config(emb_size=emb, use_scene_enc=scene_enc)
  assert _engine_config(cfg).emb_size == emb
  assert ops.cell_cpad(emb) == (emb + 31) // 32 * 32 + 256


@pytest.mark.parametrize("emb", [12, 264, 0])
def test_engine_config_refuses_emb_size(emb):
  with pytest.raises(NotImplementedError, match="--emb_size"):
    _engine_config(synthetic.make_config(emb_size=emb))


def f8_off(c, p, cpad):
  """Byte offset of channel c, e4m3 plane p inside an fp8 row (mvb_common.cuh f8_off), written from its rule."""
  cxp = cpad - 256
  if c >= cxp:
    cc = c - cxp
    return 2 * cxp + cc // 64 * 128 + p * 64 + cc % 64
  c0 = c // 64 * 64
  return 2 * c0 + p * min(64, cxp - c0) + c % 64


@pytest.mark.parametrize("cpad", [288, 320, 352, 384, 416, 512])
def test_f16f8_layout(cpad):
  """Both planes of every 64-channel chunk (and of a trailing 32-channel x chunk) lie in one 128-byte (64-byte) run,
  the row is a permutation of its 2 * cpad bytes, x blocks of up to 64 channels keep [e0 (cxp) | e1 (cxp)], and
  ops.operand_values reads that layout back."""
  cxp = cpad - 256
  offs = [f8_off(c, p, cpad) for c in range(cpad) for p in range(2)]
  assert sorted(offs) == list(range(2 * cpad))
  if cxp <= 64:
    assert all(f8_off(c, p, cpad) == p * cxp + c for c in range(cxp) for p in range(2))
  for c in range(0, cpad, 32):
    run = f8_off(c, 0, cpad) // 64
    assert f8_off(c + 31, 1, cpad) // 64 in (run, run + 1)
  # operand_values on a CPU buffer whose e1 bytes hold channel-coded values
  rows = 3
  xh = torch.zeros((2, rows, cpad), dtype=torch.bfloat16)
  xh.mvb_planes = ops.PLANES_F16F8
  raw = xh.view(torch.uint8).reshape(-1)
  f8 = raw[2 * rows * cpad:].view(rows, 2 * cpad)
  code = torch.tensor(np.float32(1.0)).to(torch.float8_e4m3fn).view(torch.uint8)
  for c in range(cpad):
    f8[:, f8_off(c, 1, cpad)] = code if c % 3 == 0 else 0
  vals, e0 = ops.operand_values(xh)
  want = torch.tensor([1.0 / 4096 if c % 3 == 0 else 0.0 for c in range(cpad)])
  assert torch.equal(vals, want.expand(rows, cpad)) and float(e0.abs().max()) == 0.0


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-12


def golden_inputs(over, seed):
  import cases
  from oracle import multiverse_ref as R
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  return cfg, w, f, cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"])


@pytest.mark.parametrize("name", sorted(EC.ROLLOUTS))
def test_truth_equals_reference_execution(name):
  """The fp64 oracle (oracle/multiverse_ref.py; tests/no_scene_enc_ref.py without scene encoding) reproduces the
  executed reference at wide emb sizes (tests/golden/rollout_emb_*.npz) to 1e-12, beam ids identical."""
  import cases
  import no_scene_enc_ref as NS
  from oracle import multiverse_ref as R
  cfg, w, f, ck = golden_inputs(*EC.ROLLOUTS[name])
  g = np.load(os.path.join(GOLD, "rollout_emb_%s.npz" % name))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  ref = R.forward(cfg, w, f, np.float64) if cfg.use_scene_enc else NS.forward(cfg, w, f, np.float64)
  for i in range(len(cfg.scene_grids)):
    if not cfg.use_grids[i]:
      continue
    for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
      kk = "%s_%d" % (k, i)
      assert abs(np.abs(ref[k][i]).max() - g[kk + "_absmax"]) <= TOL * g[kk + "_absmax"], kk
      assert np.abs(cases.sample(ref[k][i]) - g[kk]).max() <= TOL * g[kk + "_absmax"], kk
  if cfg.use_beam_search:
    lg, ids, lp = ref["beam_outputs"]
    assert np.array_equal(ids, g["beam_ids"])
    assert np.abs(cases.sample(lg) - g["beam_logits"]).max() <= TOL * g["beam_logits_absmax"]
    assert np.abs(lp - g["beam_logprobs"]).max() < 1e-11


@pytest.mark.parametrize("name", sorted(EC.TRAIN))
def test_truth_equals_reference_training_step(name):
  """The fp64 autograd truth reproduces the reference Model + Trainer step's losses and clipped gradients."""
  import cases
  import no_scene_enc_ref as NS
  from oracle import multiverse_ref_torch as RT
  over, seed = EC.TRAIN[name]
  cfg, w, f, ck = golden_inputs(dict(over, **{k: v for k, v in EC.TRAIN_ARGS.items() if k != "optimizer"}), seed)
  g = np.load(os.path.join(GOLD, "refexec_train_emb_%s.npz" % name))
  assert str(g["source"]) == "reference_exec" and abs(float(g["checksum"]) - ck) < 1e-6
  tot, losses, wd, grads = (RT.loss_and_grads if cfg.use_scene_enc else NS.loss_and_grads)(cfg, w, f)
  assert abs(tot - float(g["loss"])) <= TOL * abs(tot) and abs(wd - float(g["wd_loss"])) <= TOL * wd
  assert np.abs(np.array(losses) - g["pred_grid_loss"]).max() <= TOL * max(losses)
  assert set(g["variables"]) == set(grads)
  for k, gr in grads.items():
    bar = TOL * max(float(g["grad_absmax/" + k]), 1e-30)
    assert np.abs(cases.sample(np.clip(gr, -10, 10), cases.NATIVE_TRAIN_SAMPLE) - g["grad/" + k]).max() <= bar, k
