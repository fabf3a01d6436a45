# coding=utf-8
"""CPU tests of the single-future evaluation: the NumPy restatement (tests/single_future_eval_ref.py) against what the
reference's own pred_utils.evaluate and Dataset.get_batches returned (tests/golden/single_future_eval.npz), the
generalised multifuture.batch_feeds / split_argv, the data checks and the command-line runner."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

import single_future_eval_cases as C
import single_future_eval_ref as ref
from multiverse_b200 import multifuture, single_future_eval as sfe

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "single_future_eval.npz")


@pytest.fixture(scope="module")
def golden():
  return np.load(GOLDEN)


def case(z, name, tmp_path):
  cfg, simaug = C.case_config(name, str(tmp_path / (name + ".p")))
  data, shared = C.case_data(C.load_set(z), simaug)
  return cfg, simaug, ref.Dataset(data, "test", config=cfg, shared=shared), C.load_outputs(z, name, cfg)


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_get_batches_equals_reference(golden, name, tmp_path):
  cfg, _, ds, _ = case(golden, name, tmp_path)
  batches = list(ds.get_batches(cfg.batch_size, full=True, shuffle=False))
  assert len(batches) == -(-C.R // C.BS) and C.R % C.BS
  for b, (idxs, batch) in enumerate(batches):
    p = "%s/batch%d/" % (name, b)
    assert np.array_equal(np.array(idxs), golden[p + "idxs"])
    assert batch.data["original_batch_size"] == int(golden[p + "original_batch_size"])
    for k in ("batch_obs_scene", "batch_scene_feat"):
      assert batch.data[k].dtype == golden[p + k].dtype and np.array_equal(batch.data[k], golden[p + k])


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_restated_evaluate_equals_reference(golden, name, tmp_path):
  cfg, simaug, ds, outs = case(golden, name, tmp_path)
  it = iter(outs)
  p, out_data = ref.evaluate(ds, cfg, lambda batch: next(it), simaug=simaug)
  ref.assert_same_dict(p, pickle.loads(golden[name + "/p"].tobytes()))
  if cfg.save_output is None:
    assert name + "/out_data" not in golden.files
    return
  want = pickle.loads(golden[name + "/out_data"].tobytes())
  ref.assert_same_out_data(out_data, want)
  with open(cfg.save_output, "rb") as f:
    ref.assert_same_out_data(pickle.load(f), want)
  if name == "beam_grids_0_1":            # written only for j == 0: a model of scale 1 alone writes none
    assert want["seq_ids"] == [] and want["obs_list"] == [] and len(want["beam_grid_ids"]) == C.R


def test_tied_logits_take_the_first_maximum(golden):
  cfg, _ = C.case_config("tied_logits", None)
  outs = C.load_outputs(golden, "tied_logits", cfg)
  lg = outs[0][0][0].reshape(C.BS, C.T_PRED, -1)
  assert ((lg == lg.max(-1, keepdims=True)).sum(-1) > 1).all()       # every step has a tie at its maximum


def test_default_rows_per_forward():
  assert sfe.default_rows_per_forward(16) == 256
  assert sfe.default_rows_per_forward(20) == 240
  assert sfe.default_rows_per_forward(12) == 252
  assert sfe.default_rows_per_forward(300) == 300


def fake_model(grids, use_grids):
  h = lambda name, i=None: ("h", name, i)
  m = types.SimpleNamespace(config=types.SimpleNamespace(scene_grids=grids, use_grids=use_grids),
                            scene_feat=h("scene_feat"), obs_scene=h("obs_scene"), pred_length=h("pred_length"),
                            obs_traj=h("obs_traj"))
  m.grid_obs_labels = [h("grid_obs_labels", i) for i in range(len(grids))]
  m.grid_obs_regress = [h("grid_obs_regress", i) for i in range(len(grids))]
  m.grid_centers = [h("grid_centers", i) for i in range(len(grids))]
  return m


def feed(m, n, frames, traj, seed, centers):
  rng = np.random.default_rng(seed)
  fd = {m.scene_feat: rng.random((frames, 2, 2, 1)).astype(np.float32),
        m.obs_scene: rng.integers(0, frames, (n, 3)).astype(np.int32), m.pred_length: np.full((n,), 12, np.int32)}
  for j, (h, w) in enumerate(m.config.scene_grids):
    fd[m.grid_obs_labels[j]] = rng.integers(0, h * w, (n, 3)).astype(np.int32)
    if traj:
      fd[m.grid_centers[j]] = centers[j]
    else:
      fd[m.grid_obs_regress[j]] = rng.random((n, 3, h, w, 2)).astype(np.float32)
  if traj:
    fd[m.obs_traj] = rng.random((n, 3, 2))
  return fd


@pytest.mark.parametrize("traj", [False, True])
def test_batch_feeds_concatenates_batches(traj):
  m = fake_model([(2, 3), (1, 2)], [True, True])
  centers = [np.zeros((2, 3, 2)), np.ones((1, 2, 2))]
  fds = [feed(m, 4, f, traj, s, centers) for s, f in enumerate((3, 1, 2))]
  out, lengths = multifuture.batch_feeds(m, fds)
  assert lengths.dtype == np.int32 and (lengths == 12).all() and lengths.shape == (12,)
  assert np.array_equal(out[m.scene_feat], np.concatenate([fd[m.scene_feat] for fd in fds]))
  assert np.array_equal(out[m.obs_scene], np.concatenate([fds[0][m.obs_scene], fds[1][m.obs_scene] + 3,
                                                          fds[2][m.obs_scene] + 4]))
  for j in range(2):
    assert np.array_equal(out[m.grid_obs_labels[j]], np.concatenate([fd[m.grid_obs_labels[j]] for fd in fds]))
    if traj:
      assert out[m.grid_centers[j]] is centers[j] and m.grid_obs_regress[j] not in out
    else:
      assert np.array_equal(out[m.grid_obs_regress[j]], np.concatenate([fd[m.grid_obs_regress[j]] for fd in fds]))
  assert (m.obs_traj in out) == traj
  if traj:
    assert np.array_equal(out[m.obs_traj], np.concatenate([fd[m.obs_traj] for fd in fds]))


def test_batch_feeds_refuses_mixed_feeds():
  m = fake_model([(2, 3)], [True])
  c = [np.zeros((2, 3, 2))]
  with pytest.raises(ValueError):
    multifuture.batch_feeds(m, [feed(m, 2, 1, True, 0, c), feed(m, 2, 1, False, 1, c)])
  with pytest.raises(ValueError):
    multifuture.batch_feeds(m, [feed(m, 2, 1, True, 0, c), feed(m, 2, 1, True, 1, [np.ones((2, 3, 2))])])


def test_split_argv_takes_the_flag_name():
  assert multifuture.split_argv(["s.py", "--batch_size", "3", "--x"]) == ("s.py", ["--x"], 3)
  assert multifuture.split_argv(["s.py", "--batch_size", "20", "--eval_batch_size=40", "--y", "1"],
                                flag="--eval_batch_size", default=None) == ("s.py", ["--batch_size", "20", "--y", "1"],
                                                                             40)
  assert multifuture.split_argv(["s.py", "--batch_size", "20"], flag="--eval_batch_size", default=None)[2] is None
  with pytest.raises(SystemExit):
    multifuture.split_argv(["s.py", "--eval_batch_size", "0"], flag="--eval_batch_size", default=None)


def test_check_data_refuses_other_dtypes(golden):
  cfg, _ = C.case_config("greedy_two_scale", None)
  data, shared = C.case_data(C.load_set(golden), False)
  sfe.check_data(types.SimpleNamespace(data=data, shared=shared), cfg)
  data64 = dict(data, pred_traj=data["pred_traj"].astype(np.float64))
  sfe.check_data(types.SimpleNamespace(data=data64, shared=shared), cfg)
  with pytest.raises(TypeError):
    sfe.check_data(types.SimpleNamespace(data=dict(data, pred_traj=data["pred_traj"].astype(np.float16)),
                                         shared=shared), cfg)
  with pytest.raises(TypeError):
    sfe.check_data(types.SimpleNamespace(data=data, shared=dict(shared, grid_center_1=shared["grid_center_1"]
                                                                .astype(np.float32))), cfg)


STUB_PRED_UTILS = '''
def get_scene(key):
  return key
def evaluate(dataset, config, sess, tester):
  return {"host": True}
'''

STUB_SCRIPT = '''
import argparse
import json
import sys
import pred_utils
parser = argparse.ArgumentParser()
parser.add_argument("out")
parser.add_argument("--batch_size", type=int, default=64)
if __name__ == "__main__":
  args = parser.parse_args()
  res = pred_utils.evaluate("data", args, None, "tester")
  with open(args.out, "w") as f:
    json.dump(dict(res=res, batch_size=args.batch_size, argv=sys.argv[1:], pred_utils=pred_utils.__file__), f)
'''


@pytest.fixture
def clean_modules(monkeypatch):
  monkeypatch.setattr(sys, "path", list(sys.path))
  before = {k: sys.modules.get(k) for k in ("pred_utils", "tensorflow", "pred_models")}
  yield
  for k, v in before.items():
    if v is None:
      sys.modules.pop(k, None)
    else:
      sys.modules[k] = v


def test_runner_replaces_evaluate_and_runs_the_script(tmp_path, monkeypatch, clean_modules):
  import json
  (tmp_path / "pred_utils.py").write_text(STUB_PRED_UTILS)
  (tmp_path / "test.py").write_text(STUB_SCRIPT)
  seen = []

  def fake(dataset, config, sess, tester, rows_per_forward=None):
    seen.append((dataset, config.batch_size, tester, rows_per_forward))
    return {"device": True}

  monkeypatch.setattr(sfe, "evaluate", fake)
  out = tmp_path / "out.json"
  sys.modules.pop("pred_utils", None)
  sfe.main([str(tmp_path / "test.py"), str(out), "--batch_size", "7", "--eval_batch_size", "42"])
  got = json.loads(out.read_text())
  assert got["res"] == {"device": True} and got["batch_size"] == 7
  assert got["argv"] == [str(out), "--batch_size", "7"]
  assert os.path.dirname(got["pred_utils"]) == str(tmp_path)
  assert seen == [("data", 7, "tester", 42)]


def test_runner_refuses_pred_utils_without_evaluate(tmp_path, clean_modules):
  (tmp_path / "pred_utils.py").write_text("x = 1\n")
  (tmp_path / "test.py").write_text(STUB_SCRIPT)
  sys.modules.pop("pred_utils", None)
  with pytest.raises(SystemExit):
    sfe.main([str(tmp_path / "test.py"), str(tmp_path / "o.json")])
