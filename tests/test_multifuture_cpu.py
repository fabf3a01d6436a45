# coding=utf-8
"""CPU tests of the batched multi-future driver's host side (multiverse_b200.multifuture): on a tiny dataset directory
in the Forking Paths layout, the per-trajectory feeds the command line prepares equal those of the unmodified
reference script's own get_feed_dict (code/multifuture_inference.py, imported through the drop-in); a batch holds
exactly its trajectories' feeds; and the output entries are pickled like the script's."""
import json
import os
import pickle
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(os.environ.get("MVB_REFERENCE_ROOT", "/root/reference"), "code", "multifuture_inference.py")
needs_reference = pytest.mark.skipif(not os.path.exists(SCRIPT), reason="the reference repository is not installed")


@pytest.fixture()
def dropin(monkeypatch):
  monkeypatch.setattr(sys, "path", list(sys.path))      # load_script adds the script's directory
  monkeypatch.syspath_prepend(os.path.join(ROOT, "multiverse_b200", "dropin"))
  for m in ("tensorflow", "tensorflow.compat", "tensorflow.compat.v1", "pred_models", "pred_utils",
            "multiverse_b200.pred_models", "multifuture_inference"):
    monkeypatch.delitem(sys.modules, m, raising=False)
  import tensorflow as tf
  tf.reset_default_graph()
  yield tf
  tf.reset_default_graph()


def make_dataset(root, n=5, obs=8, sh=36, sw=64, seed=0):
  """traj_path/<id>.txt (frame, person, x, y), multifuture_path/<id>.p (future id -> x_agent_traj), scene_feat_path/
  <id>/<id>_F_<frame>.npy (class ids [sh, sw]) and the id2name json of the script's get_inputs (:158-272)."""
  rng = np.random.default_rng(seed)
  dirs = {k: os.path.join(root, k) for k in ("traj", "multifuture", "scene")}
  for d in dirs.values():
    os.makedirs(d)
  for r in range(n):
    tid = "%04d_%d_%d_cam%d" % (r, 10 + r, 3 + r, r % 4)
    frames = 100 + 12 * np.arange(obs) + r
    xy = np.cumsum(rng.normal(0, 20, (obs, 2)), 0) + [900, 500]
    with open(os.path.join(dirs["traj"], tid + ".txt"), "w") as f:
      for t in range(obs):
        f.write("%d\t%d\t%.2f\t%.2f\n" % (frames[t], 3 + r, xy[t, 0], xy[t, 1]))
        f.write("%d\t%d\t%.2f\t%.2f\n" % (frames[t], 99, xy[t, 0] + 50, xy[t, 1]))
    futures = {fid: {"x_agent_traj": [[0, 0, 0]] * int(rng.integers(10, 27))} for fid in range(3)}
    with open(os.path.join(dirs["multifuture"], tid + ".p"), "wb") as f:
      pickle.dump(futures, f)
    os.makedirs(os.path.join(dirs["scene"], tid))
    for fr in frames:
      np.save(os.path.join(dirs["scene"], tid, "%s_F_%08d.npy" % (tid, fr)), rng.integers(0, 14, (sh, sw)))
  id2name = os.path.join(root, "id2name.json")
  with open(id2name, "w") as f:
    json.dump({"oldid2new": {str(i): i for i in range(1, 11)}, "id2name": {str(i): "c%d" % i for i in range(1, 11)}},
              f)
  return [dirs["traj"], dirs["multifuture"], os.path.join(root, "model"), os.path.join(root, "out.traj.p"),
          "--save_prob_file", os.path.join(root, "out.prob.p"), "--obs_length", str(obs), "--emb_size", "32",
          "--use_scene_enc", "--scene_id2name", id2name, "--scene_feat_path", dirs["scene"], "--grid_strides", "2,4",
          "--use_grids", "1,0", "--num_out", "20", "--diverse_beam", "--use_gnn", "--diverse_gamma", "0.01",
          "--fix_num_timestep", "1"]


def test_command_line_split():
  from multiverse_b200 import multifuture
  assert multifuture.split_argv(["s.py", "a", "--batch_size", "64", "--num_out", "5"]) == ("s.py", ["a", "--num_out",
                                                                                                    "5"], 64)
  assert multifuture.split_argv(["s.py", "--batch_size=8", "b"]) == ("s.py", ["b"], 8)
  assert multifuture.split_argv(["s.py", "b"])[2] == multifuture.DEFAULT_BATCH
  with pytest.raises(SystemExit):
    multifuture.split_argv(["--batch_size", "4"])


@needs_reference
def test_feeds_equal_the_reference_scripts(dropin, tmp_path):
  import glob
  from multiverse_b200 import multifuture
  argv = make_dataset(str(tmp_path))
  args, traj_ids, model, feeds = multifuture.prepare(SCRIPT, argv, load_weights=False)
  assert len(feeds) == 5
  # the script's own set-up (:389-461), step by step, on a module of its own
  tf = dropin
  tf.reset_default_graph()
  sys.modules.pop("multifuture_inference", None)
  mod = multifuture.load_script(SCRIPT)
  a = mod.parser.parse_args(argv)
  mod.add_grid(a)
  a.use_beam_search = True
  files = glob.glob(os.path.join(a.traj_path, "*.txt"))
  ids = [os.path.splitext(os.path.basename(p))[0] for p in files]
  assert ids == traj_ids
  gt = {}
  for tid in ids:
    with open(os.path.join(a.multifuture_path, "%s.p" % tid), "rb") as f:
      gt[tid] = pickle.load(f)
  inputs = mod.get_inputs(a, files, gt)
  ref_model = mod.PredictionModelInference(multifuture.model_config(a, tf), "model")
  key = lambda h: (h.name, h.index)
  for i in range(len(ids)):
    theirs = {key(h): v for h, v in ref_model.get_feed_dict(inputs, a, i).items()}
    ours = {key(h): v for h, v in feeds[i].items()}
    assert set(ours) == set(theirs)
    for k in theirs:
      x, y = np.asarray(ours[k]), np.asarray(theirs[k])
      assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), k
  plain = lambda ns: {k: v for k, v in vars(ns).items() if k != "scene_grid_centers"}
  assert plain(args) == plain(a)
  assert all(np.array_equal(x, y) for x, y in zip(args.scene_grid_centers, a.scene_grid_centers))
  # the restated model Namespace carries what the engine reads
  cfg = model.config
  assert (cfg.beam_size, cfg.use_beam_search, cfg.diverse_beam, cfg.diverse_gamma, cfg.fix_num_timestep) == \
      (20, True, True, 0.01, 1)
  assert cfg.scene_grids == [(18, 32), (9, 16)] and cfg.use_grids == [True, False] and cfg.emb_size == 32

  # a batch: the trajectories' rows, their frames behind offset indices, their lengths
  from multiverse_b200.multifuture import batch_feeds
  batch, lengths = batch_feeds(model, feeds[1:4])
  assert lengths.dtype == np.int32 and lengths.tolist() == [inputs["max_pred_lengths"][i] for i in (1, 2, 3)]
  sf, os_ = batch[model.scene_feat], batch[model.obs_scene]
  assert sf.shape[0] == sum(np.asarray(fd[model.scene_feat]).shape[0] for fd in feeds[1:4])
  for r, fd in enumerate(feeds[1:4]):
    assert np.array_equal(sf[os_[r]], np.asarray(fd[model.scene_feat])[np.asarray(fd[model.obs_scene])[0]])
    for h in (model.grid_obs_labels[0], model.grid_obs_regress[0]):
      assert np.array_equal(batch[h][r], np.asarray(fd[h])[0])
  assert model.grid_obs_regress[1] not in batch


@pytest.mark.parametrize("greedy,center_only", [(False, False), (True, False), (False, True)])
def test_output_entries_pickle_like_the_scripts(greedy, center_only):
  """One trajectory's output_data entry against the script's per-step construction (:475-520)."""
  from multiverse_b200 import multifuture
  rng = np.random.default_rng(1)
  k, tp, v, length = (1 if greedy else 20), 26, 576, 17
  centers = rng.uniform(0, 1900, (v, 2))
  ids = rng.integers(0, v, (k, tp)).astype(np.int32)
  offs = rng.normal(0, 30, (k, tp, 2)).astype(np.float32)
  reg = np.zeros((length, v, 2), np.float32)
  trajs = []
  for j in range(k):
    reg[np.arange(length), ids[j, :length]] = offs[j, :length]
    trajs.append([centers[ids[j, t]] if center_only else centers[ids[j, t]] + reg[t, ids[j, t], :]
                  for t in range(length)])
  want = [trajs[0] for _ in range(20)] if greedy else trajs
  got = multifuture.trajectories(ids, offs, length, centers, 20, greedy, center_only)
  assert pickle.dumps(got) == pickle.dumps(want)
