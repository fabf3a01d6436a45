# coding=utf-8
"""Batched multi-future inference: what code/multifuture_inference.py computes, many trajectories per forward.

That script decodes every trajectory alone (N=1 per `sess.run`, :460-472), each to its own length, the longest of
its ground-truth futures (`max_pred_lengths`, :229-231, :311).  `infer` concatenates the script's own N=1 feeds into
batches and decodes each batch with ConvRNNEngine.forward(pred_lengths=...), whose rows equal their batch-1 decodes
byte for byte, so its `output_data` and `beam_prob` equal the script's loop in values, dtypes and structure.  From the
device it fetches the selected cells and their fp32 offsets (ops.gather_offsets), and the beam logits only when the
probabilities are asked for; the points `centre + offset` are formed in float64 on the host, as the script does
(:495-517).

Command line (the user's copy of the script, imported through the drop-in path, provides the argument parser, the
data loading and the feeds):

  python -m multiverse_b200.multifuture <path to code/multifuture_inference.py> <its arguments> [--batch_size N]
      [--eval]

--eval also scores every batch on the device against the ground truth the script loaded (multifuture_eval.Evaluation)
and prints what code/multifuture_eval_trajs.py and, for a beam decode, code/multifuture_eval_trajs_prob.py print for
the pickles; the beam logits stay on the device unless --save_prob_file asks for them.
"""
from __future__ import annotations

import argparse
import glob
import importlib.util
import os
import pickle
import sys

import numpy as np

DEFAULT_BATCH = 256


def batch_feeds(model, feeds):
  """One feed dict of N rows from the feed dicts `feeds` (the script's N=1 feeds, or get_feed_dict's batches), and
  their lengths int32 [N]: the rows concatenated, each feed's frames appended to scene_feat and its obs_scene indices
  offset to match.  Feeds that carry their observed trajectories (obs_traj + grid_centers, get_feed_dict's row f-1
  path) are concatenated as those; all feeds must then carry them, with the same centres."""
  cfg = model.config
  scene, obs_scene, frames = [], [], 0
  for fd in feeds:
    sf = np.asarray(fd[model.scene_feat])
    scene.append(sf)
    obs_scene.append(np.asarray(fd[model.obs_scene], dtype=np.int32) + frames)
    frames += sf.shape[0]
  out = {model.scene_feat: np.concatenate(scene), model.obs_scene: np.concatenate(obs_scene)}
  traj = [model.obs_traj in fd for fd in feeds]
  if any(traj) and not all(traj):
    raise ValueError("batch_feeds: feeds with dense offsets and feeds with trajectories cannot share a forward")
  if all(traj):
    out[model.obs_traj] = np.concatenate([np.asarray(fd[model.obs_traj]) for fd in feeds])
  for j in range(len(cfg.scene_grids)):
    if cfg.use_grids[j]:
      out[model.grid_obs_labels[j]] = np.concatenate([np.asarray(fd[model.grid_obs_labels[j]]) for fd in feeds])
      if all(traj):
        c = feeds[0][model.grid_centers[j]]
        if any(fd[model.grid_centers[j]] is not c and not np.array_equal(fd[model.grid_centers[j]], c) for fd in feeds):
          raise ValueError("batch_feeds: the feeds' grid centres of scale %d differ" % j)
        out[model.grid_centers[j]] = c
      else:
        out[model.grid_obs_regress[j]] = np.concatenate([np.asarray(fd[model.grid_obs_regress[j]]) for fd in feeds])
  lengths = np.concatenate([np.broadcast_to(np.asarray(fd[model.pred_length]).reshape(-1),
                                            (np.asarray(fd[model.obs_scene]).shape[0],)) for fd in feeds])
  return out, lengths.astype(np.int32)


def trajectories(ids, offs, length, centers, num_out, greedy, center_only):
  """One trajectory's entry of the script's output_data (:475-520): ids int [K,T] (greedy: [1,T]), offs fp32 [K,T,2]
  of the selected cells, centers fp64 [HW,2]."""
  if center_only:
    points = [[centers[ids[k, t]] for t in range(length)] for k in range(ids.shape[0])]
  else:
    pts = centers[ids[:, :length]] + offs[:, :length]
    points = [[pts[k, t] for t in range(length)] for k in range(ids.shape[0])]
  if greedy:
    return [points[0] for _ in range(num_out)]      # one list, num_out times (:498)
  return points[:num_out]


def infer(model, per_trajectory_feeds, batch_size, args, traj_ids, with_prob=False, evaluation=None):
  """(output_data, beam_prob) of the script's loop (:460-523) for its N=1 feeds `per_trajectory_feeds`
  (PredictionModelInference.get_feed_dict) of the trajectories `traj_ids`, decoded `batch_size` trajectories per
  forward.  `args`: the script's arguments after add_grid.  beam_prob (the beam logits and log-probabilities,
  --save_prob_file) is fetched only with `with_prob`; it is {} otherwise.  `evaluation` (a multifuture_eval.Evaluation)
  is given every batch's selections, offsets and beam outputs on the device."""
  import torch
  from . import ops
  cfg = model.config
  assert sum(cfg.use_grids) == 1, "multifuture inference decodes one scale (multifuture_inference.py:395)"
  if with_prob and not cfg.use_beam_search:
    raise ValueError("beam probabilities need beam search (the script's --greedy has no beam outputs)")
  gi = list(cfg.use_grids).index(True)
  centers = np.asarray(args.scene_grid_centers[gi]).reshape([-1, 2])
  greedy = not cfg.use_beam_search
  eng = model._ensure_engine()
  output_data, beam_prob = {}, {}
  with torch.cuda.device(eng.device):
    for b0 in range(0, len(per_trajectory_feeds), batch_size):
      chunk = per_trajectory_feeds[b0:b0 + batch_size]
      # a short last batch is padded to the batch size with length-1 rows: the engine keeps its buffers per batch
      # size, and a second set at batch 512 would not fit next to the first
      pad = batch_size - len(chunk) if b0 > 0 else 0
      feed, lengths = batch_feeds(model, chunk + chunk[-1:] * pad)
      lengths[len(chunk):] = 1
      n = len(lengths)
      out = eng.forward(model._device_feeds(feed), pred_lengths=lengths)
      if greedy:
        ids = out["grid_pred_decoded"][gi].reshape(n, int(lengths.max()), -1).argmax(-1).to(torch.int32)
        ids = ids.unsqueeze(1).contiguous()
      else:
        ids = out["beam_outputs"][1]
      offs = ops.gather_offsets(ids, out["_offs"][gi].contiguous(), out["_lengths"])
      if evaluation is not None:
        m, bo = len(chunk), out.get("beam_outputs")
        evaluation.add(traj_ids[b0:b0 + m], ids[:m], offs[:m], out["_lengths"][:m],
                       bo[0][:m] if bo is not None else None, bo[2][:m] if bo is not None else None)
      ids_h, offs_h = ids.cpu().numpy(), offs.cpu().numpy()
      if with_prob:
        logits_h, logprobs_h = out["beam_outputs"][0].cpu().numpy(), out["beam_outputs"][2].cpu().numpy()
      for r in range(len(chunk)):
        tid, length = traj_ids[b0 + r], int(lengths[r])
        output_data[tid] = trajectories(ids_h[r], offs_h[r], length, centers, args.num_out, greedy, args.center_only)
        if with_prob:
          beam_prob[tid] = (np.ascontiguousarray(logits_h[r:r + 1, :, :length]), logprobs_h[r:r + 1].copy())
  return output_data, beam_prob


def load_script(path, name="multifuture_inference"):
  """The user's script at `path` as a module named `name` (run as the script with name "__main__"), its
  `pred_models` and `tensorflow` the drop-in's and its own directory next on sys.path (its pred_utils)."""
  from . import pred_models  # noqa: F401  (puts the drop-in directory first on sys.path)
  add_script_dir(path)
  spec = importlib.util.spec_from_file_location(name, path)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def add_script_dir(path):
  """The script's directory on sys.path right after the drop-in's, so that its own modules (pred_utils) import."""
  from . import pred_models  # noqa: F401
  here = os.path.dirname(os.path.abspath(path))
  if here not in sys.path:
    sys.path.insert(1, here)         # after the drop-in: the script's own pred_utils


def model_config(args, tf):
  """The model Namespace of multifuture_inference.py:419-452."""
  return argparse.Namespace(
      modelname="model", batch_size=1,
      beam_size=args.num_out, use_beam_search=args.use_beam_search, diverse_beam=args.diverse_beam,
      diverse_gamma=args.diverse_gamma, fix_num_timestep=args.fix_num_timestep,
      use_teacher_forcing=False, is_train=False,
      scene_h=args.scene_h, scene_w=args.scene_w, scene_class=args.scene_class,
      use_soft_grid_class=args.use_soft_grid_class, use_single_decoder=args.use_single_decoder,
      pred_len=12, emb_size=args.emb_size, enc_hidden_size=args.enc_hidden_size,
      dec_hidden_size=args.dec_hidden_size, activation_func=tf.nn.tanh, scene_conv_kernel=args.scene_conv_kernel,
      use_scene_enc=args.use_scene_enc, scene_conv_dim=args.scene_conv_dim, convlstm_kernel=args.convlstm_kernel,
      use_gnn=args.use_gnn, keep_prob=1.0, scene_grid_strides=args.scene_grid_strides,
      scene_grids=args.scene_grids, use_grids=args.use_grids)


def prepare(script_path, script_argv, load_weights=True, return_gt=False):
  """The script's set-up (:389-461) through its own functions: returns (args, traj_ids, model, per-trajectory
  feeds), and with return_gt the ground truth it loaded (gt_trajs: traj id -> future dict) after them.
  load_weights=False leaves the model's initial weights (no checkpoint read)."""
  mod = load_script(script_path)
  tf = sys.modules["tensorflow"]
  args = mod.parser.parse_args(script_argv)
  mod.add_grid(args)
  args.use_beam_search = not args.greedy
  assert sum(args.use_grids) == 1
  traj_files = glob.glob(os.path.join(args.traj_path, "*.txt"))
  traj_ids = [os.path.splitext(os.path.basename(one))[0] for one in traj_files]
  gt_trajs = {}
  for traj_id in traj_ids:
    with open(os.path.join(args.multifuture_path, "%s.p" % traj_id), "rb") as f:
      gt_trajs[traj_id] = pickle.load(f)
  inputs = mod.get_inputs(args, traj_files, gt_trajs)
  cfg = model_config(args, tf)
  with tf.device("/gpu:%s" % args.gpuid):
    model = mod.PredictionModelInference(cfg, cfg.modelname)
  model.gpuid = args.gpuid
  if load_weights:
    with tf.Session() as sess:
      mod.load_model_weights(args.model_path, sess, top_scope="person_pred")
  feeds = [model.get_feed_dict(inputs, args, i) for i in range(len(traj_ids))]
  if return_gt:
    return args, traj_ids, model, feeds, gt_trajs
  return args, traj_ids, model, feeds


def split_argv(argv, flag="--batch_size", default=DEFAULT_BATCH,
               usage="python -m multiverse_b200.multifuture <multifuture_inference.py> <its arguments> "
                     "[--batch_size N]"):
  """(script path, the script's arguments, this module's value of `flag`) from this module's command line."""
  if not argv or argv[0].startswith("-"):
    raise SystemExit("usage: " + usage)
  rest, batch, i = [], default, 1
  while i < len(argv):
    a = argv[i]
    if a == flag:
      batch, i = int(argv[i + 1]), i + 2
      continue
    if a.startswith(flag + "="):
      batch = int(a.split("=", 1)[1])
    else:
      rest.append(a)
    i += 1
  if batch is not None and batch < 1:
    raise SystemExit("%s must be at least 1" % flag)
  return argv[0], rest, batch


def split_eval(argv):
  """(argv without --eval, whether it was given)."""
  rest = [a for a in argv if a != "--eval"]
  return rest, len(rest) != len(argv)


def make_evaluation(model, args, gt_trajs):
  """The multifuture_eval.Evaluation of this decode: the decoded scale's centres and grid, the script's frame size;
  NLL only for a beam decode (the greedy one has no beam logits)."""
  from . import multifuture_eval
  cfg = model.config
  gi = list(cfg.use_grids).index(True)
  return multifuture_eval.Evaluation(gt_trajs, args.scene_grid_centers[gi], args.center_only, cfg.scene_grids[gi],
                                     (args.video_h, args.video_w), with_nll=bool(cfg.use_beam_search))


def main(argv=None):
  argv, evaluate = split_eval(sys.argv[1:] if argv is None else argv)
  script, script_argv, batch = split_argv(argv)
  args, traj_ids, model, feeds, gt_trajs = prepare(script, script_argv, return_gt=True)
  with_prob = args.save_prob_file is not None
  evaluation = make_evaluation(model, args, gt_trajs) if evaluate else None
  if evaluate and not args.use_beam_search:
    print("--eval: no NLL for --greedy (it has no beam logits)", file=sys.stderr)
  output_data, beam_prob = infer(model, feeds, batch, args, traj_ids, with_prob=with_prob, evaluation=evaluation)
  with open(args.output_file, "wb") as f:
    pickle.dump(output_data, f)
  if with_prob:
    with open(args.save_prob_file, "wb") as f:
      pickle.dump(beam_prob, f)
  if evaluation is not None:
    for line in evaluation.lines():
      print(line)


if __name__ == "__main__":
  main()
