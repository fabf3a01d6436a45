# coding=utf-8
"""Regenerates tests/golden/*.npz (fp64).  Run from the repo root, in the container that has
/root/reference:
    python tests/golden/make_golden.py
The ROLLOUT goldens are outputs of the reference's own code: the unmodified
/root/reference/code/pred_models.py executed on the eager TF-1.15 stand-in of oracle/tf1_eager
(``source = "reference_exec"``); the script asserts that the oracle restatement agrees to 1e-12
with identical ids before writing them.  The unit-op goldens (cell, gnn, head, beam_step, scene)
come from the oracle functions that the same execution pins."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle.tf1_eager import run_reference as X  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
f64 = lambda d: {k: (v.astype(np.float64) if v.dtype.kind == "f" else v) for k, v in d.items()}


def save(name, **kw):
  np.savez_compressed(os.path.join(OUT, name + ".npz"), **kw)
  print("wrote", name, {k: np.asarray(v).shape for k, v in kw.items()})


def main():
  for name in cases.CELL_CASES:
    d = cases.cell_case(name)
    q = f64(d)
    c1, h1 = R.convlstm_cell(q["x"], q["c"], q["h"], q["kernel"], q["biases"])
    c0, h0 = R.convlstm_cell(q["x"], np.zeros_like(q["c"]), q["h"], q["kernel"], q["biases"])
    if c1.nbytes * 4 > 1.5e6:            # keeps every file under 1 MB: the zero-state pair in a file of its own
      save("cell_" + name, checksum=cases.checksum(*d.values()), c=c1, h=h1)
      save("cell_%s_zero" % name, c_zero=c0, h_zero=h0)
    else:
      save("cell_" + name, checksum=cases.checksum(*d.values()), c=c1, h=h1, c_zero=c0, h_zero=h0)

  d = cases.gnn_case(); q = f64(d)
  save("gnn", checksum=cases.checksum(*d.values()), with_scene=R.gnn_dense(q["h"], q["scene"]),
       no_scene=R.gnn_dense(q["h"], None))

  d = cases.head_case(); q = f64(d)
  n, h, w, _ = d["h"].shape
  lg = R.hidden2grid(q["h"], q["Wo1"]); off = R.hidden2grid(q["h"], q["Wo2"])
  ids = lg.reshape(n, -1).argmax(1).astype(np.int32)
  oh = R.one_hot(ids, h * w, np.float64).reshape(n, h, w, 1)
  save("head", checksum=cases.checksum(*d.values()), logits=lg, ids=ids, offsets=off,
       emb_onehot=R.grid_emb(oh, q["We1"], q["be"]), emb_dense=R.grid_emb(off, q["We2"], q["be"]))

  d = cases.beam_case()
  out = {}
  for tag, (first, zero, div) in dict(first=(1, 1, 1), mid=(0, 0, 1), plain=(0, 0, 0),
                                      first_plain=(1, 0, 0)).items():
    lp = R.log_softmax(d["logits"].astype(np.float32)) + d["score"][:, :, None]
    if div:
      lp = R.add_div_penalty(lp, 0.01)
    n, b, v = lp.shape
    cand = lp[:, 0] if first else lp.reshape(n, b * v)
    sc, idx = R.top_k_sorted(cand, b)
    out[tag + "_score"] = np.zeros_like(sc) if zero else sc
    out[tag + "_ids"] = (idx % v).astype(np.int32)
    out[tag + "_parents"] = (idx // v).astype(np.int32)
  save("beam_step", checksum=cases.checksum(*d.values()), **out)

  d = cases.scene_case(); q = f64(d)
  wts = {"person_pred/scene_conv1/W": q["W1"], "person_pred/scene_conv1/b": q["b1"],
         "person_pred/scene_conv2/W": q["W2"], "person_pred/scene_conv2/b": q["b2"]}
  s1, s2 = R.scene_cnn(q["scene_feat"], d["obs_scene"], wts, 2)
  save("scene", checksum=cases.checksum(*d.values()), conv1=s1, conv2=s2, mean1=s1.mean(1), mean2=s2.mean(1))

  for name, (over, seed) in cases.ROLLOUTS.items():
    cfg = R.default_config(**over)
    w = R.make_weights(cfg, seed); f = R.make_inputs(cfg, seed)
    r = R.forward(cfg, w, f, np.float64)
    source = "oracle"
    if X.available():
      x = X.forward(cfg, w, f)
      for i in range(len(cfg.scene_grids)):
        if cfg.use_grids[i]:
          for k in ("grid_pred_decoded", "grid_pred_reg_decoded"):
            assert np.abs(x[k][i] - r[k][i]).max() <= 1e-12 * np.abs(r[k][i]).max(), (name, k, i)
      if r["beam_outputs"] is not None:
        assert np.array_equal(x["beam_outputs"][1], r["beam_outputs"][1])
        assert np.abs(x["beam_outputs"][0] - r["beam_outputs"][0]).max() < 1e-11
        assert np.abs(x["beam_outputs"][2] - r["beam_outputs"][2]).max() < 1e-11
      r = dict(r, grid_pred_decoded=x["grid_pred_decoded"], grid_pred_reg_decoded=x["grid_pred_reg_decoded"],
               beam_outputs=x["beam_outputs"])
      source = "reference_exec"
    out = dict(source=source, checksum=cases.checksum(*w.values()) + cases.checksum(f["scene_feat"], f["traj"]))
    for i in range(len(cfg.scene_grids)):
      if not cfg.use_grids[i]:
        continue
      lg = r["grid_pred_decoded"][i]
      out["logits_%d" % i] = lg.astype(np.float32)
      s = np.sort(lg.reshape(lg.shape[0], lg.shape[1], -1), -1)
      out["margin_%d" % i] = s[..., -1] - s[..., -2]
      out["reg_%d" % i] = r["grid_pred_reg_decoded"][i].astype(np.float32)
    if r["beam_outputs"] is not None:
      lgb, ids, lp = r["beam_outputs"]
      out["beam_ids"] = ids
      out["beam_logprobs"] = lp
      out["beam_logits_top3"] = lgb[:, :3].astype(np.float32)
    save("rollout_" + name, **out)


if __name__ == "__main__":
  main()
