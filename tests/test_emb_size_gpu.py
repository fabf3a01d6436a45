# coding=utf-8
"""Models built with --emb_size above 64 (the reference scripts' default is 128): x blocks of up to four 64-channel K
chunks in the cell (cpad = roundup(emb_size, 32) + 256 from 288 to 512), the backward GEMMs' tiles for them, and
emb_bwd's shared-memory channel groups.

Cell and GEMMs element by element against the fp64 references of test_kernels_atsize_gpu.py at cpad 352 (a trailing
32-channel chunk), 384 and 512: bar 3e-5 forward, 2e-4 gradients.  emb_bwd against torch autograd in fp64.  Rollouts
against the fp64 oracle (oracle/multiverse_ref_torch.py) at emb_size 96 and 128, and against the executed reference
(tests/golden/make_golden_emb_size.py): greedy, K = 5 plain and K = 20 diverse beams (checked along the engine's own
selections), one training step of train.py's own defaults and one drop-in Trainer.step at emb 96; the whole-model
gradient of train.py's default model (emb_size 128, no scene encoder) against the fp64 truth."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_kernels_atsize_gpu as K
from beam_truth import beam_replay
from test_beam_no_gnn_gpu import rel, to_dev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
HID = 256
F16F8 = 16
WIDE = [96, 128, 256]          # cx: cpad 352, 384, 512


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _release_memory():
  yield
  gc.collect()
  if torch.cuda.is_available():
    torch.cuda.empty_cache()


def wide_inputs(dev, ns, h, w, cx, seed):
  """K.cell_inputs with the x block in (-1, 1): every x block wider than 64 channels is a tanh embedding (the decoders'
  grid_emb, the class encoder's without scene encoding).  The forward error of both operand formats grows with K
  (about as its square root): at cx 256 and x ~ N(0, 1) the stored gates reach 3.4e-5."""
  d = K.cell_inputs(dev, ns, h, w, cx, seed)
  d["x"] = torch.tanh(d["x"])
  return d


def single_ns(h, w):
  """Largest single-CTA launch on h x w (several tiles per CTA), R not a multiple of 128."""
  ns = 1
  while K.m_tiles(ns + 1, h, w) < 2 * K.num_sms():
    ns += 1
  while K.halo_rows(ns, h, w) % K.BLOCK_M == 0:
    ns -= 1
  return ns


# --------------------------------------------------------------------------- cell forward
@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("launch", ["single", "pair"])
@pytest.mark.parametrize("cx", WIDE)
def test_cell_wide_x_block(dev, cx, launch, planes):
  """The x block through the GEMM in nqx = ceil(cxp / 64) chunks (the last one 32 channels wide at cx 96), both
  operand formats, under the single-CTA kernel (several tiles per CTA) and the CTA-pair kernel (odd M tiles)."""
  from multiverse_b200 import ops
  h, w = (36, 18) if cx != 128 else (18, 32)
  ns = K.pair_ns(h, w, odd=True) if launch == "pair" else single_ns(h, w)
  d = wide_inputs(dev, ns, h, w, cx, seed=400 + cx + (launch == "pair"))
  out = K.run_fwd(d, planes)
  assert ops.cell_cpad(cx) == out["xh2"].shape[2] == (cx + 31) // 32 * 32 + HID
  K.check_fwd("%s cx%d %dx%d n%d" % (launch, cx, h, w, ns), ns, h, w, out,
              K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]), planes, pair=launch == "pair")


@pytest.mark.parametrize("cx", WIDE)
def test_cell_wide_x_block_stores_the_gates(dev, cx):
  """cell_fwd_train (bf16x2, gates stored for the backward) under the pair kernel."""
  ns = K.pair_ns(36, 18, odd=True)
  d = wide_inputs(dev, ns, 36, 18, cx, seed=410 + cx)
  out = K.run_fwd(d, 2, train=True)
  K.check_fwd("fwd_train cx%d n%d" % (cx, ns), ns, 36, 18, out,
              K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]), 2, pair=True)


def _wide_emb(dev, e, seed):
  g = torch.Generator(device=dev)
  g.manual_seed(seed)
  return (torch.randn((3, 3, 1, e), generator=g, device=dev) * 0.5,
          torch.randn((e,), generator=g, device=dev) * 0.1)


@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("cx", [128, 256])
def test_cell_wide_x_fold(dev, cx, planes):
  """x-fold (the class decoder's embedded one-hot input as table look-ups; every x chunk skipped) with a row map,
  under the pair kernel; the tables (cell_xfold_tables) built at E = cx."""
  from multiverse_b200 import ops
  h, w = 36, 18
  ns = K.pair_ns(h, w, odd=True)
  d, ids, _, _, g = K._onehot_case(dev, ns, h, w, 420 + cx)
  d = dict(d, **{k: v for k, v in K.cell_inputs(dev, ns, h, w, cx, seed=420 + cx).items() if k in ("kernel", "x")})
  We, be = _wide_emb(dev, cx, 421 + cx)
  rm = torch.randint(0, ns, (ns,), generator=g, device=dev, dtype=torch.int32)
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  xf = ops.XFold(d["kernel"], d["bias"], We, be)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, planes, dev))
  ops.cell_fwd_onehot(xh, pk, xf, ids, K.to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns, row_map=rm)
  out["variant"] = ops.cell_last_variant()
  x = K.ref_onehot_emb(ids, h, w, We, be)
  K.check_fwd("x-fold cx%d n%d" % (cx, ns), ns, h, w, out,
              K.ref_cell(x, d["h"], d["c"], d["kernel"], d["bias"], row_map=rm), planes, pair=True)


def epi_outputs(path, cx, launch):
  """Child side of test_cell_wide_x_block_epilogue_warpgroup: one f16f8 cell launch, outputs saved to `path`."""
  dev = torch.device("cuda:0")
  ns = K.pair_ns(36, 18, odd=True) if launch == "pair" else single_ns(36, 18)
  d = wide_inputs(dev, ns, 36, 18, cx, seed=430 + cx)
  out = K.run_fwd(d, F16F8)
  torch.save(dict(c=out["c"].cpu(), h=out["h"].cpu(), xh2=out["xh2"].view(torch.int16).cpu(),
                  variant=out["variant"]), path)


@pytest.mark.parametrize("launch", ["single", "pair"])
@pytest.mark.parametrize("cx", WIDE)
def test_cell_wide_x_block_epilogue_warpgroup(dev, tmp_path, cx, launch):
  """cell_fwd_epi_kernel (MVB_CELL_EPI_WG=1: at every size) runs the same K order as cell_fwd_kernel
  (MVB_CELL_EPI_WG=0): c', h' and the next operands bit-identical, and within the forward bar of fp64.  The variant
  code does not tell the two f16f8 kernels apart: which one runs rests on MVB_CELL_EPI_WG, as in
  test_cell_epi_wg_gpu.py."""
  res = {}
  for epi in ("0", "1"):
    path = str(tmp_path / ("out%s.pt" % epi))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_emb_size_gpu as t; t.epi_outputs(%r, %d, %r)" % (
        ROOT, TESTS, path, cx, launch)
    env = dict({k: v for k, v in os.environ.items() if not k.startswith("MVB_CELL_")}, MVB_CELL_EPI_WG=epi)
    r = subprocess.run([sys.executable, "-B", "-c", code], env=env, cwd=ROOT, timeout=900, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res[epi] = torch.load(path)
  for o in res.values():
    assert o["variant"] == F16F8 * 2 + int(launch == "pair"), o["variant"]
  for k in ("c", "h", "xh2"):
    assert torch.equal(res["0"][k], res["1"][k]), "cx%d %s: %s differs between the two f16f8 kernels" % (cx, launch, k)
  ns = K.pair_ns(36, 18, odd=True) if launch == "pair" else single_ns(36, 18)
  d = wide_inputs(dev, ns, 36, 18, cx, seed=430 + cx)
  ref = K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"])
  errs = {k: rel(K.inner(res["1"][k], ns, 36, 18).numpy(), ref[k].cpu().numpy()) for k in ("c", "h")}
  print("epilogue warpgroup cx%d %s n%d: bit-identical to cell_fwd_kernel, rel err %s" % (cx, launch, ns, errs))
  assert max(errs.values()) < K.TIGHT, errs


def test_cell_refuses_x_blocks_past_256(dev):
  """cpad 544 (an x block of 288 channels) is refused before any launch."""
  from multiverse_b200 import ops
  d = K.cell_inputs(dev, 1, 4, 4, 288, seed=440)
  pk = ops.PackedCell(d["kernel"], d["bias"], 2)
  xh = ops.alloc_xh(1, 4, 4, pk.cpad, 2, dev)
  c_out, h_out = ops.alloc_state(1, 4, 4, dev), ops.alloc_state(1, 4, 4, dev)
  torch.cuda.synchronize()
  ops.reset_launch_count()
  with pytest.raises(RuntimeError, match="cpad=544"):
    ops.cell_fwd(xh, pk, None, c_out, h_out, None, 4, 4, 1)
  assert ops.launch_count() == 0


# --------------------------------------------------------------------------- dgrad / wgrad at training size
@pytest.mark.parametrize("grid", [(36, 18), (18, 32)], ids=["36x18", "18x32"])
@pytest.mark.parametrize("cx", WIDE)
def test_cell_backward_wide_x_block(dev, monkeypatch, cx, grid):
  """Micro-batch 128: dgrad with the x block (N tiles of 192 or 256 columns past cpad 320; no column past cpad
  stored), wgrad on 8 slabs with units that divide cpad, against fp64; the slabs accumulate to exactly 2x and repeat
  bit for bit; no halo row written."""
  name = "wide_cx%d" % cx
  monkeypatch.setitem(K.BWD_CELLS, name, (cx, 1.0, True))
  h, w = grid
  o, ref = K.run_backward(dev, name, 128, h, w, seed=450 + cx + h)
  assert o["dwp"].shape[0] == 8
  K.check_backward("backward cx%d %dx%d n128" % (cx, h, w), 128, h, w, o, ref)


# --------------------------------------------------------------------------- emb_bwd
def ref_emb_grads(dxh_in, ids, in_map, We, be, h, w):
  """fp64 autograd of x = tanh(conv3x3(in) + be): (dWe, dbe, d_in) for upstream dxh_in [ns, h, w, E]."""
  import torch.nn.functional as F
  We64 = We.double().requires_grad_(True)
  be64 = be.double().requires_grad_(True)
  ns = dxh_in.shape[0]
  if ids is not None:
    x_in = torch.zeros((ns, h * w, 1), dtype=torch.float64, device=We.device)
    x_in[torch.arange(ns), ids.long(), 0] = 1.0
    x_in = x_in.view(ns, h, w, 1)
  else:
    x_in = in_map.double().view(ns, h, w, -1).requires_grad_(True)
  pre = F.conv2d(x_in.permute(0, 3, 1, 2), We64.permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1) + be64
  torch.tanh(pre).backward(dxh_in.double())
  return We64.grad, be64.grad, (None if ids is not None else x_in.grad)


@pytest.mark.parametrize("kind", ["onehot", "dense1", "dense2"])
@pytest.mark.parametrize("grid", [(36, 18), (18, 32)], ids=["36x18", "18x32"])
@pytest.mark.parametrize("E", [128, 256])
def test_emb_bwd_wide(dev, E, grid, kind):
  """emb_bwd at E = 128 and 256 (channel groups of dpre in shared memory) against autograd: the one-hot input (class
  encoder without scene encoding), the logits map (Pout 1) and the offset map (Pout 2, with d_in added into a buffer)."""
  from multiverse_b200 import ops
  h, w = grid
  ns, pout = 16, 2 if kind == "dense2" else 1
  g = torch.Generator(device=dev)
  g.manual_seed(460 + E + h)
  cpad = ops.cell_cpad(E)
  We = torch.randn((3, 3, pout, E), generator=g, device=dev) * 0.3
  be = torch.randn((E,), generator=g, device=dev) * 0.1
  dx = torch.randn((ns, h, w, E), generator=g, device=dev)
  dxh = torch.zeros((ns, h + 1, w + 1, cpad), device=dev)
  dxh[:, :h, :w, :E] = dx
  dxh = dxh.view(-1, cpad)
  ids = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32) if kind == "onehot" else None
  in_map = None if kind == "onehot" else torch.randn((ns, h * w * pout), generator=g, device=dev)
  dWe, dbe = torch.zeros_like(We), torch.zeros_like(be)
  d_in = None if kind == "onehot" else torch.ones((ns, h * w * pout), device=dev)
  ops.emb_bwd(dxh, ids, in_map, We, be, dWe, dbe, d_in, True, h, w, ns)
  rW, rb, rin = ref_emb_grads(dx, ids, in_map, We, be, h, w)
  errs = dict(dWe=rel(dWe.cpu().numpy(), rW.cpu().numpy()), dbe=rel(dbe.cpu().numpy(), rb.cpu().numpy()))
  if rin is not None:
    errs["d_in"] = rel((d_in - 1.0).cpu().numpy(), rin.reshape(ns, -1).cpu().numpy())
  print("emb_bwd E%d %dx%d %s: %s" % (E, h, w, kind, {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < 1e-5, errs


# --------------------------------------------------------------------------- rollouts against the fp64 oracle
def oracle_forward(over, seed, dev, ref_on_gpu=True):
  from multiverse_b200 import ops, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  cfg = synthetic.make_config(**over)
  w = synthetic.make_weights(cfg, seed)
  f = synthetic.make_feeds(cfg, cfg.batch_size, seed)
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
  out = eng.forward(to_dev(f, dev))
  torch.cuda.synchronize()
  seen = ops.cell_variants_seen()
  with torch.no_grad():
    rdev = dev if ref_on_gpu else None
    ref = RT._forward(R.default_config(**over), {k: torch.from_numpy(v).double().to(rdev) for k, v in w.items()}, f,
                      torch.float64, rdev)
  return cfg, out, ref, seen


def _np(t):
  return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


@pytest.mark.parametrize("emb", [96, 128])
def test_rollout_greedy_two_scale_wide_emb(dev, emb):
  """test.py --use_scene_enc --use_gnn at --emb_size 96 / 128 (greedy, both scales, 8 trajectories): arg-max ids
  equal the oracle's wherever its top-2 gap clears 1e-4 x max|logit|, logits and offsets within the 1e-4 bar."""
  cfg, out, ref, seen = oracle_forward(dict(batch_size=8, emb_size=emb, use_gnn=True), 480 + emb, dev)
  errs = {}
  for i, (h, w) in enumerate(cfg.scene_grids):
    lg, rl = _np(out["grid_pred_decoded"][i]), _np(ref["grid_pred_decoded"][i])
    n, tp = lg.shape[:2]
    lg, rl = lg.reshape(n, tp, -1), rl.reshape(n, tp, -1)
    srt = np.sort(rl, -1)
    clear = srt[..., -1] - srt[..., -2] > 1e-4 * np.abs(rl).max()
    assert (lg.argmax(-1) == rl.argmax(-1))[clear].all()
    errs["logits_%d" % i] = rel(lg, rl)
    errs["offsets_%d" % i] = rel(_np(out["grid_pred_reg_decoded"][i]), _np(ref["grid_pred_reg_decoded"][i]))
  print("greedy emb %d: cell variants %s, rel errs %s" % (emb, sorted(seen), {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < 1e-4, errs


def golden_case(name):
  import cases
  import emb_size_cases as EC
  from multiverse_b200 import synthetic
  from oracle import multiverse_ref as R
  over, seed = EC.ROLLOUTS[name]
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  g = np.load(os.path.join(ROOT, "tests", "golden", "rollout_emb_%s.npz" % name))
  assert abs(float(g["checksum"]) - cases.checksum(*w.values()) - cases.checksum(f["scene_feat"], f["traj"])) < 1e-6
  return cfg, w, f, g


def run_traced(cfg, w, f, dev):
  """ConvRNNEngine.forward, with the per-step trace of decode_class_beam (cells, parents and logits of every step)."""
  from multiverse_b200 import ops
  from multiverse_b200.engine import ConvRNNEngine
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  trace, beam = [], eng.decode_class_beam

  def traced(*a, **kw):
    r = beam(*a, **kw)
    trace.append({k: v.cpu().numpy() for k, v in r[3].items()})
    return r
  eng.decode_class_beam = traced
  ops.cell_variants_seen(reset=True)
  out = eng.forward(to_dev(f, dev))
  torch.cuda.synchronize()
  return out, (trace[0] if trace else None), ops.cell_variants_seen()


@pytest.mark.parametrize("name", ["greedy_two_scale_emb128", "defaults_three_grids"])
def test_rollout_greedy_against_reference_execution(dev, name):
  """Greedy decoding at --emb_size 128 against the executed reference (tests/golden/rollout_emb_*.npz): with scene
  encoding and attention on both scales, and train.py's own model defaults (no scene encoder, no attention, three
  grids).  Arg-max ids bit-exact wherever the reference's top-2 gap clears 1e-4 x max|logit| (and on at least 90 % of
  the steps), logits and offsets within the 1e-4 rollout bar."""
  cfg, w, f, g = golden_case(name)
  out, _, seen = run_traced(cfg, w, f, dev)
  errs = {}
  for i in range(len(cfg.scene_grids)):
    lg = out["grid_pred_decoded"][i].cpu().numpy()
    n, tp = lg.shape[:2]
    ref = g["logits_%d" % i]
    clear = g["margin_%d" % i] > 1e-4 * np.abs(ref).max()
    assert clear.mean() > 0.9
    assert (lg.reshape(n, tp, -1).argmax(-1) == ref.reshape(n, tp, -1).argmax(-1))[clear].all(), i
    errs["logits_%d" % i] = rel(lg, ref)
    errs["offsets_%d" % i] = rel(out["grid_pred_reg_decoded"][i].cpu().numpy(), g["reg_%d" % i])
  print("%s: cell variants %s, rel errs %s" % (name, sorted(seen), {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < 1e-4, errs


@pytest.mark.parametrize("name", ["beam_k20_emb128", "beam_k5_emb96"])
def test_rollout_beam_against_reference_execution(dev, name):
  """Beam decoding at a wide --emb_size against the executed reference: K = 20 diverse beam with attention (emb 128,
  the CTA-pair f16f8 cell kernel) and K = 5 plain beam without attention (emb 96, cpad 352).
  - The fp64 truth replayed along the engine's own selections (beam_replay): every live row's logits at every step
    within the 1e-4 rollout bar, and the engine's outputs are the back-trace of that trace.
  - Ids: equal to the reference's, in its order, for every trajectory none of whose selections lies within 2e-4 of a
    tie (beam_margins); elsewhere the shared id sequences are reported.  The K = 20 case's reference selects
    candidates 2e-6, 3e-7 and 6e-9 apart (one per trajectory) once the scores are zeroed after the first selection
    (fix_num_timestep = 1): such candidates take their slots in either order at fp32, and the back-trace attaches
    to a beam at step t the logits of the row in its SLOT before the selection, so the returned logits are checked
    through the trace, not against the reference's slot order.
  - Offsets within the bar."""
  from multiverse_b200 import ops
  cfg, w, f, g = golden_case(name)
  out, tr, seen = run_traced(cfg, w, f, dev)
  if cfg.beam_size == 20:
    assert (ops.PLANES_F16F8, True) in seen, seen
  blg, ids, lp = [t.cpu().numpy() for t in out["beam_outputs"]]
  i = cfg.use_grids.index(True)
  truth = beam_replay(cfg, w, f, i, tr["ids"], tr["parents"], dev)
  err = rel(tr["logits"], truth)
  n, b, tp = ids.shape
  for j in range(n):                                    # the outputs are the back-trace of the checked trace
    par = np.arange(b)
    for t in range(tp - 1, -1, -1):
      assert np.array_equal(ids[j, :, t], tr["ids"][t, j, par]) and np.array_equal(blg[j, :, t], tr["logits"][t, j, par])
      par = tr["parents"][t, j, par]
  shared, clear = [], []
  for j in range(n):
    shared.append(len(set(map(tuple, ids[j].tolist())) & set(map(tuple, g["beam_ids"][j].tolist()))))
    if g["beam_margins"][:, j].min() > 2e-4:        # no selection of the reference near a tie: its ids, in its order
      clear.append(j)
      assert np.array_equal(ids[j], g["beam_ids"][j]), j
  reg = rel(out["grid_pred_reg_decoded"][i].cpu().numpy(), g["reg_%d" % i])
  print("%s: logits along the engine's selections %.1e (every live row, every step), offsets %.1e; ids equal the "
        "reference's for the %d trajectories clear of ties; id sequences shared per trajectory %s of %d; smallest gap "
        "between consecutive selected candidates of the reference per trajectory %s"
        % (name, err, reg, len(clear), shared, b, g["beam_margins"][..., 0].min(0)))
  assert err < 1e-4 and reg < 1e-4


# --------------------------------------------------------------------------- training
@pytest.mark.parametrize("use_gnn", [False, True], ids=["train_py_defaults", "gnn"])
def test_whole_model_gradient_emb128_without_scene_encoding(dev, use_gnn):
  """train.py's model defaults: --emb_size 128, no scene encoder (the class encoder's input is the embedded one-hot,
  cpad 384), without and with the attention; 256 trajectories in micro-batches of 128 against the fp64 truth along the
  engine's arg-max path (test_no_scene_enc_gpu's check), every gradient within 2e-4."""
  import no_scene_enc_ref as NS
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  from test_train_atsize_gpu import FRAMES, GTOL, LTOL, T_PRED, chunk_feeds, on, shared_frame_feeds
  n, mb, chunk = 256, 128, 16
  over = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, emb_size=128, use_gnn=use_gnn)
  cfg = synthetic.make_config(batch_size=mb, clip_gradient_norm=10.0, use_scene_enc=False, **over)
  rcfg = NS.config(batch_size=chunk, **over)
  seed = 500 + int(use_gnn)
  w = synthetic.make_weights(cfg, seed)
  assert w[NS.ENC_EMB[0]].shape == (3, 3, 1, 128)
  f = shared_frame_feeds(synthetic.make_config(batch_size=n, use_scene_enc=False, **over), n, FRAMES, seed)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  got, ids, mine = 0.0, [[], []], [[], []]
  for lo in range(0, n, mb):
    part = chunk_feeds(f, slice(lo, lo + mb))
    feeds = {k: ([on(dev, a) for a in v] if isinstance(v, list) else on(dev, v)) for k, v in part.items()}
    l, _ = eng.loss_and_grads(feeds, loss_scale=mb / n, zero=(lo == 0))
    got = got + l.cpu().numpy()
    for i in range(2):
      ids[i].append(eng._store[("ids", i, mb)][0].cpu().numpy().T)
      mine[i].append(eng.last_logits[i].cpu().numpy().transpose(1, 0, 2))
  torch.cuda.synchronize()
  ids = [np.concatenate(a) for a in ids]
  mine = [np.concatenate(a) for a in mine]
  eng_grads = {k: v.cpu().numpy() for k, v in eng.grads.items()}
  del eng, feeds                     # the fp64 truth below needs the device memory
  gc.collect()
  torch.cuda.empty_cache()
  grads = {k: np.zeros(v.shape) for k, v in w.items()}
  losses = np.zeros(4)
  logits = [[], []]
  for lo in range(0, n, chunk):
    sl = slice(lo, lo + chunk)
    _, l, _, gr, lg = NS.loss_and_grads(rcfg, w, chunk_feeds(f, sl), device=dev, return_logits=True,
                                        fed_ids=[a[sl] for a in ids])
    losses += np.array(l) * chunk / n
    for k in grads:
      grads[k] += gr[k] * chunk / n
    for i in range(2):
      logits[i].append(lg[i].reshape(chunk, T_PRED, -1))
  for k in grads:
    if k.endswith("/W"):
      grads[k] -= cfg.wd * w[k]
  for i in range(2):
    ref = np.concatenate(logits[i])
    err = rel(mine[i], ref)
    srt = np.sort(ref, -1)
    clear = srt[..., -1] - srt[..., -2] > 2 * err * np.abs(ref).max()
    assert err < 1e-4 and (ref.argmax(-1) == ids[i])[clear].all(), (i, err)
  assert np.abs(got - losses).max() < LTOL * np.abs(losses).max(), (got, losses)
  worst = {k: rel(eng_grads[k], grads[k]) for k in sorted(grads)}
  print("emb 128 without scene encoding (gnn %s): losses %.1e, worst gradient errors %s"
        % (use_gnn, np.abs(got - losses).max() / np.abs(losses).max(),
           sorted(worst.items(), key=lambda kv: -kv[1])[:4]))
  bad = {k: v for k, v in worst.items() if v > GTOL}
  assert not bad, bad


def train_golden(name):
  import cases
  import emb_size_cases as EC
  from multiverse_b200 import synthetic
  from oracle import multiverse_ref as R
  over, seed = EC.TRAIN[name]
  over = dict(over, **{k: v for k, v in EC.TRAIN_ARGS.items() if k != "optimizer"})
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  g = np.load(os.path.join(ROOT, "tests", "golden", "refexec_train_emb_%s.npz" % name))
  assert abs(float(g["checksum"]) - cases.checksum(*w.values()) - cases.checksum(f["scene_feat"], f["traj"])) < 1e-6
  return over, cfg, w, f, g


def test_dropin_trainer_step_emb96_equals_reference_execution(dev, monkeypatch):
  """One Trainer.step through the drop-in at --use_scene_enc --use_gnn --emb_size 96 (both decoders at cpad 352) on
  the inputs of tests/golden/refexec_train_emb_scene_enc_emb96.npz: losses, every clipped gradient and the variables
  after Adadelta equal the unmodified reference Model + Trainer's (test_train_options_gpu's check)."""
  from test_train_options_gpu import _dropin_model, check_step_against_reference_execution
  over, cfg, w, f, g = train_golden("scene_enc_emb96")
  dover = dict(use_grids=[True, True], emb_size=96, use_gnn=True, grid_loss_weight=over["grid_loss_weight"],
               grid_reg_loss_weight=over["grid_reg_loss_weight"], wd=over["wd"])
  tf, pred_models, model, args, _, _, _, batch = _dropin_model(monkeypatch, w=w, f=f, n=cfg.batch_size, over=dover,
                                                               train_w_onehot=True, init_lr=over["init_lr"])
  assert set(model.weights()) == set(g["variables"])
  check_step_against_reference_execution("emb96", tf, pred_models, model, args, batch, w, g, "")


def test_train_step_on_train_py_defaults_equals_reference_execution(dev):
  """TrainEngine.loss_and_grads on train.py's own model defaults (emb_size 128, no scene encoder, no attention, three
  grids 36x18 / 18x9 / 9x4) against the reference Model's step (tests/golden/refexec_train_emb_defaults_three_grids.npz):
  losses within 1e-4, every clipped gradient within 2e-4 of its largest element."""
  import cases
  from multiverse_b200 import synthetic
  from multiverse_b200.train_engine import TrainEngine
  over, cfg, w, f, g = train_golden("defaults_three_grids")
  ecfg = synthetic.make_config(is_train=True, **over)
  assert len(ecfg.scene_grids) == 3 and ecfg.emb_size == 128
  eng = TrainEngine(ecfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  feeds = {k: ([up(a) for a in f[k]] if isinstance(f[k], list) else up(f[k]))
           for k in ("scene_feat", "obs_scene", "grid_obs_labels", "grid_obs_regress", "grid_pred_labels",
                     "grid_pred_regress")}
  l, _ = eng.loss_and_grads(feeds)
  torch.cuda.synchronize()
  l = l.cpu().numpy()
  assert np.abs(l - g["pred_grid_loss"]).max() <= 1e-4 * g["pred_grid_loss"].max(), (l, g["pred_grid_loss"])
  worst = {}
  for k in g["variables"]:
    gr = eng.grads[k].double().cpu().numpy() + (over["wd"] * w[k] if k.endswith("/W") else 0.0)
    worst[k] = np.abs(cases.sample(np.clip(gr, -10.0, 10.0), cases.NATIVE_TRAIN_SAMPLE) - g["grad/" + k]).max() / max(
        float(g["grad_absmax/" + k]), 1e-30)
  print("train.py defaults: losses %s vs %s, worst gradient errors %s" % (
      l, g["pred_grid_loss"], sorted(worst.items(), key=lambda kv: -kv[1])[:4]))
  bad = {k: v for k, v in worst.items() if v > 2e-4}
  assert not bad, bad
