# coding=utf-8
"""Every kernel of the inference rollout around the ConvLSTM cell, element by element, at the batch the benchmark
decodes: the K = 20 beam decoder of 512 trajectories on the 36x18 grid (10 240 beam rows per step, f16f8 operands)
and the greedy two-scale decoder of 256 trajectories on 36x18 and 18x9 (and on the 9x16 grid of the published 36x64
scene, whose encoders run the f16f8 pair kernel at that batch); then the feed and post-decode kernels and the
evaluation metrics at that batch.

The unit tests of test_parity_gpu.py run these kernels on a handful of rows, and the at-size rollout tests compare
whole-rollout statistics at a 1e-4 bar.  What only happens at size, or only in the f16f8 format:
  - the graph attention reads its state through a parent row map of a real beam selection (parents repeat and are
    not monotone) and writes the class decoder's f16f8 operands;
  - the regression head and the dense embedding write their embedding as f16f8 x planes; a dropped residual plane
    (about 2^-11 relative) hides under the rollout bar;
  - beam_step selects among 20 x 648 candidates per sample over 12 chained steps, with exact ties across beams;
  - the back-trace, traj_to_grid (about 5 grid-stride passes at 512 x 8 points) and the metrics run over 512
    trajectories, where rare rounding differences become likely.
Every output is compared with a plain fp64 torch (or numpy) reference on the kernel's own inputs, over chunks of
sample rows; values stored in f16f8 operand planes are decoded with ops.operand_values.

Bars (max|diff| / max|ref| per tensor, the suite's existing ones): FTOL 1e-5 for fp32 logits and offsets, F8TOL 2e-5
for values decoded from f16f8 planes (test_gnn_shapes_against_dense_oracle), TIGHT 3e-5 for a cell step, TOL 1e-4 for a
chain of stages (the rollout bar).  Selections (ids, parents, arg-max) are exact wherever the fp64 margin clears the
kernel's error; the fraction of rows kept is asserted and printed.  Metric errors and selections are bit-exact.  The
GPU tests are marked one by one so that the CPU tests run under -m "not gpu"."""
import gc
import math
import os

import numpy as np
import pytest
import torch

import cases
from test_kernels_atsize_gpu import TIGHT, _taps, halo_bits, inner, m_tiles, num_sms, ref_cell, ref_onehot_emb, rel
from test_train_atsize_gpu import CLAMPED, gen, on, ref_emb, ref_gnn, ref_head, ref_onehot, report
from oracle import multiverse_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FTOL = 1e-5      # fp32 logits and offsets
F8TOL = 2e-5     # values decoded from f16f8 operand planes (test_gnn_shapes_against_dense_oracle)
TOL = 1e-4       # a chain of stages (the rollout bar)
HID = 256
E = 32
T_PRED = 12
CHUNK = 128      # sample rows per reference chunk (fp64 im2col of the head at 36x18: 1.5 GB)
SENT = 0x5A      # byte sentinel written into the operand blocks a kernel must not touch
GAMMA = 0.01
LOG_GAMMA = float(np.float32(math.log(GAMMA)))     # the fp32 log(gamma) beam_step receives
C4 = dict(use_grids=[True, False], use_beam_search=True, beam_size=20, diverse_beam=True, diverse_gamma=GAMMA,
          fix_num_timestep=1)
C3 = dict(use_grids=[True, True])
NATIVE = dict(C4, scene_h=36, scene_w=64)         # K = 20 on the native 18x32 grid
NATIVE_C3 = dict(C3, scene_h=36, scene_w=64)      # greedy two-scale on the native 18x32 and 9x16 grids
N_C4, N_C3 = 512, 256


# --------------------------------------------------------------------------- references
def ref_beam_step(lg, sc, first, diverse, log_gamma):
  """fp64 selection of decoder_loop_fn (code/pred_models.py:557-591) on the kernel's inputs: log_softmax + running
  score, + log(gamma) x the stable descending rank inside each beam row (add_div_penalty, :1197-1223), then a stable
  top-B over the B*V candidates (beam 0 only on the first step).  Returns the candidates sorted (descending, ties by
  flat index), their flat indices b * V + v, and each row's log-probs sorted (descending)."""
  n, _, v = lg.shape
  lp = torch.log_softmax(lg.double(), -1) + sc.double()[..., None]
  if first:
    lp = lp[:, :1]
  srt, order = torch.sort(lp, dim=-1, descending=True, stable=True)
  cand = lp
  if diverse:
    rank = torch.empty_like(order)
    rank.scatter_(-1, order, torch.arange(v, device=lg.device).expand_as(order))
    cand = lp + log_gamma * rank.double()
  vals, idx = torch.sort(cand.reshape(n, -1), dim=-1, descending=True, stable=True)
  return vals, idx, srt


def ref_min_ade_fde(pred, gt, gt_len):
  """code/multifuture_eval_trajs.py:41-78 vectorised in numpy: per prediction k and step t < len the error
  sqrt(dx**2 + dy**2) with both squares rounded and then added, as `np.sqrt(np.sum(diff**2, axis=1))` computes it;
  minADE picks the smallest sum over t formed left to right with one rounding per step (Python's `sum` before 3.12,
  which compensates; np.sum would add pairwise), minFDE the smallest last error, first index on ties.  pred [N,K,Tp,2],
  gt [N,G,Tg,2] float32, gt_len [N,G] -> ade_err [N,G,Tg], ade_idx, fde, fde_idx (-1 / 0 where gt_len is 0)."""
  tg = gt.shape[2]
  diff = gt[:, :, None].astype(np.float64) - pred[:, None, :, :tg].astype(np.float64)      # [N,G,K,Tg,2]
  sq = diff ** 2
  d = np.sqrt(sq[..., 0] + sq[..., 1])
  ln = gt_len[:, :, None]
  tot = np.zeros(d.shape[:3])
  for t in range(tg):
    tot = np.where(t < ln, tot + d[..., t], tot)
  last = np.take_along_axis(d, np.maximum(ln - 1, 0)[..., None], -1)[..., 0]
  ade_idx, fde_idx = tot.argmin(-1), last.argmin(-1)
  ade_err = np.take_along_axis(d, ade_idx[:, :, None, None], 2)[:, :, 0] * (np.arange(tg) < gt_len[..., None])
  fde = np.take_along_axis(last, fde_idx[..., None], -1)[..., 0]
  none = gt_len == 0
  ade_idx[none], fde_idx[none], fde[none] = -1, -1, 0.0
  return ade_err, ade_idx.astype(np.int32), fde, fde_idx.astype(np.int32)


class Worst(object):
  """max|diff| / max|ref| of one tensor compared chunk by chunk."""

  def __init__(self):
    self.diff, self.ref = 0.0, 0.0

  def add(self, got, ref):
    ref = ref.double()
    self.diff = max(self.diff, float((got.double() - ref).abs().max()))
    self.ref = max(self.ref, float(ref.abs().max()))

  def value(self):
    return self.diff / max(self.ref, 1e-30)


def ulp32(x):
  return 2.0 ** (math.floor(math.log2(x)) - 23)


# --------------------------------------------------------------------------- CPU: the references against the oracle
def test_min_ade_fde_restatement_matches_the_references_numpy():
  """ref_min_ade_fde equals, bit for bit, the vectors tests/golden/make_golden_metrics.py produced with the
  reference's own get_min inside the loop of code/multifuture_eval_trajs.py (incl. two identical predictions and
  futures of length 0)."""
  g = cases.load_golden(os.path.join(GOLD, "metrics"))
  ade_err, ade_idx, fde, fde_idx = ref_min_ade_fde(g["pred"], g["gt"], g["gt_len"])
  assert np.array_equal(ade_idx, g["ade_idx"]) and np.array_equal(fde_idx, g["fde_idx"])
  assert np.array_equal(ade_err, g["ade_err"]) and np.array_equal(fde, g["fde"])


def test_beam_step_reference_matches_the_oracle():
  """ref_beam_step equals the numpy oracle's log_softmax / add_div_penalty / top_k_sorted in fp64 (flat indices
  exactly, values to 1e-12) and selects the golden ids and parents of test_beam_step_golden, incl. its exact tie
  inside a row."""
  d = cases.beam_case()
  g = cases.load_golden(os.path.join(GOLD, "beam_step"))
  n, b, v = d["logits"].shape
  lg64, sc64 = d["logits"].astype(np.float64), d["score"].astype(np.float64)
  for tag, first, div in (("first", 1, 1), ("mid", 0, 1), ("plain", 0, 0), ("first_plain", 1, 0)):
    vals, idx, _ = ref_beam_step(torch.from_numpy(d["logits"]), torch.from_numpy(d["score"]), first, div,
                                 math.log(GAMMA))
    lp = R.log_softmax(lg64) + sc64[:, :, None]
    if div:
      lp = R.add_div_penalty(lp, GAMMA)
    want_v, want_i = R.top_k_sorted(lp[:, 0] if first else lp.reshape(n, b * v), b)
    assert np.array_equal(idx[:, :b].numpy(), want_i), tag
    assert np.abs(vals[:, :b].numpy() - want_v).max() < 1e-12, tag
    assert np.array_equal((idx[:, :b] % v).numpy(), g[tag + "_ids"]), tag
    assert np.array_equal((idx[:, :b] // v).numpy(), g[tag + "_parents"]), tag


# --------------------------------------------------------------------------- GPU helpers
@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _release_memory():
  """The GPU is shared: every test starts its peak count afresh and gives its memory back when it ends."""
  if torch.cuda.is_available():
    torch.cuda.reset_peak_memory_stats()
  yield
  gc.collect()
  if torch.cuda.is_available():
    torch.cuda.empty_cache()


def beam_decoder_bytes(n, b, h, w, cpad):
  """Device memory of the beam decoder's buffers in ConvRNNEngine.decode_class_beam: two operand buffers and three
  fp32 states of n * b halo-layout rows (38.8 GB for the c4 benchmark)."""
  rows = n * b * (h + 1) * (w + 1)
  return 2 * (2 * rows * cpad * 2) + 3 * rows * HID * 4


def assert_peak_below_the_beam_decoder(n, b, h, w):
  from multiverse_b200 import ops
  peak = torch.cuda.max_memory_allocated()
  cap = beam_decoder_bytes(n, b, h, w, ops.cell_cpad(E))
  assert peak < cap, "peak %.1f GB, the beam decoder itself allocates %.1f GB" % (peak / 1e9, cap / 1e9)
  return peak


def f16f8_bytes(xh, ns, h, w):
  """Raw bytes of an f16f8 operand buffer as [region, ns, h + 1, w + 1, 2 * cpad]: region 0 holds the fp16 values,
  region 1 the two e4m3 planes; in both regions the first 2 * cxp bytes of a row are its x block, the rest its h
  block (the layout ops.operand_values reads)."""
  return xh.view(torch.uint8).view(2, ns, h + 1, w + 1, 2 * xh.shape[2])


def fill_block(xh, ns, h, w, block):
  """SENT into every byte of the x block (block "x") or the h block of the grid cells' rows, in both regions."""
  cxp = xh.shape[2] - HID
  v = f16f8_bytes(xh, ns, h, w)[:, :, :h, :w]
  (v[..., :2 * cxp] if block == "x" else v[..., 2 * cxp:]).fill_(SENT)


def block_intact(xh, ns, h, w, block):
  cxp = xh.shape[2] - HID
  v = f16f8_bytes(xh, ns, h, w)[:, :, :h, :w]
  return bool(((v[..., :2 * cxp] if block == "x" else v[..., 2 * cxp:]) == SENT).all())


def decoded(xh, ns, h, w, sl):
  """ops.operand_values of the sample rows `sl` of an f16f8 operand buffer -> [rows, h, w, cpad].  The two regions
  of those rows are copied into a buffer of their own: decoding 10 240 beam rows at once would take ~35 GB."""
  from multiverse_b200 import ops
  m = sl.stop - sl.start
  part = torch.empty((2, m * (h + 1) * (w + 1), xh.shape[2]), dtype=torch.bfloat16, device=xh.device)
  part.mvb_planes = ops.PLANES_F16F8
  f16f8_bytes(part, m, h, w).copy_(f16f8_bytes(xh, ns, h, w)[:, sl])
  vals, _ = ops.operand_values(part)
  return inner(vals, m, h, w)


def chunks(n, step=CHUNK):
  return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def raw_weights(dev, wts, i, kind):
  from multiverse_b200.engine import _names
  k, b = _names(i)[kind]
  return on(dev, wts[k]), on(dev, wts[b])


def encoded(dev, over, n, seed):
  """ConvRNNEngine of a benchmark config (synthetic.make_config(**over), synthetic.make_weights) and n trajectories of
  synthetic.make_feeds through the scene CNN and both encoders.  Per used scale: the class encoder's c / h (halo
  layout), the scene mean the graph attention reads, the last observed cell, the regression encoder's h and the last
  observed offsets (what the regression decoder embeds first), and the cell variants the scale's encoders ran."""
  from multiverse_b200 import ops, synthetic
  from multiverse_b200.engine import ConvRNNEngine
  cfg = synthetic.make_config(batch_size=n, **over)
  wts = synthetic.make_weights(cfg, seed)
  f = synthetic.make_feeds(cfg, n, seed)
  eng = ConvRNNEngine(cfg, {k: torch.from_numpy(a) for k, a in wts.items()}, dev, 2)
  obs = on(dev, f["obs_scene"])
  obs_t = obs.t().contiguous()
  convs, means = eng.scene_cnn(on(dev, f["scene_feat"]), obs)
  out = dict(cfg=cfg, eng=eng, w=wts)
  for i, (h, w) in enumerate(cfg.scene_grids):
    if not cfg.use_grids[i]:
      continue
    lab_t = on(dev, f["grid_obs_labels"][i]).t().contiguous()
    ops.cell_variants_seen(reset=True)
    c, h32 = eng.encode_class(i, convs[i], obs_t, lab_t, None)
    reg_t = on(dev, f["grid_obs_regress"][i]).transpose(0, 1).contiguous()
    xr = ops.alloc_xh(n, h, w, eng.scales[i].dec_reg.cpad, eng.fast_planes, dev)
    _, hr = eng.encode_reg(i, reg_t, xr)
    torch.cuda.synchronize()
    out[i] = dict(c=c.clone(), h=h32.clone(), mean=means[i], last_label=lab_t[-1].contiguous(), h_reg=hr.clone(),
                  reg_last=reg_t[-1].contiguous(), variants=ops.cell_variants_seen())
  return out


def assert_encoder_variant(enc, i, n):
  """The encoders of scale i ran the f16f8 cell, as the CTA-pair kernel from 2 x SMs M tiles up (single-CTA below)."""
  from multiverse_b200 import ops
  h, w = enc["cfg"].scene_grids[i]
  want = (ops.PLANES_F16F8, m_tiles(n, h, w) >= 2 * num_sms())
  assert enc[i]["variants"] == {want}, "the encoders of %dx%d n%d ran %s, expected %s" % (
      h, w, n, sorted(enc[i]["variants"]), want)
  return "f16f8 %s, %d M tiles" % ("pair" if want[1] else "single-CTA", m_tiles(n, h, w))


def beam_state(dev, over, n, seed):
  """The class decoder of a beam config up to its second selection, launched as ConvRNNEngine.decode_class_beam
  launches it (time 0 once per sample, the first selection, the K-child fan-out, the head, the second selection) on
  the encoder state of n trajectories.  Returns the n * K-row state that step t = 2 reads (c, h32), the logits, ids,
  parents, row map and scores of the second selection, the scene mean and the weights."""
  from multiverse_b200 import ops
  enc = encoded(dev, over, n, seed)
  cfg, e, sw = enc["cfg"], enc[0], enc["eng"].scales[0]
  h, w = cfg.scene_grids[0]
  b, v = cfg.beam_size, h * w
  pk, xf = sw.dec_class, sw.dec_class_xf
  xh1 = ops.alloc_xh(n, h, w, pk.cpad, pk.planes, dev)
  c0, h0 = ops.alloc_state(n, h, w, dev), ops.alloc_state(n, h, w, dev)
  lg0 = torch.empty((n, v), device=dev)
  ops.gnn_attend_fwd(e["h"], e["mean"], xh1, h, w, n)
  ops.cell_fwd_onehot(xh1, pk, xf, e["last_label"], e["c"], c0, h0, None, h, w, n)
  ops.head_class_fwd(h0, sw.head_class, lg0, None, None, None, None, h, w, n)
  sel = lambda: (torch.empty((n, b), device=dev), torch.empty((n, b), dtype=torch.int32, device=dev),
                 torch.empty((n, b), dtype=torch.int32, device=dev), torch.empty((n * b,), dtype=torch.int32, device=dev))
  s1, ids1, par1, rm1 = sel()
  ops.beam_step(lg0.unsqueeze(1).expand(n, b, v).contiguous(), torch.zeros((n, b), device=dev), s1, ids1, par1, rm1,
                n, b, v, True, cfg.fix_num_timestep >= 1, cfg.diverse_beam, cfg.diverse_gamma)
  ops.gnn_attend_fwd(h0, e["mean"], xh1, h, w, n)
  c1, h1 = ops.alloc_state(n * b, h, w, dev), ops.alloc_state(n * b, h, w, dev)
  ops.cell_fwd_onehot_fanout(xh1, pk, xf, ids1.view(-1), c0, c1, h1, h, w, n, b)
  lg2 = torch.empty((n, b, v), device=dev)
  ops.head_class_fwd(h1, sw.head_class, lg2, None, None, None, None, h, w, n * b)
  s2, ids2, par2, rm2 = sel()
  ops.beam_step(lg2, s1, s2, ids2, par2, rm2, n, b, v, False, cfg.fix_num_timestep >= 2, cfg.diverse_beam,
                cfg.diverse_gamma)
  kernel, bias = raw_weights(dev, enc["w"], 0, "dec_class")
  return dict(cfg=cfg, h=h, w=w, n=n, b=b, v=v, c=c1, h32=h1, logits=lg2, scores=s2, ids=ids2, parents=par2,
              row_map=rm2, mean=e["mean"], sw=sw, kernel=kernel, bias=bias)


def clamp_cells(src, mean, h, w, row_map, b, g):
  """Put the cells of test_train_atsize_gpu.CLAMPED under l2_normalize's 1e-12 clamp in what the attention of output
  rows 0..2 reads: their source rows of the state `src` (through the row map) and their sample's scene mean."""
  hv = inner(src, src.shape[0] // ((h + 1) * (w + 1)), h, w)
  for s, fy, fx, mag in CLAMPED:
    y, x = int(fy * (h - 1)), int(fx * (w - 1))
    r = s if row_map is None else int(row_map[s])
    hv[r, y, x] = mag * torch.sign(torch.randn((HID,), generator=g, device=src.device))
    mean[s // b, y, x] = 0.0


def check_gnn(xh, src, mean, ns, h, w, row_map, b):
  """Worst error of the decoded h block of xh against ref_gnn(src[row_map], mean[s // b]), chunk by chunk."""
  cxp = xh.shape[2] - HID
  hv = inner(src, src.shape[0] // ((h + 1) * (w + 1)), h, w)
  err = Worst()
  for sl in chunks(ns):
    rows = torch.arange(sl.start, sl.stop, device=src.device)
    srows = rows if row_map is None else row_map[sl].long()
    err.add(decoded(xh, ns, h, w, sl)[..., cxp:], ref_gnn(hv[srows].double(), mean[rows // b].double()))
  return err.value()


# --------------------------------------------------------------------------- 1. graph attention into f16f8 planes
GNN_CASES = {
    # name: (config, trajectories, scale, beam)
    "c4_beam_36x18": (C4, N_C4, 0, True),
    "c3_36x18": (C3, N_C3, 0, False),
    "c3_18x9": (C3, N_C3, 1, False),
    "native_18x32_k20": (NATIVE, 8, 0, True),
    "native_c3_9x16": (NATIVE_C3, N_C3, 1, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GNN_CASES))
def test_gnn_into_f16f8_planes_at_size(dev, case):
  """gnn_attend_fwd into the h block of the class decoder's f16f8 operands (cpad = cell_cpad(32)): at the beam shape
  with beam = 20 and the row map of a real second selection (the scene mean per sample, s // 20), and with beam = 1
  on the greedy grids; three cells under l2_normalize's clamp.  A byte sentinel in the x block (both regions) must
  survive, the halo must stay zero."""
  from multiverse_b200 import ops
  over, n, i, beam = GNN_CASES[case]
  g = gen(dev, 500 + len(case))
  if beam:
    st = beam_state(dev, over, n, 500 + n)
    h, w, b = st["h"], st["w"], st["b"]
    src, rm, mean = st["h32"], st["row_map"], st["mean"].clone()
    del st
    parents = rm.view(n, b) - (torch.arange(n, device=dev) * b)[:, None]
    order = "; parents out of slot order in %.2f of the samples, repeated in %.2f" % (
        float((parents.diff(1) < 0).any(1).float().mean()), float((parents.sort(1).values.diff(1) == 0).any(1).float().mean()))
    assert bool((parents.diff(1) < 0).any(1).all()), "the row map of the selection is in slot order"
  else:
    enc = encoded(dev, over, n, 510 + i)
    h, w = enc["cfg"].scene_grids[i]
    b, rm, order = 1, None, "; encoders ran " + assert_encoder_variant(enc, i, n)
    src, mean = enc[i]["h"], enc[i]["mean"].clone()
    del enc
  ns = n * b
  clamp_cells(src, mean, h, w, rm, b, g)
  xh = ops.alloc_xh(ns, h, w, ops.cell_cpad(E), ops.PLANES_F16F8, dev)
  fill_block(xh, ns, h, w, "x")
  ops.gnn_attend_fwd(src, mean, xh, h, w, ns, beam=b, row_map=rm)
  assert block_intact(xh, ns, h, w, "x"), "the attention wrote into the x block"
  assert halo_bits(xh, ns, h, w) == 0, "the attention wrote into the zero halo"
  err = check_gnn(xh, src, mean, ns, h, w, rm, b)
  peak = assert_peak_below_the_beam_decoder(N_C4, 20, 36, 18)
  report("gnn f16f8 %s: %d rows of %dx%d, beam %d%s (peak %.1f GB)" % (case, ns, h, w, b, order, peak / 1e9),
         {"h' planes": err})
  assert err < F8TOL


# --------------------------------------------------------------------------- 2. heads and embeddings
@pytest.mark.gpu
def test_class_head_at_beam_rows(dev):
  """head_class_fwd over the 10 240 beam rows of the second selection, no feedback, as decode_class_beam runs it."""
  st = beam_state(dev, C4, N_C4, 520)
  h, w, ns = st["h"], st["w"], st["n"] * st["b"]
  hv = inner(st["h32"], ns, h, w)
  lg = st["logits"].view(ns, h * w)
  err = Worst()
  for sl in chunks(ns):
    err.add(lg[sl], ref_head(hv[sl].double(), st["sw"].head_class.double())[..., 0])
  report("class head, %d beam rows of %dx%d" % (ns, h, w), {"logits": err.value()})
  assert err.value() < FTOL


@pytest.mark.gpu
@pytest.mark.parametrize("over,i", [(C3, 0), (C3, 1), (NATIVE_C3, 1)], ids=["36x18", "18x9", "9x16"])
def test_class_head_ids_and_f16f8_feedback(dev, over, i):
  """head_class_fwd on 256 greedy rows with its arg-max ids and the embedded one-hot of the ids written as f16f8 x
  planes; a sentinel in the h block must survive, the halo must stay zero."""
  from multiverse_b200 import ops
  enc = encoded(dev, over, N_C3, 530)
  h, w = enc["cfg"].scene_grids[i]
  variant = assert_encoder_variant(enc, i, N_C3)
  sw, hs = enc["eng"].scales[i], enc[i]["h"]
  We, be = sw.emb_class
  n = N_C3
  logits = torch.empty((n, h * w), device=dev)
  ids = torch.empty((n,), dtype=torch.int32, device=dev)
  xh = ops.alloc_xh(n, h, w, ops.cell_cpad(E), ops.PLANES_F16F8, dev)
  fill_block(xh, n, h, w, "h")
  ops.head_class_fwd(hs, sw.head_class, logits, ids, We, be, xh, h, w, n)
  ref = ref_head(inner(hs, n, h, w).double(), sw.head_class.double())[..., 0]
  err_abs = float((logits.double() - ref).abs().max())
  srt = ref.sort(-1, descending=True).values
  clear = (srt[:, 0] - srt[:, 1]) > 10 * err_abs
  assert torch.equal(ids.long(), logits.argmax(-1)), "ids are not the arg-max of the kernel's logits"
  assert bool((ids.long() == ref.argmax(-1))[clear].all())
  emb = ref_emb(ref_onehot(ids, h, w), We.double(), be.double())
  errs = {"logits": rel(logits, ref), "one-hot emb planes": rel(decoded(xh, n, h, w, slice(0, n))[..., :E], emb)}
  assert block_intact(xh, n, h, w, "h") and halo_bits(xh, n, h, w) == 0
  report("class head %dx%d, %d rows (encoders ran %s), ids kept %.3f (top-2 gap > 10 x fp32 error)"
         % (h, w, n, variant, float(clear.float().mean())), errs)
  assert float(clear.float().mean()) >= 0.9
  assert errs["logits"] < FTOL and errs["one-hot emb planes"] < F8TOL


REG_CASES = {"c4_36x18": (C4, N_C4, 0), "c3_36x18": (C3, N_C3, 0), "c3_18x9": (C3, N_C3, 1),
             "native_c3_9x16": (NATIVE_C3, N_C3, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(REG_CASES))
def test_reg_head_and_dense_embedding_into_f16f8(dev, case):
  """The regression decoder's feedback in f16f8: head_reg_fwd (offsets, their dense embedding as f16f8 x planes) on
  the regression encoder's h, and emb_dense_fwd of the last observed raw offsets (up to +-1.9e3 px) as decode_reg
  embeds them first.  Sentinels in the h block must survive, the halo must stay zero."""
  from multiverse_b200 import ops
  over, n, i = REG_CASES[case]
  enc = encoded(dev, over, n, 540 + i)
  h, w = enc["cfg"].scene_grids[i]
  variant = assert_encoder_variant(enc, i, n)
  sw, hs, x0 = enc["eng"].scales[i], enc[i]["h_reg"], enc[i]["reg_last"]
  We, be = sw.emb_reg
  cpad = ops.cell_cpad(E)
  offs = torch.empty((n, h * w, 2), device=dev)
  xh = ops.alloc_xh(n, h, w, cpad, ops.PLANES_F16F8, dev)
  fill_block(xh, n, h, w, "h")
  ops.head_reg_fwd(hs, sw.head_reg, offs, We, be, xh, h, w, n)
  ref = ref_head(inner(hs, n, h, w).double(), sw.head_reg.double())
  emb = ref_emb(offs.double().view(n, h, w, 2), We.double(), be.double())
  errs = {"offsets": rel(offs, ref), "dense emb planes": rel(decoded(xh, n, h, w, slice(0, n))[..., :E], emb)}
  assert block_intact(xh, n, h, w, "h") and halo_bits(xh, n, h, w) == 0
  xh0 = ops.alloc_xh(n, h, w, cpad, ops.PLANES_F16F8, dev)
  fill_block(xh0, n, h, w, "h")
  ops.emb_dense_fwd(x0, We, be, xh0, h, w)
  assert float(x0.abs().max()) > 1e3
  got = decoded(xh0, n, h, w, slice(0, n))[..., :E].double()
  ref = ref_emb(x0.double(), We.double(), be.double())
  errs["first input emb planes"] = rel(got, ref)
  errs["first input, beyond fp32 summation"] = float(((got - ref).abs() - fp32_emb_bound(x0, We, be, ref)).clamp(min=0).max()
                                                     / ref.abs().max())
  assert block_intact(xh0, n, h, w, "h") and halo_bits(xh0, n, h, w) == 0
  report("regression feedback %s: %d rows of %dx%d (encoders ran %s)" % (case, n, h, w, variant), errs)
  assert errs["offsets"] < FTOL
  assert errs["dense emb planes"] < F8TOL and errs["first input, beyond fp32 summation"] < F8TOL


def fp32_emb_bound(x, We, be, ref):
  """Element-wise a-priori error of grid_emb of x [n, h, w, P] when its pre-activation (the bias plus 9 P products)
  is summed in fp32, as any fp32 implementation sums it: gamma_{9P} (|be| + sum |x| |We|) times tanh' there, with
  gamma_k = k u / (1 - k u), u = 2^-24.  The raw offsets the regression decoder embeds first reach +-1.9e3 px, so
  this term (~2e-4 where a cell's pre-activation cancels to ~0) exceeds the f16f8 bar on its own."""
  n, h, w, p = x.shape
  k = 9 * p
  gamma = k * 2.0 ** -24 / (1 - k * 2.0 ** -24)
  s = (_taps(x.double().abs()) @ We.double().abs().reshape(k, -1) + be.double().abs()).reshape(ref.shape)
  return gamma * s * (1 - ref * ref + 2 * gamma * s)


# --------------------------------------------------------------------------- 3. beam selection at size
def check_beam_step(lg, s_in, out, first, zero, diverse, b):
  """One beam_step output (score_out, ids, parents, row_map) against ref_beam_step on the same inputs.  Ids and
  parents must be exact on every sample whose fp64 candidates are clear of the kernel's error serr (8 fp32 ulps of
  the largest selected |score|): the gaps between consecutive selected candidates and between the B-th and the best
  unselected one, and with the penalty the gaps between consecutive ranks of a row wherever that rank's candidate is
  among the best B + 1, are 0 (identical inputs: an exact tie in any precision, broken by the flat index) or above
  serr.  Where only the gaps between selected candidates fall inside serr (the near-twin beams of a real rollout,
  see test_rollout_atsize), the SET of selected flat indices must be exact.  Scores must lie within serr of the fp64
  ones (zero after a reset).  Returns (clear mask, set-clear mask, score error, serr)."""
  so, ids, par, rm = out
  n, _, v = lg.shape
  vals, idx, srt = ref_beam_step(lg, s_in, first, diverse, LOG_GAMMA)
  top = vals[:, :b]
  serr = 8 * ulp32(float(top.abs().max()))
  near = lambda gp: (gp > 0) & (gp <= serr)
  gaps = vals[:, :b] - vals[:, 1:b + 1]
  bad_rank = torch.zeros(n, dtype=torch.bool, device=lg.device)
  if diverse:
    cand_r = srt + LOG_GAMMA * torch.arange(v, device=lg.device, dtype=torch.float64)
    rg = srt[..., :-1] - srt[..., 1:]
    bad_rank = ((cand_r[..., :-1] >= vals[:, b, None, None]) & near(rg)).flatten(1).any(-1)
  set_clear = ~(near(gaps[:, -1]) | bad_rank)
  clear = set_clear & ~near(gaps).any(-1)
  assert torch.equal(ids[clear].long(), (idx[:, :b] % v)[clear]), "ids differ on samples clear of the fp32 error"
  assert torch.equal(par[clear].long(), (idx[:, :b] // v)[clear]), "parents differ on samples clear of the fp32 error"
  got_set = (par.long() * v + ids.long()).sort(-1).values
  assert torch.equal(got_set[set_clear], idx[:, :b].sort(-1).values[set_clear]), \
      "the selected candidates differ on samples whose B-th candidate is clear of the fp32 error"
  assert torch.equal(rm.view(n, b).long(), par.long() + (torch.arange(n, device=lg.device) * b)[:, None])
  if zero:
    assert float(so.abs().max()) == 0.0
    s_err = 0.0
  else:
    s_err = float((so.double() - top).abs().max())
    assert s_err <= serr, (s_err, serr)
  return clear, set_clear, s_err, serr


def beam_chain(dev, monkeypatch, n, b, v, diverse, quantised, seed):
  """12 chained beam_step launches with ping-pong scores and the rollout's flags (step 1: first_step, and with the
  penalty zero_scores as fix_num_timestep = 1; later steps: gamma = 0.01 or no penalty), on logits of N(0, 2.5^2)
  (rounded to 0.1: frequent exact ties), all beams equal at step 1 as the rollout tiles them.  Samples 8k + 1 give
  every beam whose running score equals a lower beam's bit for bit that beam's logit row (exact ties across beams);
  samples 8k + 3 repeat every even logit of a row at the next odd index (exact ties inside rows).  Each launch is
  checked (check_beam_step) and must be bit-identical to the rank-count kernel (MVB_BEAM_FULL_RANK=1)."""
  from multiverse_b200 import ops
  g = gen(dev, seed)
  scores = [torch.zeros((n, b), device=dev) for _ in range(2)]
  twins = (torch.arange(n, device=dev) % 8 == 1)[:, None, None]
  inrow = torch.arange(n, device=dev) % 8 == 3
  steps = dict(ids=[], parents=[], logits=[], kept=[], s_err=[], serr=[])
  for t in range(1, T_PRED + 1):
    lg = torch.randn((n, b, v), generator=g, device=dev) * 2.5
    if quantised:
      lg = torch.round(lg * 10) / 10
    lg[inrow, :, 1::2] = lg[inrow, :, 0::2]
    s_in, s_out = scores[(t - 1) % 2], scores[t % 2]
    if t == 1:
      lg = lg[:, :1].expand(n, b, v).contiguous()
    else:
      same = (s_in[:, :, None] == s_in[:, None, :]).float().argmax(-1)       # lowest beam with the same score
      lg = torch.where(twins, lg.gather(1, same[..., None].expand(n, b, v)), lg).contiguous()
    first, zero = t == 1, diverse and t == 1
    outs = {}
    for full in ("1", "0"):
      monkeypatch.setenv("MVB_BEAM_FULL_RANK", full)
      o = (torch.empty((n, b), device=dev), torch.empty((n, b), dtype=torch.int32, device=dev),
           torch.empty((n, b), dtype=torch.int32, device=dev), torch.empty((n * b,), dtype=torch.int32, device=dev))
      ops.beam_step(lg, s_in, o[0], o[1], o[2], o[3], n, b, v, first, zero, diverse, GAMMA)
      outs[full] = o
    for a, c in zip(outs["0"], outs["1"]):
      assert torch.equal(a, c), "step %d: the top-B kernel differs from the rank-count kernel" % t
    clear, _, s_err, serr = check_beam_step(lg, s_in, outs["0"], first, zero, diverse, b)
    s_out.copy_(outs["0"][0])
    steps["ids"].append(outs["0"][1])
    steps["parents"].append(outs["0"][2])
    steps["logits"].append(lg)
    steps["kept"].append(float(clear.float().mean()))
    steps["s_err"].append(s_err)
    steps["serr"].append(serr)
  monkeypatch.setenv("MVB_BEAM_FULL_RANK", "0")
  for k in ("ids", "parents", "logits"):
    steps[k] = torch.stack(steps[k])
  return steps


BEAM_CASES = {
    # name: (n, b, v, diverse, quantised)
    "diverse_512x20x648": (N_C4, 20, 648, True, False),
    "diverse_32x20x576": (32, 20, 576, True, False),
    "plain_512x20x648": (N_C4, 20, 648, False, False),
    "quantised_diverse_512x20x648": (N_C4, 20, 648, True, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(BEAM_CASES))
def test_beam_step_chained_at_size(dev, monkeypatch, case):
  n, b, v, diverse, quantised = BEAM_CASES[case]
  st = beam_chain(dev, monkeypatch, n, b, v, diverse, quantised, 550 + len(case))
  kept = float(np.mean(st["kept"]))
  report("beam_step %s, 12 steps: samples kept %.3f (worst step %.3f)" % (case, kept, min(st["kept"])),
         {"score err (worst step)": max(st["s_err"]), "fp32 error bound": max(st["serr"])})
  assert kept >= 0.8 and min(st["kept"]) >= 0.5


# --------------------------------------------------------------------------- 4. back-trace at size
@pytest.mark.gpu
def test_beam_backtrace_at_size(dev, monkeypatch):
  """beam_backtrace on (Tp 12, N 512, B 20, V 648) with the ids, parents and logits of the chained diverse steps,
  bit-exact against the literal loop of code/pred_models.py:722-764 restated with torch gathers (the logits gathered
  with the parents before they advance, :738 before :749)."""
  from multiverse_b200 import ops
  n, b, v, _, _ = BEAM_CASES["diverse_512x20x648"]
  st = beam_chain(dev, monkeypatch, n, b, v, True, False, 560)
  ids, par, lg = st["ids"], st["parents"], st["logits"]
  out_ids = torch.full((n, b, T_PRED), -7, dtype=torch.int32, device=dev)
  out_lg = torch.full((n, b, T_PRED, v), float("nan"), device=dev)
  ops.beam_backtrace(ids, par, lg, out_ids, out_lg)
  rows = torch.arange(n, device=dev)[:, None]
  p = torch.arange(b, device=dev).expand(n, b)
  for tau in range(T_PRED - 1, -1, -1):
    assert torch.equal(out_ids[:, :, tau], ids[tau][rows, p]), tau
    assert torch.equal(out_lg[:, :, tau], lg[tau][rows, p]), tau
    p = par[tau][rows, p].long()
  moved = float((out_ids != ids.permute(1, 2, 0)).float().mean())
  print("backtrace (12, %d, %d, %d): bit-exact; %.2f of the ids differ from the per-step slot order" % (n, b, v, moved))
  assert moved > 0.1


# --------------------------------------------------------------------------- 5. one decode step chained at size
@pytest.mark.gpu
def test_decode_step_chained_at_beam_size(dev, monkeypatch):
  """Step t = 2 of the c4 beam decoder on its own buffers and shapes (10 240 rows of 36x18): gnn_attend_fwd (f16f8,
  row map) -> cell_fwd_onehot (f16f8 pair kernel, x-fold, row map, h' written over the state the attention read, as
  decode_class_beam does) -> head_class_fwd -> beam_step.  Each stage against its fp64 reference fed the kernel's
  previous stage - the cell reading the attention's f16f8 output is the real consumer of that format; then the
  whole fp64 chain from the step's inputs on the 20 rows of every 16th sample (rows are independent:
  test_full_size_batch_is_its_shards)."""
  from multiverse_b200 import ops
  st = beam_state(dev, C4, N_C4, 570)
  h, w, n, b, v = st["h"], st["w"], st["n"], st["b"], st["v"]
  ns = n * b
  sw, rm, ids = st["sw"], st["row_map"], st["ids"].view(-1)
  We, be = sw.emb_class
  h32, c_in, mean = st["h32"], st["c"], st["mean"]
  pk, xf = sw.dec_class, sw.dec_class_xf
  # the inputs of the whole-chain check: every 16th sample's rows (its row map stays inside the sample)
  picked = torch.arange(0, n, 16, device=dev)
  prow = (picked[:, None] * b + torch.arange(b, device=dev)[None]).reshape(-1)
  h_pick, c_pick = inner(h32, ns, h, w)[prow].clone(), inner(c_in, ns, h, w)[prow].clone()
  # stage 1: attention
  xh = ops.alloc_xh(ns, h, w, pk.cpad, pk.planes, dev)
  ops.gnn_attend_fwd(h32, mean, xh, h, w, ns, beam=b, row_map=rm)
  errs = {"gnn h' planes": check_gnn(xh, h32, mean, ns, h, w, rm, b)}
  # stage 2: the cell
  c_out = ops.alloc_state(ns, h, w, dev)
  ops.cell_fwd_onehot(xh, pk, xf, ids, c_in, c_out, h32, None, h, w, ns, row_map=rm)
  assert ops.cell_last_variant() == ops.PLANES_F16F8 * 2 + 1, "the f16f8 pair cell kernel did not run"
  ec, eh = Worst(), Worst()
  cv = inner(c_in, ns, h, w)
  for sl in chunks(ns):
    ref = ref_cell(ref_onehot_emb(ids[sl], h, w, We, be), decoded(xh, ns, h, w, sl)[..., pk.cxp:],
                   cv[rm[sl].long()], st["kernel"], st["bias"])
    ec.add(inner(c_out, ns, h, w)[sl], ref["c"])
    eh.add(inner(h32, ns, h, w)[sl], ref["h"])
  errs.update({"cell c'": ec.value(), "cell h'": eh.value()})
  del xh
  # stage 3: the head
  logits = torch.empty((n, b, v), device=dev)
  ops.head_class_fwd(h32, sw.head_class, logits, None, None, None, None, h, w, ns)
  el = Worst()
  hv = inner(h32, ns, h, w)
  for sl in chunks(ns):
    el.add(logits.view(ns, v)[sl], ref_head(hv[sl].double(), sw.head_class.double())[..., 0])
  errs["logits"] = el.value()
  # stage 4: the selection
  o = (torch.empty((n, b), device=dev), torch.empty((n, b), dtype=torch.int32, device=dev),
       torch.empty((n, b), dtype=torch.int32, device=dev), torch.empty((ns,), dtype=torch.int32, device=dev))
  monkeypatch.setenv("MVB_BEAM_FULL_RANK", "0")
  ops.beam_step(logits, st["scores"], o[0], o[1], o[2], o[3], n, b, v, False, False, True, GAMMA)
  clear, set_clear, s_err, _ = check_beam_step(logits, st["scores"], o, False, False, True, b)
  errs["scores"] = s_err
  # the whole fp64 chain on the picked samples
  parent = rm[prow].long() - (prow // b) * b
  src = torch.arange(picked.numel(), device=dev).repeat_interleave(b) * b + parent     # row of h_pick / c_pick
  hg = ref_gnn(h_pick[src].double(), mean[picked].double().repeat_interleave(b, 0))
  ref = ref_cell(ref_onehot_emb(ids[prow], h, w, We, be), hg, c_pick[src], st["kernel"], st["bias"])
  chain = {"chain c'": rel(inner(c_out, ns, h, w)[prow], ref["c"]), "chain h'": rel(hv[prow], ref["h"]),
           "chain logits": rel(logits.view(ns, v)[prow], ref_head(ref["h"], sw.head_class.double())[..., 0])}
  errs.update(chain)
  peak = assert_peak_below_the_beam_decoder(n, b, h, w)
  report("decode step t=2, %d rows of %dx%d, selection: ids exact-checked in %.3f of the samples, sets in %.3f (peak "
         "%.1f GB)" % (ns, h, w, float(clear.float().mean()), float(set_clear.float().mean()), peak / 1e9), errs)
  assert float(set_clear.float().mean()) >= 0.75
  assert errs["gnn h' planes"] < F8TOL
  assert errs["cell c'"] < TIGHT and errs["cell h'"] < TIGHT
  assert errs["logits"] < FTOL
  for k, e in chain.items():
    assert e < TOL, (k, e)


# --------------------------------------------------------------------------- 6. feeds and post-decode
@pytest.mark.gpu
def test_traj_to_grid_at_size(dev):
  """traj_to_grid for 512 x 8 points (about 5 grid-stride passes at 36x18) on both grids, bit-identical to the
  oracle's get_grid_input (R.traj_to_grid): labels and every cell's offset, incl. the frame origin, the far corner
  and exact cell borders spread over many blocks.  The outputs start as sentinels."""
  from multiverse_b200 import ops
  cfg = R.default_config()
  n, t = N_C4, 8
  rng = np.random.default_rng(580)
  traj = rng.uniform(0, [cfg.video_w, cfg.video_h], size=(n, t, 2))
  traj[0, 0], traj[n - 1, t - 1] = [0.0, 0.0], [cfg.video_w, cfg.video_h]
  fh, fw = cfg.scene_grids[0]
  for k, p in enumerate(range(3, n * t, 37)):       # borders of the fine grid (every 2nd also of the coarse one)
    traj.reshape(-1, 2)[p] = [cfg.video_w * 1.0 / fw * (k % (fw + 1)), cfg.video_h * 1.0 / fh * (k % (fh + 1))]
  want_l, want_r = R.traj_to_grid(cfg, traj.reshape(-1, 2))
  centers = R.grid_centers(cfg)
  for i, (h, w) in enumerate(cfg.scene_grids):
    lab = torch.full((n, t), -7, dtype=torch.int32, device=dev)
    reg = torch.full((n, t, h, w, 2), 1234.5, device=dev)
    ops.traj_to_grid(on(dev, traj), on(dev, centers[i].reshape(h * w, 2)), cfg.video_h * 1.0 / h,
                     cfg.video_w * 1.0 / w, lab, reg, h, w)
    assert np.array_equal(lab.cpu().numpy().reshape(-1), want_l[i]), (h, w)
    assert np.array_equal(reg.cpu().numpy().reshape(n * t, h, w, 2), want_r[i]), (h, w)
  print("traj_to_grid: %d points bit-identical on %s" % (n * t, cfg.scene_grids))


@pytest.mark.gpu
def test_decode_trajectories_at_size(dev):
  """decode_trajectories on (512, 20, 12) beam ids of 36x18 (every corner cell among them) and offsets of +-600 px:
  bit-exact against centre + offset added in float32 by torch."""
  from multiverse_b200 import ops
  n, k, tp = N_C4, 20, T_PRED
  h, w = 36, 18
  v = h * w
  g = gen(dev, 590)
  ids = torch.randint(0, v, (n, k, tp), generator=g, device=dev, dtype=torch.int32)
  for j, c in enumerate((0, w - 1, v - w, v - 1)):
    ids.view(-1)[j::97] = c
  offs = torch.randn((tp, n, v, 2), generator=g, device=dev) * 200
  centers = on(dev, R.grid_centers(R.default_config())[0].reshape(v, 2).astype(np.float32))
  out = torch.full((n, k, tp, 2), float("nan"), device=dev)
  ops.decode_trajectories(ids, offs, centers, out)
  il = ids.long()
  t_idx = torch.arange(tp, device=dev)[None, None].expand(n, k, tp)
  n_idx = torch.arange(n, device=dev)[:, None, None].expand(n, k, tp)
  want = centers[il] + offs[t_idx, n_idx, il]
  assert torch.equal(out, want)


# --------------------------------------------------------------------------- 7. metrics at size
@pytest.mark.gpu
def test_min_ade_fde_at_size(dev):
  """min_ade_fde at N 512, K 20, Tp 12, G 4 with lengths from {0, 1, 5, 12}, predictions and futures drawn
  independently over the 1920x1080 frame (coordinates of unlike magnitude: the case in which a contracted
  dx*dx + dy*dy differs from numpy's rounding), some below 1 px, and duplicated best predictions (the first index
  must win): errors and selections bit-exact against ref_min_ade_fde."""
  from multiverse_b200 import ops
  n, k, tp, gg = N_C4, 20, T_PRED, 4
  rng = np.random.default_rng(600)
  pred = rng.uniform(0, [1920, 1080], size=(n, k, tp, 2)).astype(np.float32)
  gt = rng.uniform(0, [1920, 1080], size=(n, gg, tp, 2)).astype(np.float32)
  pred[::5, :, :, 1] = rng.uniform(0, 1, size=pred[::5, :, :, 1].shape)
  gt[1::5, :, 2:4] = rng.uniform(0, 1, size=gt[1::5, :, 2:4].shape)
  dup = np.arange(5, n, 16)
  pred[dup, 11] = pred[dup, 4]                                 # prediction 4 is the best for future 0, twice
  gt[dup, 0] = pred[dup, 4] + rng.normal(0, 0.5, size=gt[dup, 0].shape).astype(np.float32)
  gt_len = rng.choice([0, 1, 5, 12], size=(n, gg)).astype(np.int32)
  gt_len[dup, 0] = 12
  want = ref_min_ade_fde(pred, gt, gt_len)
  got = [a.cpu().numpy() for a in ops.min_ade_fde(on(dev, pred), on(dev, gt), on(dev, gt_len))]
  assert np.all(want[1][dup, 0] == 4) and np.all(want[3][dup, 0] == 4)
  names = ("ade_err", "ade_idx", "fde", "fde_idx")
  diff = {nm: int((a != b).sum()) for nm, a, b in zip(names, got, want)}
  print("min_ade_fde %d x %d futures, K %d: elements that differ from numpy %s" % (n, gg, k, diff))
  for nm, a, b in zip(names, got, want):
    assert np.array_equal(a, b), (nm, diff[nm])


@pytest.mark.gpu
def test_beam_nll_at_size(dev):
  """beam_nll at N 512, K 20, Tp 12, V 648 over J 12 evaluated steps, one of them (12) past the rollout (count 0),
  absent futures (-1) and one step of one trajectory with none present, against the fp64 beam mixture at 1e-5 of
  the largest nll; counts exact."""
  from multiverse_b200 import ops
  n, k, tp, v, gg = N_C4, 20, T_PRED, 648, 4
  g = gen(dev, 610)
  logits = torch.randn((n, k, tp, v), generator=g, device=dev) * 3
  logprobs = -torch.randn((n, k), generator=g, device=dev).abs() * 4
  steps = torch.tensor(list(range(11)) + [12], dtype=torch.int32, device=dev)
  j = steps.numel()
  gt_idx = torch.randint(0, v, (n, j, gg), generator=g, device=dev, dtype=torch.int32)
  gt_idx[torch.rand((n, j, gg), generator=g, device=dev) < 0.3] = -1
  gt_idx[7, 3] = -1
  nll, cnt = ops.beam_nll(logits, logprobs, gt_idx, steps)
  wb = torch.softmax(logprobs.double(), -1)
  present = gt_idx >= 0
  want_cnt = present.sum(-1).int()
  want_cnt[:, steps >= tp] = 0
  want = torch.zeros((n, j), dtype=torch.float64, device=dev)
  for jj in range(j):
    t = int(steps[jj])
    if t >= tp:
      continue
    p = torch.einsum("nk,nkv->nv", wb, torch.softmax(logits[:, :, t].double(), -1))
    pg = p.gather(1, gt_idx[:, jj].clamp(min=0).long())
    terms = torch.where(present[:, jj], -torch.log(pg + np.finfo(np.float64).eps), torch.zeros_like(pg))
    want[:, jj] = terms.sum(-1) / want_cnt[:, jj].clamp(min=1)
  assert torch.equal(cnt, want_cnt) and int(cnt[7, 3]) == 0 and not bool(cnt[:, -1].any())
  err = float((nll - want).abs().max()) / float(want.abs().max())
  report("beam_nll %d x %d steps, K %d, V %d" % (n, j, k, v), {"nll": err})
  assert err < 1e-5
