# coding=utf-8
"""The fused ConvLSTM cell and the backward GEMMs of the training step, element by element, at the sizes and launch
variants the product runs.

The unit tests of test_parity_gpu.py / test_train_gpu.py stop at 300 halo rows: one tile per CTA, the single-CTA cell
kernel only.  Which kernel runs, and how many tiles each CTA loops over, depends on the size of the launch:
  - the cell runs its CTA-pair kernel (two CTAs of a cluster share every weight tile by TMA multicast) from
    2 x (number of SMs) M tiles of 128 rows up; with an odd count, rank 1 of the last pair owns a tile wholly past R;
  - grids of 31 columns and more leave room for three weight slots instead of four; W = 62 fills the A stage (256 rows);
  - cell_dgrad loops over up to 11 tiles per CTA, cell_wgrad_direct splits K (the rows) over 5 or 2 fp32 slabs.
Here every output is compared on the full tensors with an fp64 reference computed by torch on the same device
(ref_cell / ref_cell_grads: no multiverse_b200 kernel involved), which the CPU test of this file pins to the oracle.

Bars: TIGHT (3e-5) for the forward, GTOL (2e-4) for the gradients, as in the unit tests: max|diff| / max|ref| per
tensor.  The GPU tests are marked one by one so that the CPU test runs under -m "not gpu"."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from oracle import multiverse_ref as R
from oracle import multiverse_ref_torch as RT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
TIGHT = 3e-5     # forward: what the P=2 / f16f8 operand schemes deliver per kernel (test_parity_gpu.py)
GTOL = 2e-4      # gradients (test_train_gpu.py)
HID = 256
BLOCK_M = 128    # rows of a cell / dgrad M tile
CHUNK_ELEMS = 1 << 25      # fp64 elements of one chunk's im2col matrix in the reference (256 MB)
# packed column n = tile * 256 + gate * 64 + j of the kernels' [R, 1024] gate buffers -> TF column gate * 256 + channel
PACKED = [g * HID + t * 64 + j for t in range(4) for g in range(4) for j in range(64)]
SENTINEL = 1234.5


# --------------------------------------------------------------------------- fp64 reference (plain torch)
def _taps(a):
  """[n, h, w, C] -> [n*h*w, 9*C]: the 3x3 SAME neighbourhood of every cell, tap-major (tap = 3 dy + dx), zero
  outside the grid: the rows of the convolution's im2col matrix."""
  n, h, w, c = a.shape
  p = F.pad(a, (0, 0, 1, 1, 1, 1))
  return torch.cat([p[:, dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)], -1).reshape(n * h * w, 9 * c)


def _untaps(d, n, h, w):
  """Adjoint of _taps: [n*h*w, 9*C] -> [n, h, w, C]."""
  c = d.shape[1] // 9
  d = d.reshape(n, h, w, 9, c)
  p = d.new_zeros((n, h + 2, w + 2, c))
  for t in range(9):
    p[:, t // 3:t // 3 + h, t % 3:t % 3 + w] += d[:, :, :, t]
  return p[:, 1:h + 1, 1:w + 1]


def _chunks(n, h, w, c, chunk):
  step = chunk or max(1, CHUNK_ELEMS // (h * w * 9 * c))
  return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def _step(x, h, c, W, b, sl, row_map):
  """Gate activations and new state of the sample rows `sl`, fp64, rows flattened: (im2col, a_i, a_j, a_f, a_o,
  c_prev, c')."""
  cols = _taps(torch.cat([x[sl], h[sl]], -1).double())
  g = cols @ W + b
  gi, gj, gf, go = g.split(HID, -1)
  ai, aj, af, ao = torch.sigmoid(gi), torch.tanh(gj), torch.sigmoid(gf + 1.0), torch.sigmoid(go)
  if c is None:
    cp = torch.zeros_like(ai)
  else:
    cp = (c[sl] if row_map is None else c[row_map[sl].long()]).double().reshape(-1, HID)
  return cols, ai, aj, af, ao, cp, af * cp + ai * aj


def ref_cell(x, h, c, kernel, bias, row_map=None, chunk=None):
  """One ConvLSTM step in fp64 (ConvLSTMCell.call: conv3x3 SAME of concat([x, h]) + bias -> i, j, f, o,
  forget bias 1), over chunks of sample rows.  x [n,H,W,cx], h [n,H,W,256], c [n_src,H,W,256] or None (zero state),
  row_map [n]: sample row of c that sample row s reads.  Returns fp64 c', h' [n,H,W,256] and the activated gates
  [n,H,W,1024] (TF column order i, j, f, o)."""
  n, hh, ww, cx = x.shape
  W = kernel.double().reshape(9 * (cx + HID), 4 * HID)
  b = bias.double()
  cs, hs, gs = [], [], []
  for sl in _chunks(n, hh, ww, cx + HID, chunk):
    _, ai, aj, af, ao, _, cn = _step(x, h, c, W, b, sl, row_map)
    cs.append(cn)
    hs.append(torch.tanh(cn) * ao)
    gs.append(torch.cat([ai, aj, af, ao], -1))
  return dict(c=torch.cat(cs).reshape(n, hh, ww, HID), h=torch.cat(hs).reshape(n, hh, ww, HID),
              gates=torch.cat(gs).reshape(n, hh, ww, 4 * HID))


def ref_cell_grads(x, h, c, kernel, bias, dh, dc, chunk=None):
  """Backward of ref_cell for the loss sum(dh * h') + sum(dc * c'), fp64: dc_prev, dx, dh_prev [n,H,W,.],
  dW [3,3,cx+256,1024], db [1024].  dW and db are sums over the sample rows, accumulated chunk by chunk."""
  n, hh, ww, cx = x.shape
  W = kernel.double().reshape(9 * (cx + HID), 4 * HID)
  b = bias.double()
  dW = torch.zeros_like(W)
  db = torch.zeros_like(b)
  dcp, dxs, dhs = [], [], []
  for sl in _chunks(n, hh, ww, cx + HID, chunk):
    cols, ai, aj, af, ao, cp, cn = _step(x, h, c, W, b, sl, None)
    th = torch.tanh(cn)
    dhc, dcc = dh[sl].double().reshape(-1, HID), dc[sl].double().reshape(-1, HID)
    dct = dcc + dhc * ao * (1 - th * th)
    dG = torch.cat([dct * aj * ai * (1 - ai), dct * ai * (1 - aj * aj), dct * cp * af * (1 - af),
                    dhc * th * ao * (1 - ao)], -1)
    dcp.append(dct * af)
    dW += cols.t() @ dG
    db += dG.sum(0)
    dxh = _untaps(dG @ W.t(), sl.stop - sl.start, hh, ww)
    dxs.append(dxh[..., :cx])
    dhs.append(dxh[..., cx:])
  return dict(dc_prev=torch.cat(dcp).reshape(n, hh, ww, HID), dx=torch.cat(dxs), dh_prev=torch.cat(dhs),
              dW=dW.reshape(3, 3, cx + HID, 4 * HID), db=db)


def ref_onehot_emb(ids, h, w, We, be):
  """grid_emb(one_hot(ids)) in fp64: tanh(conv3x3 SAME of the one-hot map + be) -> [n, h, w, E]."""
  n = ids.shape[0]
  oh = torch.zeros((n, h * w), dtype=torch.float64, device=ids.device)
  oh[torch.arange(n, device=ids.device), ids.long()] = 1.0
  e = We.shape[-1]
  return torch.tanh(_taps(oh.reshape(n, h, w, 1)) @ We.double().reshape(9, e) + be.double()).reshape(n, h, w, e)


def rel(a, b):
  a = torch.as_tensor(a).double()
  b = torch.as_tensor(b).to(a.device).double()
  return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# --------------------------------------------------------------------------- CPU: the reference against the oracle
@pytest.mark.parametrize("name", sorted(cases.CELL_CASES))
def test_reference_helpers_match_the_oracle(name):
  """ref_cell / ref_cell_grads (the at-size reference of the GPU tests below) equal the numpy oracle's cell and torch
  autograd through the oracle's torch restatement to 1e-12, in one chunk and chunk by chunk (one sample row each),
  with and without a row map."""
  d = cases.cell_case(name)
  ns, h, w, cx = d["x"].shape
  t = {k: torch.from_numpy(v) for k, v in d.items()}
  q = {k: v.astype(np.float64) for k, v in d.items()}
  rng = np.random.default_rng(5)
  dh = rng.standard_normal((ns, h, w, HID))
  dc = rng.standard_normal((ns, h, w, HID))
  perm = rng.integers(0, ns, size=ns).astype(np.int32)
  c_o, h_o = R.convlstm_cell(q["x"], q["c"], q["h"], q["kernel"], q["biases"])
  c_m, h_m = R.convlstm_cell(q["x"], q["c"][perm], q["h"], q["kernel"], q["biases"])
  pre = RT.conv2d_same(torch.cat([t["x"], t["h"]], -1).double(), t["kernel"].double()) + t["biases"].double()
  gi, gj, gf, go = pre.split(HID, -1)
  gates = torch.cat([torch.sigmoid(gi), torch.tanh(gj), torch.sigmoid(gf + 1.0), torch.sigmoid(go)], -1)
  a = {k: v.double().requires_grad_(True) for k, v in t.items()}
  c1, h1 = RT.convlstm_cell(a["x"], a["c"], a["h"], a["kernel"], a["biases"])
  ((h1 * torch.from_numpy(dh)).sum() + (c1 * torch.from_numpy(dc)).sum()).backward()
  for chunk in (None, 1):
    ref = ref_cell(t["x"], t["h"], t["c"], t["kernel"], t["biases"], chunk=chunk)
    assert rel(ref["c"], c_o) < 1e-12 and rel(ref["h"], h_o) < 1e-12
    assert rel(ref["gates"], gates) < 1e-12
    ref = ref_cell(t["x"], t["h"], t["c"], t["kernel"], t["biases"], row_map=torch.from_numpy(perm), chunk=chunk)
    assert rel(ref["c"], c_m) < 1e-12 and rel(ref["h"], h_m) < 1e-12
    gr = ref_cell_grads(t["x"], t["h"], t["c"], t["kernel"], t["biases"], torch.from_numpy(dh), torch.from_numpy(dc),
                        chunk=chunk)
    for k, want in (("dc_prev", a["c"]), ("dx", a["x"]), ("dh_prev", a["h"]), ("dW", a["kernel"]),
                    ("db", a["biases"])):
      assert gr[k].shape == want.shape and rel(gr[k], want.grad) < 1e-12, k


# --------------------------------------------------------------------------- GPU helpers
@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def num_sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def halo_rows(ns, h, w):
  return ns * (h + 1) * (w + 1)


def m_tiles(ns, h, w):
  return -(-halo_rows(ns, h, w) // BLOCK_M)


def pair_ns(h, w, odd):
  """Fewest sample rows of an h x w grid for which the cell runs its CTA-pair kernel (at least 2 M tiles per SM), with
  an odd (the last pair's rank 1 owns a tile wholly past R) or even number of M tiles, and R not a multiple of 128."""
  ns = 1
  while m_tiles(ns, h, w) < 2 * num_sms() or m_tiles(ns, h, w) % 2 != int(odd) or halo_rows(ns, h, w) % BLOCK_M == 0:
    ns += 1
  return ns


def single_cta_max_size():
  """(ns, h, w) of a product grid with exactly 2 * SMs - 1 M tiles (the largest single-CTA launch: ~8 work items per
  CTA), or the largest single-CTA launch on 36x18 if no grid hits it exactly."""
  target = 2 * num_sms() - 1
  for h, w in ((36, 18), (18, 9), (18, 32)):
    for ns in range(1, target * BLOCK_M // halo_rows(1, h, w) + 2):
      if m_tiles(ns, h, w) == target:
        return ns, h, w
  return max(ns for ns in range(1, target * 2) if m_tiles(ns, 36, 18) <= target), 36, 18


def inner(t, ns, h, w):
  """[R, C] halo-layout rows -> [ns, h, w, C] view of the grid cells."""
  return t.view(ns, h + 1, w + 1, -1)[:, :h, :w]


def to_halo(a):
  """[ns, h, w, C] -> fp32 [R, C] in the halo layout (zero halo)."""
  ns, h, w, c = a.shape
  t = torch.zeros((ns, h + 1, w + 1, c), dtype=torch.float32, device=a.device)
  t[:, :h, :w] = a
  return t.view(-1, c)


def halo_bits(t, ns, h, w):
  """Number of non-zero bit patterns in the halo row / column of the buffer t, whose rows are the R halo-layout rows
  (leading plane dimension allowed).  f16f8 operand buffers are checked in both of their regions."""
  from multiverse_b200 import ops
  if t.dtype == torch.bfloat16 and ops.planes_of(t) == ops.PLANES_F16F8:
    raw = t.view(torch.uint8).reshape(-1)
    nel = t.shape[1] * t.shape[2]
    views = [raw[:2 * nel].view(torch.int16).view(1, ns, h + 1, w + 1, -1),
             raw[2 * nel:].view(torch.int8).view(1, ns, h + 1, w + 1, -1)]
  else:
    bits = {4: torch.int32, 2: torch.int16}[t.element_size()]
    views = [t.view(bits).view(-1, ns, h + 1, w + 1, t.shape[-1])]
  return sum(int(v[:, :, h].ne(0).sum()) + int(v[:, :, :, w].ne(0).sum()) for v in views)


def cell_inputs(dev, ns, h, w, cx, seed, x_scale=1.0):
  """Seeded cell inputs generated on the device (the cases.cell_case distributions): Glorot-uniform kernel."""
  g = torch.Generator(device=dev)
  g.manual_seed(seed)
  lim = math.sqrt(6.0 / (9 * (cx + HID) + 9 * 4 * HID))
  r = lambda *s: torch.randn(s, generator=g, device=dev)
  return dict(kernel=(torch.rand((3, 3, cx + HID, 4 * HID), generator=g, device=dev) * 2 - 1) * lim,
              bias=r(4 * HID) * 0.1, x=r(ns, h, w, cx) * x_scale, h=torch.tanh(r(ns, h, w, HID)), c=r(ns, h, w, HID))


def variant_name(v):
  return "%s %s" % ("f16f8" if v // 2 == 16 else "P=%d" % (v // 2), "pair" if v % 2 else "single-CTA")


def check_fwd(tag, ns, h, w, out, ref, planes, pair, gemm_ns=None):
  """Every check of a forward case: the kernel variant, c' / h' (and the stored gates) against the fp64 reference,
  the next step's operand planes against h', and the halo of every output buffer.  gemm_ns: sample rows of the GEMM
  launch when they differ from the output's (fan-out)."""
  from multiverse_b200 import ops
  want = planes * 2 + int(pair)
  assert out["variant"] == want, "%s: ran %s, expected %s" % (tag, variant_name(out["variant"]), variant_name(want))
  errs = {"c": rel(inner(out["c"], ns, h, w), ref["c"]), "h": rel(inner(out["h"], ns, h, w), ref["h"])}
  if out.get("gates") is not None:
    errs["gates"] = rel(inner(out["gates"], ns, h, w), ref["gates"][..., PACKED])
  ho = inner(out["h"], ns, h, w)
  xh2 = out.get("xh2")
  if xh2 is not None:
    vals, e0 = ops.operand_values(xh2)
    cxp = xh2.shape[2] - HID
    errs["planes-h'"] = float((inner(vals[:, cxp:], ns, h, w) - ho).abs().max())
    assert float(vals[:, :cxp].abs().max()) == 0.0, "%s: the kernel wrote into the x block of the next operands" % tag
    if e0 is not None:      # the e4m3 copy of a0 carries 4 significant bits of it
      a0 = vals[:, cxp:]
      assert float((e0[:, cxp:] - a0).abs().max()) <= 2.0 ** -4 * float(a0.abs().max()) + 2.0 ** -9
  print("%s: %s, %d M tiles (%d rows) on %d SMs; rel err %s"
        % (tag, variant_name(out["variant"]), m_tiles(gemm_ns or ns, h, w), halo_rows(gemm_ns or ns, h, w), num_sms(),
           " ".join("%s %.2e" % kv for kv in errs.items())))
  for k in ("c", "h", "gates"):
    if k in errs:
      assert errs[k] < TIGHT, (tag, k, errs[k])
  if xh2 is not None:      # bf16 x 2 planes / a0 + e4m3(a1) sum back to h' (test_parity_gpu.py bounds)
    assert errs["planes-h'"] < (1e-5 if planes == ops.PLANES_F16F8 else 2e-5), (tag, errs["planes-h'"])
  for k in ("c", "h", "gates", "xh2"):
    if out.get(k) is not None:
      assert halo_bits(out[k], ns, h, w) == 0, "%s: the kernel wrote into the zero halo of %s" % (tag, k)


def run_fwd(d, planes, zero_c=False, train=False):
  """cell_fwd (or cell_fwd_train) on the inputs d, with next-step operand planes of the same format."""
  from multiverse_b200 import ops
  ns, h, w, _ = d["x"].shape
  dev = d["x"].device
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(d["x"], xh, 0, h, w)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, planes, dev))
  c_in = None if zero_c else to_halo(d["c"])
  if train:
    out["gates"] = torch.zeros((halo_rows(ns, h, w), 4 * HID), device=dev)
    ops.cell_fwd_train(xh, pk, c_in, out["c"], out["h"], out["xh2"], out["gates"], h, w, ns)
  else:
    ops.cell_fwd(xh, pk, c_in, out["c"], out["h"], out["xh2"], h, w, ns)
  out["variant"] = ops.cell_last_variant()
  return out


# --------------------------------------------------------------------------- forward cell at size
@pytest.mark.gpu
@pytest.mark.parametrize("planes", [2, 16])
@pytest.mark.parametrize("launch", ["persistent", "strided"])
def test_cell_single_cta_at_size(dev, launch, planes):
  """The single-CTA kernel with several tiles per CTA: the largest launch below the pair threshold (2 x SMs - 1 M
  tiles, ~8 work items per CTA, back-to-back order), and ~40 M tiles (160 work items on the SMs: strided order, two
  items on some CTAs)."""
  ns, h, w = single_cta_max_size() if launch == "persistent" else (8, 36, 18)
  assert m_tiles(ns, h, w) < 2 * num_sms() and 4 * m_tiles(ns, h, w) > num_sms()
  d = cell_inputs(dev, ns, h, w, 32, seed=101)
  out = run_fwd(d, planes)
  check_fwd("single-CTA %s %dx%d n%d" % (launch, h, w, ns), ns, h, w, out,
            ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]), planes, pair=False)


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [2, 16])
@pytest.mark.parametrize("odd", [False, True])
@pytest.mark.parametrize("grid", [(36, 18), (18, 32), (4, 62)])
def test_cell_pair_at_size(dev, grid, odd, planes):
  """The CTA-pair kernel on the 36x18 grid (4 weight slots), the native 18x32 grid (3 slots) and 4x62 (A stage of
  exactly 256 rows), with an even and an odd number of M tiles (odd: rank 1 of the last pair owns a tile past R);
  R is never a multiple of 128."""
  h, w = grid
  ns = pair_ns(h, w, odd)
  d = cell_inputs(dev, ns, h, w, 32, seed=102 + h)
  out = run_fwd(d, planes)
  check_fwd("pair %dx%d n%d" % (h, w, ns), ns, h, w, out, ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]),
            planes, pair=True)


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [2, 16])
def test_cell_pair_zero_state(dev, planes):
  ns = pair_ns(36, 18, odd=True)
  d = cell_inputs(dev, ns, 36, 18, 32, seed=103)
  out = run_fwd(d, planes, zero_c=True)
  check_fwd("pair zero state n%d" % ns, ns, 36, 18, out,
            ref_cell(d["x"], d["h"], None, d["kernel"], d["bias"]), planes, pair=True)


@pytest.mark.gpu
def test_cell_refuses_a_grid_wider_than_the_a_stage(dev):
  """W = 63 needs an A stage of 264 rows, over the TMA box limit of 256: refused before any launch."""
  from multiverse_b200 import ops
  d = cell_inputs(dev, 1, 4, 63, 32, seed=104)
  pk = ops.PackedCell(d["kernel"], d["bias"], 2)
  xh = ops.alloc_xh(1, 4, 63, pk.cpad, 2, dev)
  c_out, h_out = ops.alloc_state(1, 4, 63, dev), ops.alloc_state(1, 4, 63, dev)
  torch.cuda.synchronize()
  ops.reset_launch_count()
  with pytest.raises(RuntimeError, match="W=63"):
    ops.cell_fwd(xh, pk, None, c_out, h_out, None, 4, 63, 1)
  assert ops.launch_count() == 0


@pytest.mark.gpu
def test_cell_fwd_train_pair_stores_the_gates(dev):
  ns = pair_ns(36, 18, odd=True)
  d = cell_inputs(dev, ns, 36, 18, 32, seed=105)
  out = run_fwd(d, 2, train=True)
  check_fwd("pair fwd_train n%d" % ns, ns, 36, 18, out, ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]),
            2, pair=True)


def _onehot_case(dev, ns, h, w, seed):
  """Class-decoder inputs: ids in the four corners, on the four edges and random, the class embedding of
  cases.head_case."""
  hd = cases.head_case()
  d = cell_inputs(dev, ns, h, w, 32, seed=seed)
  g = torch.Generator(device=dev)
  g.manual_seed(seed)
  ids = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32)
  ids[:8] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1, 3, 4 * w, 5 * w + w - 1, (h - 1) * w + 7],
                         dtype=torch.int32)
  We = torch.from_numpy(hd["We1"]).to(dev)
  be = torch.from_numpy(hd["be"]).to(dev)
  return d, ids, We, be, g


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [2, 16])
def test_cell_onehot_row_map_pair(dev, planes):
  """x-fold (the embedded one-hot input as table look-ups) with a row map (beam parents) under the pair kernel,
  against the reference cell fed the explicit embedding."""
  from multiverse_b200 import ops
  h, w = 36, 18
  ns = pair_ns(h, w, odd=True)
  d, ids, We, be, g = _onehot_case(dev, ns, h, w, 106)
  rm = torch.randint(0, ns, (ns,), generator=g, device=dev, dtype=torch.int32)
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  xf = ops.XFold(d["kernel"], d["bias"], We, be)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, planes, dev))
  ops.cell_fwd_onehot(xh, pk, xf, ids, to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns, row_map=rm)
  out["variant"] = ops.cell_last_variant()
  x = ref_onehot_emb(ids, h, w, We, be)
  check_fwd("pair onehot + row_map n%d" % ns, ns, h, w, out,
            ref_cell(x, d["h"], d["c"], d["kernel"], d["bias"], row_map=rm), planes, pair=True)


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [2, 16])
def test_cell_onehot_fanout_pair(dev, planes):
  """The first K-row beam step: the GEMM on the parent rows under the pair kernel (raw accumulators out), then the
  children kernel; against the reference of every child's explicit embedding with its parent's h and c."""
  from multiverse_b200 import ops
  h, w, k = 36, 18, 4
  ns = pair_ns(h, w, odd=True)
  d, _, We, be, g = _onehot_case(dev, ns, h, w, 107)
  ids = torch.randint(0, h * w, (ns * k,), generator=g, device=dev, dtype=torch.int32)
  ids[:4] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1], dtype=torch.int32)
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  xf = ops.XFold(d["kernel"], d["bias"], We, be)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns * k, h, w, dev), h=ops.alloc_state(ns * k, h, w, dev))
  ops.cell_fwd_onehot_fanout(xh, pk, xf, ids, to_halo(d["c"]), out["c"], out["h"], h, w, ns, k)
  out["variant"] = ops.cell_last_variant()
  parent = torch.arange(ns, device=dev).repeat_interleave(k)
  ref = ref_cell(ref_onehot_emb(ids, h, w, We, be), d["h"][parent], d["c"], d["kernel"], d["bias"], row_map=parent)
  check_fwd("pair onehot fan-out n%d x K%d" % (ns, k), ns * k, h, w, out, ref, planes, pair=True, gemm_ns=ns)


@pytest.mark.gpu
def test_cell_xsparse_pair(dev):
  """The class encoder's sparse x path (per-sample table rows added around the label cell) under the pair kernel,
  labels in corners, on edges, inside and out of range (-1, H*W)."""
  from multiverse_b200 import ops
  h, w, cx = 36, 18, 64
  ns = pair_ns(h, w, odd=True)
  d = cell_inputs(dev, ns, h, w, cx, seed=108)
  g = torch.Generator(device=dev)
  g.manual_seed(108)
  conv = torch.tanh(torch.randn((7, h * w, 64), generator=g, device=dev))
  frames = torch.randint(0, 7, (ns,), generator=g, device=dev, dtype=torch.int32)
  labels = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32)
  labels[:8] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1, 5, 6 * w, -1, h * w], dtype=torch.int32)
  x = torch.zeros((ns, h * w, 64), device=dev)
  ok = (labels >= 0) & (labels < h * w)
  s = torch.nonzero(ok).squeeze(1)
  x[s, labels[s].long()] = conv[frames[s].long(), labels[s].long()]
  pk = ops.PackedCell(d["kernel"], d["bias"], ops.PLANES_F16F8)
  xs = ops.XSparse(d["kernel"])
  xh = ops.alloc_xh(ns, h, w, pk.cpad, ops.PLANES_F16F8, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  table = torch.empty((ns, 9, 4 * HID), device=dev)
  ops.cell_xsparse_table(conv, frames, labels, xs, table, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, ops.PLANES_F16F8, dev))
  ops.cell_fwd_xsparse(xh, pk, table, labels, to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns)
  out["variant"] = ops.cell_last_variant()
  check_fwd("pair xsparse n%d" % ns, ns, h, w, out,
            ref_cell(x.view(ns, h, w, 64), d["h"], d["c"], d["kernel"], d["bias"]), ops.PLANES_F16F8, pair=True)


@pytest.mark.gpu
def test_cell_xdense_pair(dev):
  """The regression encoder's dense x path (raw 2-channel input of +-1e3 added in fp32 in the epilogue) under the
  pair kernel."""
  from multiverse_b200 import ops
  h, w = 36, 18
  ns = pair_ns(h, w, odd=True)
  d = cell_inputs(dev, ns, h, w, 2, seed=109, x_scale=600.0)
  assert float(d["x"].abs().max()) > 1e3
  pk = ops.PackedCell(d["kernel"], d["bias"], ops.PLANES_F16F8)
  xd = ops.XDense(d["kernel"])
  xh = ops.alloc_xh(ns, h, w, pk.cpad, ops.PLANES_F16F8, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, ops.PLANES_F16F8, dev))
  ops.cell_fwd_xdense(xh, pk, xd, d["x"].contiguous(), to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns)
  out["variant"] = ops.cell_last_variant()
  check_fwd("pair xdense n%d" % ns, ns, h, w, out, ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]),
            ops.PLANES_F16F8, pair=True)


# --------------------------------------------------------------------------- launch switches
SWITCHES = [{}, {"MVB_CELL_MULTICAST": "0"}, {"MVB_CELL_ORDER": "0"}, {"MVB_CELL_ORDER": "1"},
            {"MVB_CELL_MULTICAST": "0", "MVB_CELL_ORDER": "0"}]


def switch_outputs(path):
  """Child side of test_cell_launch_switches_are_bit_identical: the odd pair-size cell in P=2 and f16f8 under this
  process's MVB_CELL_* settings, outputs saved to `path`."""
  from multiverse_b200 import ops
  dev = torch.device("cuda:0")
  ns = pair_ns(36, 18, odd=True)
  d = cell_inputs(dev, ns, 36, 18, 32, seed=110)
  res = {}
  for planes in (2, ops.PLANES_F16F8):
    out = run_fwd(d, planes)
    res[planes] = dict(c=out["c"].cpu(), h=out["h"].cpu(), xh2=out["xh2"].view(torch.int16).cpu(),
                       variant=out["variant"])
  torch.save(res, path)


@pytest.mark.gpu
def test_cell_launch_switches_are_bit_identical(dev, tmp_path):
  """MVB_CELL_MULTICAST and MVB_CELL_ORDER change which CTA computes which tile and how the weight tile arrives, not
  the K order inside a tile: c', h' and the output planes are bit-identical under every setting.  The library reads
  both variables once per process, so every setting runs in a child interpreter."""
  from multiverse_b200 import ops
  env0 = {k: v for k, v in os.environ.items() if not k.startswith("MVB_CELL_")}
  base = None
  for sw in SWITCHES:
    path = str(tmp_path / "out.pt")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_kernels_atsize_gpu as t; t.switch_outputs(%r)" % (
        ROOT, TESTS, path)
    r = subprocess.run([sys.executable, "-B", "-c", code], env=dict(env0, **sw), cwd=ROOT, timeout=900,
                       capture_output=True, text=True)
    assert r.returncode == 0, "child with %s failed:\n%s\n%s" % (sw, r.stdout[-3000:], r.stderr[-3000:])
    res = torch.load(path)
    os.remove(path)
    for planes, o in sorted(res.items()):
      pair = sw.get("MVB_CELL_MULTICAST") != "0"
      assert o["variant"] == planes * 2 + int(pair), (sw, variant_name(o["variant"]))
      print("switches %s: %s ran" % (sw or "default", variant_name(o["variant"])))
      if base is None:
        continue
      for k in ("c", "h", "xh2"):
        a, b = o[k], base[planes][k]
        assert torch.equal(a, b), "%s, planes %d: %s differs from the default launch (max |diff| %.3e)" % (
            sw, planes, k, float((a.float() - b.float()).abs().max()) if k != "xh2" else float("nan"))
    if base is None:
      base = res
  assert base[ops.PLANES_F16F8]["variant"] == ops.PLANES_F16F8 * 2 + 1


# --------------------------------------------------------------------------- backward at training size
BWD_CELLS = {
    # name: (cx, x scale, need_dx)   decoder / class-encoder cells, and the compensated regression encoder (raw
    # pixel offsets as input: no gradient to its input, the single N = 256 dgrad tile)
    "dec_cx32": (32, 1.0, True),
    "enc_class_cx64": (64, 1.0, True),
    "enc_reg_cx2": (2, 600.0, False),
}


def run_backward(dev, name, ns, h, w, seed):
  """One BPTT step of a cell chained as TrainEngine._cell_bwd, P = 2:  cell_fwd_train -> lstm_gates_bwd ->
  cell_dgrad (into a dxh prefilled with SENTINEL) -> cell_wgrad_direct -> unpack_cell_wgrad; then the weight gradient
  again into the same slabs (accumulation) and into fresh ones (determinism).  Returns kernel outputs, reference."""
  from multiverse_b200 import ops
  cx, xs, need_dx = BWD_CELLS[name]
  d = cell_inputs(dev, ns, h, w, cx, seed, x_scale=xs)
  g = torch.Generator(device=dev)
  g.manual_seed(seed + 1)
  dh = torch.randn((ns, h, w, HID), generator=g, device=dev)
  dc = torch.randn((ns, h, w, HID), generator=g, device=dev)
  pk = ops.PackedCell(d["kernel"], d["bias"], 2, comp=cx == 2)
  wd = ops.pack_dgrad(pk, d["kernel"])
  xh = ops.alloc_xh(ns, h, w, pk.cpad, 2, dev)
  ops.nhwc_to_planes(d["x"], xh, 0, h, w, comp=pk.comp)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  rows = halo_rows(ns, h, w)
  c_in = to_halo(d["c"])
  c_out, h_out = ops.alloc_state(ns, h, w, dev), ops.alloc_state(ns, h, w, dev)
  gates = torch.zeros((rows, 4 * HID), device=dev)
  ops.cell_fwd_train(xh, pk, c_in, c_out, h_out, None, gates, h, w, ns)
  o = dict(variant=ops.cell_last_variant(), need_dx=need_dx, cx=cx, cxp=pk.cxp)
  dg = torch.zeros((2, rows, 4 * HID), dtype=torch.bfloat16, device=dev)
  o["dc_prev"] = ops.alloc_state(ns, h, w, dev)
  dbp = torch.zeros((4 * HID,), device=dev)
  ops.lstm_gates_bwd(gates, c_in, c_out, to_halo(dh), to_halo(dc), dg, o["dc_prev"], dbp, h, w, ns)
  o["dxh"] = torch.full((rows, pk.cpad), SENTINEL, device=dev)
  ops.cell_dgrad(dg, wd, o["dxh"], h, w, ns, need_dx=need_dx)
  dwp = torch.zeros((ops.wgrad_slabs(pk.cpad), 4 * HID, 9 * pk.cpad), device=dev)
  ops.cell_wgrad_direct(dg, xh, dwp, h, w, ns)
  o["dW"] = torch.empty((3, 3, cx + HID, 4 * HID), device=dev)
  o["db"] = torch.empty((4 * HID,), device=dev)
  ops.unpack_cell_wgrad(dwp, dbp, o["dW"], o["db"], cx, comp=pk.comp)
  o["dwp"] = dwp.clone()
  ops.cell_wgrad_direct(dg, xh, dwp, h, w, ns)
  o["dwp_twice"] = dwp
  o["dwp_again"] = torch.zeros_like(dwp)
  ops.cell_wgrad_direct(dg, xh, o["dwp_again"], h, w, ns)
  ref = ref_cell_grads(d["x"], d["h"], d["c"], d["kernel"], d["bias"], dh, dc)
  return o, ref


def check_backward(tag, ns, h, w, o, ref):
  dxh = inner(o["dxh"], ns, h, w)
  cx, cxp = o["cx"], o["cxp"]
  errs = {"dc_prev": rel(inner(o["dc_prev"], ns, h, w), ref["dc_prev"]), "dh_prev": rel(dxh[..., cxp:], ref["dh_prev"]),
          "dW": rel(o["dW"], ref["dW"]), "db": rel(o["db"], ref["db"])}
  if o["need_dx"]:
    errs["dx"] = rel(dxh[..., :cx], ref["dx"])
  print("%s: forward %s, %d halo rows, %d dgrad M tiles on %d SMs, %d wgrad slabs; worst rel err %s"
        % (tag, variant_name(o["variant"]), halo_rows(ns, h, w), m_tiles(ns, h, w), num_sms(), o["dwp"].shape[0],
           " ".join("%s %.2e" % kv for kv in errs.items())))
  for k, e in errs.items():
    assert e < GTOL, (tag, k, e)
  # dgrad writes the grid cells' rows only, and with need_dx=False only the h block of them
  full = o["dxh"].view(ns, h + 1, w + 1, -1)
  assert bool((full[:, h] == SENTINEL).all()) and bool((full[:, :, w] == SENTINEL).all()), "dgrad wrote a halo row"
  if not o["need_dx"]:
    assert bool((o["dxh"][:, :cxp] == SENTINEL).all()), "dgrad with need_dx=False wrote the x block"
  # the slabs accumulate (x + x = 2x exactly), and dW is deterministic: no atomics in the weight gradient
  for s in range(o["dwp"].shape[0]):
    assert torch.equal(o["dwp_twice"][s], 2 * o["dwp"][s]), "slab %d did not accumulate" % s
  assert torch.equal(o["dwp_again"], o["dwp"]), "the weight gradient differs between two runs"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BWD_CELLS))
def test_cell_backward_at_training_size(dev, name):
  """Micro-batch 128 of 36x18 (89 984 halo rows, 703 M tiles): the forward runs the pair kernel with stored gates,
  dgrad loops over 5-11 tiles per CTA, wgrad splits the rows over 5 (cpad 288) or 2 (cpad 320) slabs."""
  ns, h, w = 128, 36, 18
  o, ref = run_backward(dev, name, ns, h, w, seed=120 + BWD_CELLS[name][0])
  assert m_tiles(ns, h, w) >= 2 * num_sms()
  assert o["variant"] == 2 * 2 + 1, "the forward ran %s, not the P=2 pair kernel" % variant_name(o["variant"])
  check_backward("backward %s n%d" % (name, ns), ns, h, w, o, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BWD_CELLS))
def test_cell_backward_tiny_launch(dev, name):
  """One 4x4 sample (25 halo rows, one k-block): every k-split but the first has no rows at all."""
  o, ref = run_backward(dev, name, 1, 4, 4, seed=130 + BWD_CELLS[name][0])
  check_backward("backward %s 4x4 n1" % name, 1, 4, 4, o, ref)
