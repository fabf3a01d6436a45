# coding=utf-8
"""Every --emb_size the engine accepts (every multiple of 8 from 8 to 256): the cell row widths cpad 416, 448 and 480
(three x chunks, and four with a trailing 32-channel chunk at channel 192) and x blocks narrower than their 32-channel
padding (cx < cxp), whose channels [cx, cxp) every kernel must keep inert.  tests/emb_matrix_cases.py lists one
embedding width per cpad with and without padding; test_emb_matrix_cpu.py checks that it reaches every cpad.

Kernels element by element against the fp64 references of test_kernels_atsize_gpu.py (3e-5 forward, 2e-4 gradients,
1e-5 emb_bwd):
  - the cell forward in both operand formats under the single-CTA and the CTA-pair kernel, cell_fwd_train, x-fold
    with a row map and fan-out, the epilogue-warpgroup kernel bit for bit against cell_fwd_kernel;
  - padded x channels filled with +-1e3 leave every output bit unchanged (zero packed weights in the pad);
  - dgrad / wgrad / unpack at micro-batch 128 on 36x18, 18x32 and 9x16: exact zeros in the pad of dx and of every
    wgrad slab, no store past the end of dx;
  - the embedding writers (heads, emb_onehot_fwd, emb_dense_fwd) in both formats, emb_bwd with partial channel groups.
Models against the fp64 oracle: greedy two-scale rollouts at emb 40 and 200, a K = 5 beam at emb 136, the whole-model
gradient at emb 200 (scene encoding) and 136 (without), and one drop-in Trainer.step at emb 136 against the executed
reference (tests/golden/make_golden_emb_matrix.py)."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import emb_matrix_cases as EM
import test_emb_size_gpu as ES
import test_kernels_atsize_gpu as K
from test_beam_no_gnn_gpu import rel

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
GOLD = os.path.join(TESTS, "golden")
HID = 256
F16F8 = 16
GRID_IDS = {(36, 18): "36x18", (18, 32): "18x32", (9, 16): "9x16"}
# forward cases: every new cpad with and without padding on both grids
FWD = [(e, (36, 18) if i % 2 == 0 else (18, 32)) for i, e in enumerate(EM.MATRIX)]
FWD_IDS = ["E%d-%s" % (e, GRID_IDS[g]) for e, g in FWD]
GUARD_ROWS = 8          # rows past the end of dx that dgrad must leave alone


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


def channel_bytes(xh, lo, hi):
  """The bytes of channels [lo, hi) of every row of the operand buffer xh, [rows, k] uint8: both bf16 planes, or the
  fp16 value and the two e4m3 bytes of the f16f8 format (ops.operand_values's layout)."""
  from multiverse_b200 import ops
  r, cpad = xh.shape[1], xh.shape[2]
  raw = xh.view(torch.uint8).reshape(-1)
  ch = torch.arange(lo, hi, device=xh.device)
  two = torch.stack([2 * ch, 2 * ch + 1], 1).reshape(-1)
  if ops.planes_of(xh) != ops.PLANES_F16F8:
    planes = raw.view(2, r, 2 * cpad)
    return torch.cat([planes[0][:, two], planes[1][:, two]], 1)
  a0, f8 = raw[:2 * r * cpad].view(r, 2 * cpad), raw[2 * r * cpad:].view(r, 2 * cpad)
  cxp = cpad - HID
  c0 = torch.where(ch >= cxp, cxp + (ch - cxp) // 64 * 64, ch // 64 * 64)
  width = torch.where(ch >= cxp, 64, (cxp - c0).clamp(max=64))
  off0 = 2 * c0 + (ch - c0)
  return torch.cat([a0[:, two], f8[:, off0], f8[:, off0 + width]], 1)


# --------------------------------------------------------------------------- cell forward
@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("launch", ["single", "pair"])
@pytest.mark.parametrize("cx,grid", FWD, ids=FWD_IDS)
def test_cell_forward(dev, cx, grid, launch, planes):
  """Three x chunks (cpad 416, 448), four with a trailing 32-channel one (480), and x blocks narrower than their
  padding, both operand formats, under the single-CTA kernel (several tiles per CTA, R not a multiple of 128) and the
  CTA-pair kernel (odd M tiles)."""
  from multiverse_b200 import ops
  h, w = grid
  ns = K.pair_ns(h, w, odd=True) if launch == "pair" else ES.single_ns(h, w)
  assert K.halo_rows(ns, h, w) % K.BLOCK_M != 0
  d = ES.wide_inputs(dev, ns, h, w, cx, seed=600 + cx + h + (launch == "pair"))
  out = K.run_fwd(d, planes)
  assert out["xh2"].shape[2] == ops.cell_cpad(cx) == EM.cpad_of(cx)
  K.check_fwd("%s cx%d cpad %d %dx%d n%d" % (launch, cx, ops.cell_cpad(cx), h, w, ns), ns, h, w, out,
              K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]), planes, pair=launch == "pair")


@pytest.mark.parametrize("cx", EM.MATRIX)
def test_cell_forward_stores_the_gates(dev, cx):
  """cell_fwd_train (bf16x2, gates stored for the backward) under the pair kernel."""
  ns = K.pair_ns(36, 18, odd=True)
  d = ES.wide_inputs(dev, ns, 36, 18, cx, seed=620 + cx)
  out = K.run_fwd(d, 2, train=True)
  K.check_fwd("fwd_train cx%d n%d" % (cx, ns), ns, 36, 18, out,
              K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"]), 2, pair=True)


@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("cx", EM.PADDED)
def test_padded_x_channels_are_inert(dev, cx, planes):
  """x channels [cx, cxp) of the operands filled with +-1e3 (both planes / the fp16 and both e4m3 bytes): c', h' and
  the next operands bit-identical to the launch with zeros there.  Any non-zero packed weight in the pad (the bf16x2
  pack kernel or the f16f8 one) changes them."""
  from multiverse_b200 import ops
  h, w, ns = 36, 18, 6
  d = ES.wide_inputs(dev, ns, h, w, cx, seed=640 + cx)
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  assert pk.cxp > cx
  g = torch.Generator(device=dev)
  g.manual_seed(641 + cx)
  big = torch.where(torch.rand((ns, h, w, pk.cxp - cx), generator=g, device=dev) < 0.5, -1e3, 1e3)
  res = []
  for pad in (None, big):
    xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
    ops.nhwc_to_planes(d["x"] if pad is None else torch.cat([d["x"], pad], -1).contiguous(), xh, 0, h, w)
    ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
    if pad is not None:
      vals, e0 = ops.operand_values(xh)
      assert float(K.inner(vals, ns, h, w)[..., cx:pk.cxp].abs().min()) > 900.0
    out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
               xh2=ops.alloc_xh(ns, h, w, pk.cpad, planes, dev))
    ops.cell_fwd(xh, pk, K.to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns)
    res.append(out)
  for k in ("c", "h", "xh2"):
    assert torch.equal(res[0][k].view(torch.int16), res[1][k].view(torch.int16)), (cx, planes, k)
  print("cx%d (cxp %d) %s: outputs bit-identical with +-1e3 in the %d padded channels"
        % (cx, pk.cxp, K.variant_name(ops.cell_last_variant()), pk.cxp - cx))


def _xfold_inputs(dev, cx, seed):
  h, w = 36, 18
  ns = K.pair_ns(h, w, odd=True)
  d, ids, _, _, g = K._onehot_case(dev, ns, h, w, seed)
  d = dict(d, **{k: v for k, v in K.cell_inputs(dev, ns, h, w, cx, seed=seed).items() if k in ("kernel", "x")})
  We, be = ES._wide_emb(dev, cx, seed + 1)
  return h, w, ns, d, ids, We, be, g


@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("cx", [136, 192, 200])
def test_cell_x_fold(dev, cx, planes):
  """x-fold (the embedded one-hot input as table look-ups, cell_xfold_tables at E = cx) with a row map under the pair
  kernel, at padded x blocks (cpad 416, 480) and at cpad 448."""
  from multiverse_b200 import ops
  h, w, ns, d, ids, We, be, g = _xfold_inputs(dev, cx, 660 + cx)
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


@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("cx", [136, 192, 200])
def test_cell_x_fold_fanout(dev, cx, planes):
  """The first K-row beam step (GEMM on the parent rows under the pair kernel, then the children kernel) with the
  x-fold tables at E = cx."""
  from multiverse_b200 import ops
  h, w, ns, d, _, We, be, g = _xfold_inputs(dev, cx, 680 + cx)
  k = 4
  ids = torch.randint(0, h * w, (ns * k,), generator=g, device=dev, dtype=torch.int32)
  ids[:4] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1], dtype=torch.int32)
  pk = ops.PackedCell(d["kernel"], d["bias"], planes)
  xf = ops.XFold(d["kernel"], d["bias"], We, be)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns * k, h, w, dev), h=ops.alloc_state(ns * k, h, w, dev))
  ops.cell_fwd_onehot_fanout(xh, pk, xf, ids, K.to_halo(d["c"]), out["c"], out["h"], h, w, ns, k)
  out["variant"] = ops.cell_last_variant()
  parent = torch.arange(ns, device=dev).repeat_interleave(k)
  ref = K.ref_cell(K.ref_onehot_emb(ids, h, w, We, be), d["h"][parent], d["c"], d["kernel"], d["bias"], row_map=parent)
  K.check_fwd("x-fold fan-out cx%d n%d x K%d" % (cx, ns, k), ns * k, h, w, out, ref, planes, pair=True, gemm_ns=ns)


EPI_CASES = [(cx, launch) for cx in (136, 192, 200) for launch in ("single", "pair")]


def _epi_inputs(dev, cx, launch):
  ns = K.pair_ns(36, 18, odd=True) if launch == "pair" else ES.single_ns(36, 18)
  return ns, ES.wide_inputs(dev, ns, 36, 18, cx, seed=700 + cx + (launch == "pair"))


def epi_outputs(path):
  """Child side of test_cell_epilogue_warpgroup: the f16f8 cell launches of EPI_CASES, outputs saved to `path`."""
  dev = torch.device("cuda:0")
  res = {}
  for cx, launch in EPI_CASES:
    _, d = _epi_inputs(dev, cx, launch)
    out = K.run_fwd(d, F16F8)
    res[(cx, launch)] = dict(c=out["c"].cpu(), h=out["h"].cpu(), xh2=out["xh2"].view(torch.int16).cpu(),
                             variant=out["variant"])
  torch.save(res, path)


def test_cell_epilogue_warpgroup(dev, tmp_path):
  """cell_fwd_epi_kernel (MVB_CELL_EPI_WG=1) and cell_fwd_kernel (=0) at cpad 416, 448 and 480, single-CTA and pair:
  c', h' and the next operands bit-identical, and within the forward bar of fp64.  The library reads the switch once
  per process, so each setting runs in a child interpreter."""
  res = {}
  for epi in ("0", "1"):
    path = str(tmp_path / ("out%s.pt" % epi))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_emb_matrix_gpu as t; t.epi_outputs(%r)" % (
        ROOT, TESTS, path)
    env = dict({k: v for k, v in os.environ.items() if not k.startswith("MVB_CELL_")}, MVB_CELL_EPI_WG=epi)
    r = subprocess.run([sys.executable, "-B", "-c", code], env=env, cwd=ROOT, timeout=900, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res[epi] = torch.load(path)
  for cx, launch in EPI_CASES:
    a, b = res["0"][(cx, launch)], res["1"][(cx, launch)]
    assert a["variant"] == b["variant"] == F16F8 * 2 + int(launch == "pair"), (a["variant"], b["variant"])
    for k in ("c", "h", "xh2"):
      assert torch.equal(a[k], b[k]), "cx%d %s: %s differs between the two f16f8 kernels" % (cx, launch, k)
    ns, d = _epi_inputs(dev, cx, launch)
    ref = K.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"])
    errs = {k: rel(K.inner(b[k], ns, 36, 18).numpy(), ref[k].cpu().numpy()) for k in ("c", "h")}
    print("epilogue warpgroup cx%d (cpad %d) %s n%d: bit-identical to cell_fwd_kernel, rel err %s"
          % (cx, EM.cpad_of(cx), launch, ns, {k: "%.2e" % v for k, v in errs.items()}))
    assert max(errs.values()) < K.TIGHT, errs


# --------------------------------------------------------------------------- dgrad / wgrad / unpack
def run_guarded_backward(dev, monkeypatch, cx, ns, h, w, seed):
  """K.run_backward at an x block of cx channels, its dgrad writing into rows [0, R) of a buffer with GUARD_ROWS
  SENTINEL rows after them.  Returns (outputs, reference, guard rows after the dgrad)."""
  from multiverse_b200 import ops
  name = "matrix_cx%d" % cx
  monkeypatch.setitem(K.BWD_CELLS, name, (cx, 1.0, True))
  dgrad, guard = ops.cell_dgrad, []

  def guarded(dg, wd, dxh, h_, w_, ns_, need_dx=True):
    r = dxh.shape[0]
    buf = torch.full((r + GUARD_ROWS, dxh.shape[1]), K.SENTINEL, device=dxh.device)
    buf[:r] = dxh
    dgrad(dg, wd, buf[:r], h_, w_, ns_, need_dx=need_dx)
    dxh.copy_(buf[:r])
    guard.append(buf[r:].clone())
  monkeypatch.setattr(ops, "cell_dgrad", guarded)
  o, ref = K.run_backward(dev, name, ns, h, w, seed)
  assert len(guard) == 1
  return o, ref, guard[0]


def check_padding(tag, ns, h, w, o, guard):
  """dgrad writes exact zeros into the padded x channels and nothing past dx; every wgrad slab is exactly zero in
  the padded channels of every tap."""
  from multiverse_b200 import ops
  cx, cxp = o["cx"], o["cxp"]
  cpad = cxp + HID
  assert bool((guard == K.SENTINEL).all()), "%s: dgrad stored past the end of dx" % tag
  assert o["dwp"].shape[0] == ops.wgrad_slabs(cpad)
  if cx < cxp:
    pad = K.inner(o["dxh"], ns, h, w)[..., cx:cxp]
    assert bool((pad == 0).all()), "%s: dgrad wrote %s into the padded x channels" % (tag, float(pad.abs().max()))
    for k in ("dwp", "dwp_twice", "dwp_again"):
      slabs = o[k].view(o[k].shape[0], 4 * HID, 9, cpad)[..., cx:cxp]
      assert bool((slabs == 0).all()), "%s: %s is not zero in the padded channels" % (tag, k)


BWD = [(e, g) for e in EM.MATRIX for g in K.BWD_GRIDS]


@pytest.mark.parametrize("cx,grid", BWD, ids=["E%d-%s" % (e, GRID_IDS[g]) for e, g in BWD])
def test_cell_backward(dev, monkeypatch, cx, grid):
  """Micro-batch 128: dgrad with the x block (the second N tile 256 wide with 160, 192 or 224 valid columns at cpad
  416, 448, 480), wgrad on its slabs (cpad 416: 32-channel units, 13 per tap; 448: three 64-channel units per N tile
  of 192; 480: one 160-channel unit, 3 per tap), unpack to the TF layout, against fp64; the slabs accumulate to
  exactly 2x and repeat bit for bit; no halo row written; the padded channels exactly zero."""
  from multiverse_b200 import ops
  h, w = grid
  ns = 128
  o, ref, guard = run_guarded_backward(dev, monkeypatch, cx, ns, h, w, seed=720 + cx + h)
  pair = K.m_tiles(ns, h, w) >= 2 * K.num_sms()
  assert o["variant"] == 2 * 2 + int(pair), K.variant_name(o["variant"])
  tag = "backward cx%d cpad %d (wgrad %d slabs) %dx%d n%d" % (cx, ops.cell_cpad(cx), o["dwp"].shape[0], h, w, ns)
  K.check_backward(tag, ns, h, w, o, ref)
  check_padding(tag, ns, h, w, o, guard)


@pytest.mark.parametrize("cx", [136, 184, 200])
def test_cell_backward_tiny_launch(dev, monkeypatch, cx):
  """One 4x4 sample (25 halo rows, one k-block) at cpad 416, 448 and 480."""
  o, ref, guard = run_guarded_backward(dev, monkeypatch, cx, 1, 4, 4, seed=760 + cx)
  tag = "backward cx%d 4x4 n1" % cx
  K.check_backward(tag, 1, 4, 4, o, ref)
  check_padding(tag, 1, 4, 4, o, guard)


# --------------------------------------------------------------------------- embedding writers
def _dense_emb(x, We, be):
  """fp64 tanh(conv3x3 SAME(x) + be) of a map x [n, h, w, P]."""
  n, h, w, p = x.shape
  e = We.shape[-1]
  return torch.tanh(K._taps(x.double()) @ We.double().reshape(9 * p, e) + be.double()).reshape(n, h, w, e)


EMB_CASES = [(e, [(36, 18), (18, 32), (9, 16)][i % 3]) for i, e in enumerate(EM.PADDED)]


@pytest.mark.parametrize("planes", [2, F16F8])
@pytest.mark.parametrize("E,grid", EMB_CASES, ids=["E%d-%s" % (e, GRID_IDS[g]) for e, g in EMB_CASES])
def test_embedding_writers(dev, E, grid, planes):
  """emb_onehot_fwd, emb_dense_fwd (Pout 2), head_class_fwd, head_class_fwd_dense (bf16x2 only) and head_reg_fwd write
  tanh(conv3x3 + be) into channels [0, E) of the next operands, in 8-channel groups that stop inside a 32-channel
  chunk: values within the format's rounding of fp64, channels [E, cxp) and the halo bit-zero, and a pre-filled h
  block left as it was."""
  from multiverse_b200 import ops
  h, w = grid
  ns = 16
  cpad = ops.cell_cpad(E)
  cxp = cpad - HID
  g = torch.Generator(device=dev)
  g.manual_seed(780 + E)
  rn = lambda *s: torch.randn(s, generator=g, device=dev)
  We1, We2, be = rn(3, 3, 1, E) * 0.5, rn(3, 3, 2, E) * 0.3, rn(E) * 0.1
  Wo1, Wo2 = rn(3, 3, HID, 1) * 0.05, rn(3, 3, HID, 2) * 0.05
  hs = torch.tanh(rn(ns, h, w, HID))
  h32 = K.to_halo(hs)
  ids = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32)
  ids[:4] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1], dtype=torch.int32)
  dense = rn(ns, h * w, 2)
  hblock = torch.tanh(rn(ns, h, w, HID))

  def run(write):
    xh = ops.alloc_xh(ns, h, w, cpad, planes, dev)
    ops.nhwc_to_planes(hblock, xh, cxp, h, w)
    before = channel_bytes(xh, cxp, cpad).clone()
    want = write(xh)
    vals, _ = ops.operand_values(xh)
    assert torch.equal(channel_bytes(xh, cxp, cpad), before), "the h block changed"
    assert int(channel_bytes(xh, E, cxp).ne(0).sum()) == 0, "channels [E, cxp) are not bit-zero"
    assert K.halo_bits(xh, ns, h, w) == 0, "the halo is not bit-zero"
    return K.rel(K.inner(vals, ns, h, w)[..., :E], want)

  errs = {}

  def onehot(xh):
    ops.emb_onehot_fwd(ids, We1, be, xh, h, w)
    return K.ref_onehot_emb(ids, h, w, We1, be)
  errs["emb_onehot_fwd"] = run(onehot)

  def dense2(xh):
    ops.emb_dense_fwd(dense, We2, be, xh, h, w)
    return _dense_emb(dense.view(ns, h, w, 2), We2, be)
  errs["emb_dense_fwd"] = run(dense2)

  def head_class(xh):
    logits, out_ids = torch.empty((ns, h * w), device=dev), torch.empty((ns,), dtype=torch.int32, device=dev)
    ops.head_class_fwd(h32, Wo1, logits, out_ids, We1, be, xh, h, w, ns, planes=planes)
    assert torch.equal(out_ids.long(), logits.argmax(-1))
    return K.ref_onehot_emb(out_ids, h, w, We1, be)
  errs["head_class_fwd"] = run(head_class)

  if planes == 2:
    def head_class_dense(xh):
      logits, out_ids = torch.empty((ns, h * w), device=dev), torch.empty((ns,), dtype=torch.int32, device=dev)
      ops.head_class_fwd_dense(h32, Wo1, logits, out_ids, We1, be, xh, h, w, ns, planes=planes)
      return _dense_emb(logits.view(ns, h, w, 1), We1, be)
    errs["head_class_fwd_dense"] = run(head_class_dense)

  def head_reg(xh):
    offs = torch.empty((ns, h * w, 2), device=dev)
    ops.head_reg_fwd(h32, Wo2, offs, We2, be, xh, h, w, ns, planes=planes)
    return _dense_emb(offs.view(ns, h, w, 2), We2, be)
  errs["head_reg_fwd"] = run(head_reg)

  print("embedding writers E%d (cxp %d) %dx%d %s: rel err %s"
        % (E, cxp, h, w, "f16f8" if planes == F16F8 else "bf16x2", {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < 3e-5, errs


# --------------------------------------------------------------------------- emb_bwd
def emb_groups(E, h, w):
  """emb_bwd's channel groups (mvb_train2.cu emb_bwd, restated): [HW][2 + EG] floats in 160 KB."""
  fit = 160 * 1024 // 4 // (h * w) - 2
  eg = E if fit >= E else fit // 8 * 8
  return [min(eg, E - e0) for e0 in range(0, E, eg)]


@pytest.mark.parametrize("kind", ["onehot", "dense1", "dense2"])
@pytest.mark.parametrize("grid", [(36, 18), (18, 32), (9, 16)], ids=["36x18", "18x32", "9x16"])
@pytest.mark.parametrize("E", [8, 40, 136, 200, 248])
def test_emb_bwd(dev, E, grid, kind):
  """emb_bwd against fp64 autograd, channel groups ending inside a 32-channel chunk (E 136 on 36x18: 56/56/24; E 200
  on 18x32: 64/64/64/8).  The rest of the dx row (padded x channels, the h block) and the halo hold SENTINEL: the
  kernel reads channels [0, E) of the grid cells only."""
  from multiverse_b200 import ops
  h, w = grid
  ns, pout = 16, 2 if kind == "dense2" else 1
  g = torch.Generator(device=dev)
  g.manual_seed(800 + E + h)
  cpad = ops.cell_cpad(E)
  We = torch.randn((3, 3, pout, E), generator=g, device=dev) * 0.3
  be = torch.randn((E,), generator=g, device=dev) * 0.1
  dx = torch.randn((ns, h, w, E), generator=g, device=dev)
  dxh = torch.full((ns, h + 1, w + 1, cpad), K.SENTINEL, device=dev)
  dxh[:, :h, :w, :E] = dx
  dxh = dxh.view(-1, cpad)
  ids = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32) if kind == "onehot" else None
  in_map = None if kind == "onehot" else torch.randn((ns, h * w * pout), generator=g, device=dev)
  dWe, dbe = torch.zeros_like(We), torch.zeros_like(be)
  d_in = None if kind == "onehot" else torch.ones((ns, h * w * pout), device=dev)
  ops.emb_bwd(dxh, ids, in_map, We, be, dWe, dbe, d_in, True, h, w, ns)
  rW, rb, rin = ES.ref_emb_grads(dx, ids, in_map, We, be, h, w)
  errs = dict(dWe=rel(dWe.cpu().numpy(), rW.cpu().numpy()), dbe=rel(dbe.cpu().numpy(), rb.cpu().numpy()))
  if rin is not None:
    errs["d_in"] = rel((d_in - 1.0).cpu().numpy(), rin.reshape(ns, -1).cpu().numpy())
  print("emb_bwd E%d %dx%d %s, channel groups %s: %s"
        % (E, h, w, kind, emb_groups(E, h, w), {k: "%.1e" % v for k, v in errs.items()}))
  assert max(errs.values()) < 1e-5, errs


# --------------------------------------------------------------------------- models against the fp64 oracle
@pytest.mark.parametrize("emb", [40, 200])
def test_rollout_greedy_two_scale(dev, emb):
  """test.py --use_scene_enc --use_gnn --emb_size 40 (cpad 320, 24 padded channels) and 200 (cpad 480, 24 padded):
  test_emb_size_gpu's greedy check (ids clear of ties equal, logits and offsets within 1e-4)."""
  ES.test_rollout_greedy_two_scale_wide_emb(dev, emb)


def test_rollout_beam_k5_emb136(dev):
  """test.py --use_scene_enc --use_beam_search --emb_size 136 (cpad 416), K = 5 plain beam on 18x9: every live beam
  row's logits at every step within 1e-4 of the fp64 truth replayed along the engine's own selections, the outputs
  the back-trace of that trace, offsets within 1e-4 of the oracle."""
  from multiverse_b200 import synthetic
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  over = dict(batch_size=4, emb_size=136, use_grids=[False, True], use_beam_search=True, beam_size=5,
              diverse_beam=False, fix_num_timestep=0, use_gnn=False)
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, 840), R.make_inputs(cfg, 840)
  out, tr, seen = ES.run_traced(cfg, w, f, dev)
  blg, ids, _ = [t.cpu().numpy() for t in out["beam_outputs"]]
  i = 1
  err = rel(tr["logits"], ES.beam_replay(cfg, w, f, i, tr["ids"], tr["parents"], dev))
  n, b, tp = ids.shape
  for j in range(n):
    par = np.arange(b)
    for t in range(tp - 1, -1, -1):
      assert np.array_equal(ids[j, :, t], tr["ids"][t, j, par]) and np.array_equal(blg[j, :, t], tr["logits"][t, j, par])
      par = tr["parents"][t, j, par]
  with torch.no_grad():          # the oracle's beam returns numpy arrays: on the CPU
    ref = RT._forward(cfg, {k: torch.from_numpy(v).double() for k, v in w.items()}, f, torch.float64)
  reg = rel(out["grid_pred_reg_decoded"][i].cpu().numpy(), ES._np(ref["grid_pred_reg_decoded"][i]))
  print("beam K5 emb 136: cell variants %s, logits along the engine's selections %.1e, offsets %.1e"
        % (sorted(seen), err, reg))
  assert err < 1e-4 and reg < 1e-4


def _fed_decoder(monkeypatch, ids_of_grid):
  """RT.decoder_greedy whose class decoder (one-hot feedback) follows ids_of_grid[(h, w)] [N, Tp] instead of its own
  arg-max: the truth along the engine's arg-max path, as no_scene_enc_ref.decoder_greedy_fed without scene encoding."""
  from oracle import multiverse_ref_torch as RT
  base = RT.decoder_greedy

  def dec(first, state, tp, cell_w, emb_w, head_w, scene_mean, mask, use_gnn, onehot):
    if not onehot:
      return base(first, state, tp, cell_w, emb_w, head_w, scene_mean, mask, use_gnn, onehot)
    c, hs = state
    _, hh, ww, _ = first.shape
    ids = ids_of_grid[(hh, ww)]
    inp, outs = first, []
    for t in range(tp):
      h_in = RT.gnn_dense(hs, scene_mean, mask) if use_gnn else hs
      c, hs = RT.convlstm_cell(RT.grid_emb(inp, *emb_w), c, h_in, *cell_w)
      outs.append(RT.conv2d_same(hs, head_w))
      inp = RT.one_hot_map(ids[:, t], hh, ww, hs.dtype, hs.device)
    return torch.stack(outs, 1)
  monkeypatch.setattr(RT, "decoder_greedy", dec)


@pytest.mark.parametrize("emb,scene_enc", [(200, True), (136, False)], ids=["emb200_scene_enc", "emb136_no_scene_enc"])
def test_whole_model_gradient(dev, monkeypatch, emb, scene_enc):
  """256 trajectories in micro-batches of 128 against the fp64 truth along the engine's arg-max path, every gradient
  within 2e-4: --emb_size 200 with scene encoding and attention (both decoders at cpad 480, 24 padded channels) and
  --emb_size 136 without scene encoding (class encoder and both decoders at cpad 416, 24 padded channels)."""
  import no_scene_enc_ref as NS
  from multiverse_b200 import ops, synthetic
  from multiverse_b200.train_engine import TrainEngine
  from oracle import multiverse_ref as R
  from oracle import multiverse_ref_torch as RT
  from test_train_atsize_gpu import FRAMES, GTOL, LTOL, T_PRED, chunk_feeds, on, shared_frame_feeds
  n, mb, chunk = 256, 128, 16
  over = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001, emb_size=emb, use_gnn=scene_enc)
  cfg = synthetic.make_config(batch_size=mb, clip_gradient_norm=10.0, use_scene_enc=scene_enc, **over)
  rcfg = R.default_config(batch_size=chunk, use_scene_enc=scene_enc, **over)
  seed = 860 + emb
  w = synthetic.make_weights(cfg, seed)
  f = shared_frame_feeds(synthetic.make_config(batch_size=n, use_scene_enc=scene_enc, **over), n, FRAMES, seed)
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  ops.cell_variants_seen(reset=True)
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
  seen = ops.cell_variants_seen()
  ids = [np.concatenate(a) for a in ids]
  mine = [np.concatenate(a) for a in mine]
  eng_grads = {k: v.cpu().numpy() for k, v in eng.grads.items()}
  del eng, feeds
  gc.collect()
  torch.cuda.empty_cache()
  grads = {k: np.zeros(v.shape) for k, v in w.items()}
  losses = np.zeros(4)
  logits = [[], []]
  fed = {}
  if scene_enc:
    _fed_decoder(monkeypatch, fed)
  for lo in range(0, n, chunk):
    sl = slice(lo, lo + chunk)
    if scene_enc:
      for i, (h, ww) in enumerate(rcfg.scene_grids):
        fed[(h, ww)] = torch.from_numpy(ids[i][sl]).to(dev)
      _, l, _, gr, lg = RT.loss_and_grads(rcfg, w, chunk_feeds(f, sl), device=dev, return_logits=True)
    else:
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
  print("whole model emb %d (scene encoding %s): cell variants %s, losses %.1e, worst gradient errors %s"
        % (emb, scene_enc, sorted(seen), np.abs(got - losses).max() / np.abs(losses).max(),
           sorted(worst.items(), key=lambda kv: -kv[1])[:4]))
  bad = {k: v for k, v in worst.items() if v > GTOL}
  assert not bad, bad


def test_dropin_trainer_step_emb136_equals_reference_execution(dev, monkeypatch):
  """One Trainer.step through the drop-in at --emb_size 136 without --use_scene_enc (the class encoder and both
  decoders at cpad 416) on the inputs of tests/golden/refexec_train_emb_no_scene_enc_emb136.npz: losses, every clipped
  gradient and the variables after Adadelta equal the unmodified reference Model + Trainer's."""
  import cases
  from multiverse_b200 import synthetic
  from oracle import multiverse_ref as R
  from test_train_options_gpu import _dropin_model, check_step_against_reference_execution
  over, seed = EM.TRAIN["no_scene_enc_emb136"]
  over = dict(over, **{k: v for k, v in EM.TRAIN_ARGS.items() if k != "optimizer"})
  cfg = R.default_config(**over)
  w, f = synthetic.make_weights(cfg, seed), R.make_inputs(cfg, seed)
  g = np.load(os.path.join(GOLD, "refexec_train_emb_no_scene_enc_emb136.npz"))
  assert abs(float(g["checksum"]) - cases.checksum(*w.values()) - cases.checksum(f["scene_feat"], f["traj"])) < 1e-6
  dover = dict(use_grids=[True, True], emb_size=136, use_scene_enc=False, use_gnn=False,
               grid_loss_weight=over["grid_loss_weight"], grid_reg_loss_weight=over["grid_reg_loss_weight"],
               wd=over["wd"])
  tf, pred_models, model, args, _, _, _, batch = _dropin_model(monkeypatch, w=w, f=f, n=cfg.batch_size, over=dover,
                                                               train_w_onehot=True, init_lr=over["init_lr"])
  assert set(model.weights()) == set(g["variables"])
  check_step_against_reference_execution("emb136", tf, pred_models, model, args, batch, w, g, "")
