# coding=utf-8
"""The f16f8 cell kernel's format-sized shared-memory rings, at every ring layout the product grids reach.

An f16f8 pass loads one 128-byte row per A row, so its A stages hold one plane and the space buys a deeper weight
ring: 5 weight slots at every width, plus a third A stage up to W = 21 (36x18, 18x9; two stages at 18x32 and 4x62,
whose A stage is the full 256-row TMA box).  The ring depth changes when a slot or stage is refilled, never which
products go into which accumulator in which order, so every output must be bit-identical to a run with the
bf16x2-sized rings (MVB_CELL_FORMAT_RINGS=0: two-plane A stages, 4 or 3 slots - the layout f16f8 used before).
The library reads that variable once per process, so the reference run is a child interpreter.

Cases: the CTA-pair kernel with an even and an odd number of M tiles on each grid, the single-CTA kernel with about
eight tiles per CTA (the stage and slot parities wrap across tile boundaries), and the class-decoder launch of the
beam steps (x-fold: four chunks per pass instead of five, row map).  Each is also checked against the fp64 reference
as in test_kernels_atsize_gpu.py."""
import os
import subprocess
import sys

import pytest
import torch

import test_kernels_atsize_gpu as atsize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
F16F8 = 16
GRIDS = [(36, 18), (18, 9), (18, 32), (4, 62)]


# name -> (input, h, w, launch, seed); launch "even" / "odd": pair kernel with that parity of M tiles, "single":
# the most sample rows that still run the single-CTA kernel (2 x SMs - 1 M tiles or just under)
CASES = {}
for _i, (_h, _w) in enumerate(GRIDS):
  for _launch in ("even", "odd", "single"):
    CASES["%s_%dx%d" % (_launch, _h, _w)] = ("plain", _h, _w, _launch, 200 + 10 * _i)
CASES["onehot_odd_36x18"] = ("onehot", 36, 18, "odd", 240)
CASES["onehot_even_18x9"] = ("onehot", 18, 9, "even", 241)


def sample_rows(h, w, launch):
  if launch != "single":
    return atsize.pair_ns(h, w, launch == "odd")
  ns = 1
  while atsize.m_tiles(ns + 1, h, w) < 2 * atsize.num_sms():
    ns += 1
  return ns


def run_case(kind, h, w, ns, seed):
  """One f16f8 cell launch on seeded inputs: outputs, and its fp64 reference (computed only when asked)."""
  from multiverse_b200 import ops
  dev = torch.device("cuda:0")
  if kind == "plain":
    d = atsize.cell_inputs(dev, ns, h, w, 32, seed=seed)
    out = atsize.run_fwd(d, F16F8)
    ref = lambda: atsize.ref_cell(d["x"], d["h"], d["c"], d["kernel"], d["bias"])
    return out, ref
  d, ids, We, be, g = atsize._onehot_case(dev, ns, h, w, seed)
  rm = torch.randint(0, ns, (ns,), generator=g, device=dev, dtype=torch.int32)
  pk = ops.PackedCell(d["kernel"], d["bias"], F16F8)
  xf = ops.XFold(d["kernel"], d["bias"], We, be)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, F16F8, dev)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  out = dict(c=ops.alloc_state(ns, h, w, dev), h=ops.alloc_state(ns, h, w, dev),
             xh2=ops.alloc_xh(ns, h, w, pk.cpad, F16F8, dev))
  ops.cell_fwd_onehot(xh, pk, xf, ids, atsize.to_halo(d["c"]), out["c"], out["h"], out["xh2"], h, w, ns, row_map=rm)
  out["variant"] = ops.cell_last_variant()
  ref = lambda: atsize.ref_cell(atsize.ref_onehot_emb(ids, h, w, We, be), d["h"], d["c"], d["kernel"], d["bias"],
                                row_map=rm)
  return out, ref


def bits(out):
  return dict(c=out["c"].cpu(), h=out["h"].cpu(), xh2=out["xh2"].view(torch.int16).cpu(), variant=out["variant"])


def ring_outputs(path):
  """Child side of the reference fixture: every case under this process's MVB_CELL_FORMAT_RINGS, saved to path."""
  res = {}
  for name, (kind, h, w, launch, seed) in sorted(CASES.items()):
    res[name] = bits(run_case(kind, h, w, sample_rows(h, w, launch), seed)[0])
  torch.save(res, path)


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


@pytest.fixture(scope="module")
def bf16x2_rings(dev, tmp_path_factory):
  """Outputs of every case with the bf16x2-sized rings, from a child interpreter."""
  path = str(tmp_path_factory.mktemp("rings") / "ref.pt")
  env = {k: v for k, v in os.environ.items() if not k.startswith("MVB_CELL_")}
  env["MVB_CELL_FORMAT_RINGS"] = "0"
  code = "import sys; sys.path[:0] = [%r, %r]; import test_cell_rings_gpu as t; t.ring_outputs(%r)" % (
      ROOT, TESTS, path)
  r = subprocess.run([sys.executable, "-B", "-c", code], env=env, cwd=ROOT, timeout=1800, capture_output=True,
                     text=True)
  assert r.returncode == 0, "reference child failed:\n%s\n%s" % (r.stdout[-3000:], r.stderr[-3000:])
  return torch.load(path)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_f16f8_rings_bit_identical(dev, bf16x2_rings, name):
  """Format-sized rings against the fp64 reference and bit for bit against the bf16x2-sized rings."""
  if os.environ.get("MVB_CELL_FORMAT_RINGS", "1") == "0":
    pytest.skip("MVB_CELL_FORMAT_RINGS=0 in this process: both runs would use the bf16x2 rings")
  kind, h, w, launch, seed = CASES[name]
  ns = sample_rows(h, w, launch)
  out, ref = run_case(kind, h, w, ns, seed)
  atsize.check_fwd("rings %s n%d" % (name, ns), ns, h, w, out, ref(), F16F8, pair=launch != "single")
  base = bf16x2_rings[name]
  assert base["variant"] == out["variant"]
  for k, a in bits(out).items():
    if k != "variant":
      assert torch.equal(a, base[k]), "%s: %s differs from the bf16x2-ring run" % (name, k)
