# coding=utf-8
"""The f16f8 cell kernel with an epilogue warpgroup (cell_fwd_epi_kernel, MVB_CELL_EPI_WG=1: at every launch size),
bit for bit against the kernel whose MMA warpgroups run the epilogue themselves (cell_fwd_kernel, MVB_CELL_EPI_WG=0).

The new kernel computes each accumulator over the same K order with the same passes (m64n128 instead of m64n256 MMAs,
which sum every output element alone) and hands it through shared memory to the unchanged epilogue functions, so
c', h', the next step's operands (f16f8 or bf16x2 planes) and the fan-out step's raw accumulators must be identical.
The library reads the variable once per process, so each kernel runs in a child interpreter.

Cases: every f16f8 launch variant of the product - plain, one-hot x-fold with a row map (beam steps), the fan-out
step (stage-1 accumulators and the children), the sparse and the dense x paths, h' written as bf16x2 planes - on the
product grids 36x18, 18x9, 18x32, on 4x62 (the 256-row A stage) and on an odd width (5x13), under the CTA-pair kernel
with an odd number of M tiles and under the single-CTA kernel with several tiles per CTA; no launch has a row count
that is a multiple of 128."""
import os
import subprocess
import sys

import pytest
import torch

import test_kernels_atsize_gpu as atsize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
F16F8 = 16
GRIDS = [(36, 18), (18, 9), (18, 32), (4, 62), (5, 13)]

# name -> (kind, h, w, launch, seed); launch "pair": the pair kernel with an odd number of M tiles, "single": the
# single-CTA kernel with about eight tiles per CTA
CASES = {}
for _i, (_h, _w) in enumerate(GRIDS):
  for _launch in ("pair", "single"):
    CASES["plain_%s_%dx%d" % (_launch, _h, _w)] = ("plain", _h, _w, _launch, 300 + 10 * _i)
CASES["hp_bf16x2_pair_36x18"] = ("hp_bf16x2", 36, 18, "pair", 350)
CASES["onehot_pair_36x18"] = ("onehot", 36, 18, "pair", 351)
CASES["onehot_single_18x9"] = ("onehot", 18, 9, "single", 352)
CASES["onehot_pair_18x32"] = ("onehot", 18, 32, "pair", 353)
CASES["fanout_pair_36x18"] = ("fanout", 36, 18, "pair", 354)
CASES["fanout_single_18x32"] = ("fanout", 18, 32, "single", 355)
CASES["xsparse_pair_36x18"] = ("xsparse", 36, 18, "pair", 356)
CASES["xsparse_single_18x9"] = ("xsparse", 18, 9, "single", 357)
CASES["xdense_pair_36x18"] = ("xdense", 36, 18, "pair", 358)
CASES["xdense_single_4x62"] = ("xdense", 4, 62, "single", 359)


def sample_rows(h, w, launch):
  if launch == "pair":
    return atsize.pair_ns(h, w, odd=True)
  ns = 1
  while atsize.m_tiles(ns + 1, h, w) < 2 * atsize.num_sms():
    ns += 1
  while atsize.halo_rows(ns, h, w) % atsize.BLOCK_M == 0:
    ns -= 1
  return ns


def run_case(kind, h, w, ns, seed):
  """One f16f8 cell launch on seeded inputs: every output buffer, raw bits."""
  from multiverse_b200 import ops
  dev = torch.device("cuda:0")
  cx = {"xsparse": 64, "xdense": 2}.get(kind, 32)
  if kind in ("onehot", "fanout"):
    d, ids, We, be, g = atsize._onehot_case(dev, ns, h, w, seed)
  else:
    d = atsize.cell_inputs(dev, ns, h, w, cx, seed=seed, x_scale=600.0 if kind == "xdense" else 1.0)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
  pk = ops.PackedCell(d["kernel"], d["bias"], F16F8)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, F16F8, dev)
  if kind in ("plain", "hp_bf16x2"):
    ops.nhwc_to_planes(d["x"], xh, 0, h, w)
  ops.nhwc_to_planes(d["h"], xh, pk.cxp, h, w)
  c_in = atsize.to_halo(d["c"])
  out = {}
  if kind == "fanout":
    k = 4
    ids = torch.randint(0, h * w, (ns * k,), generator=g, device=dev, dtype=torch.int32)
    xf = ops.XFold(d["kernel"], d["bias"], We, be)
    out["c"], out["h"] = ops.alloc_state(ns * k, h, w, dev), ops.alloc_state(ns * k, h, w, dev)
    out["preact"] = torch.full((atsize.halo_rows(ns, h, w), 1024), atsize.SENTINEL, device=dev)
    ops.cell_fwd_onehot_fanout(xh, pk, xf, ids, c_in, out["c"], out["h"], h, w, ns, k, workspace=out["preact"])
  else:
    out["c"], out["h"] = ops.alloc_state(ns, h, w, dev), ops.alloc_state(ns, h, w, dev)
    out["xh2"] = ops.alloc_xh(ns, h, w, pk.cpad, 2 if kind == "hp_bf16x2" else F16F8, dev)
    if kind in ("plain", "hp_bf16x2"):
      ops.cell_fwd(xh, pk, c_in, out["c"], out["h"], out["xh2"], h, w, ns)
    elif kind == "onehot":
      rm = torch.randint(0, ns, (ns,), generator=g, device=dev, dtype=torch.int32)
      xf = ops.XFold(d["kernel"], d["bias"], We, be)
      ops.cell_fwd_onehot(xh, pk, xf, ids, c_in, out["c"], out["h"], out["xh2"], h, w, ns, row_map=rm)
    elif kind == "xsparse":
      conv = torch.tanh(torch.randn((7, h * w, 64), generator=g, device=dev))
      frames = torch.randint(0, 7, (ns,), generator=g, device=dev, dtype=torch.int32)
      labels = torch.randint(-1, h * w + 1, (ns,), generator=g, device=dev, dtype=torch.int32)
      labels[:4] = torch.tensor([0, w - 1, (h - 1) * w, h * w - 1], dtype=torch.int32)
      table = torch.empty((ns, 9, 1024), device=dev)
      ops.cell_xsparse_table(conv, frames, labels, ops.XSparse(d["kernel"]), table, h, w)
      ops.cell_fwd_xsparse(xh, pk, table, labels, c_in, out["c"], out["h"], out["xh2"], h, w, ns)
    else:
      ops.cell_fwd_xdense(xh, pk, ops.XDense(d["kernel"]), d["x"].contiguous(), c_in, out["c"], out["h"], out["xh2"],
                          h, w, ns)
  res = {k: (v.view(torch.int16) if v.dtype == torch.bfloat16 else v.view(torch.int32)).cpu() for k, v in out.items()}
  res["variant"] = ops.cell_last_variant()
  return res


def epi_outputs(path):
  """Child side of the reference fixture: every case under this process's MVB_CELL_EPI_WG, saved to path."""
  res = {}
  for name, (kind, h, w, launch, seed) in sorted(CASES.items()):
    res[name] = run_case(kind, h, w, sample_rows(h, w, launch), seed)
  torch.save(res, path)


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def child_outputs(tmp_path_factory, epi_wg):
  """Outputs of every case under MVB_CELL_EPI_WG=epi_wg, from a child interpreter."""
  path = str(tmp_path_factory.mktemp("epi") / "out.pt")
  env = {k: v for k, v in os.environ.items() if not k.startswith("MVB_CELL_")}
  env["MVB_CELL_EPI_WG"] = epi_wg
  code = "import sys; sys.path[:0] = [%r, %r]; import test_cell_epi_wg_gpu as t; t.epi_outputs(%r)" % (
      ROOT, TESTS, path)
  r = subprocess.run([sys.executable, "-B", "-c", code], env=env, cwd=ROOT, timeout=1800, capture_output=True,
                     text=True)
  assert r.returncode == 0, "child with MVB_CELL_EPI_WG=%s failed:\n%s\n%s" % (epi_wg, r.stdout[-3000:],
                                                                                r.stderr[-3000:])
  return torch.load(path)


@pytest.fixture(scope="module")
def mma_epilogue(dev, tmp_path_factory):
  return child_outputs(tmp_path_factory, "0")


@pytest.fixture(scope="module")
def epi_warpgroup(dev, tmp_path_factory):
  return child_outputs(tmp_path_factory, "1")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_epilogue_warpgroup_bit_identical(dev, mma_epilogue, epi_warpgroup, name):
  kind, h, w, launch, seed = CASES[name]
  ns = sample_rows(h, w, launch)
  out = epi_warpgroup[name]
  base = mma_epilogue[name]
  pair = launch == "pair"
  assert out["variant"] == F16F8 * 2 + int(pair), (name, atsize.variant_name(out["variant"]))
  assert (atsize.m_tiles(ns, h, w) >= 2 * atsize.num_sms()) == pair
  assert atsize.halo_rows(ns, h, w) % atsize.BLOCK_M != 0
  assert base["variant"] == out["variant"]
  print("%s: %s, %d sample rows, %d M tiles" % (name, atsize.variant_name(out["variant"]), ns,
                                                atsize.m_tiles(ns, h, w)))
  for k, a in out.items():
    if k != "variant":
      assert torch.equal(a, base[k]), "%s: %s differs between the two kernels (%d of %d words)" % (
          name, k, int((a != base[k]).sum()), a.numel())
