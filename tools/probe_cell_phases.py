# coding=utf-8
"""Where the clocks of the f16f8 cell kernel go: phase profile per warpgroup (GPU).

  python tools/probe_cell_phases.py [--lib PATH] [--reps N] [--compare]

Builds the library with -DMVB_CELL_PROBE into a temporary directory (or loads PATH, a library built that way by
multiverse_b200.build.build_variant) and runs the class-decoder cell - x-fold, row map, c in, h' out, the launch
of every beam step after the first - with the pair kernel on three grids: the c4 beam step (10 240 sample rows of
36x18), 18x32 and 18x9.  In the probe build every warpgroup's first thread sums clock64() per phase:
  MMA warpgroups:  waiting for a weight slot (full_bar), for an A stage (afull_bar), in wgmma.wait_group, in the
                   epilogue (state update and stores; with the epilogue warpgroup: the copy of the accumulators into
                   the staging buffer), waiting for the staging buffer to be free, and the rest (descriptors, MMA
                   issue, barrier arrivals);
  TMA producer:    waiting for a free weight slot (empty_bar), for a free A stage (aempty_bar), the rest;
  epilogue warpgroup (cell_fwd_epi_kernel only): waiting for a staged tile, and the rest (the epilogue).
Shares are of each role's total cycles.  The clocks of a launch are the consumer cycles per warpgroup over the
event-timed launch time.  --compare runs it once per kernel (MVB_CELL_EPI_WG=0: the MMA warpgroups run the
epilogue; 1: the epilogue warpgroup does) in child processes.  The probe build adds clock reads to the mainloop, so its launch times are a little longer than the
product's; the shares are what it is for.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# CellProbePhase (csrc/mvb_cell.cu), then the ring of the last launch
PHASES = ["full_wait", "afull_wait", "mma_wait", "epilogue", "consumer", "empty_wait", "aempty_wait", "producer",
          "free_wait", "staged_wait", "epi_busy", "tiles"]
SHAPES = [("c4 beam step", 36, 18, 10240), ("18x32", 18, 32, 4096), ("18x9", 18, 9, 10240)]
MMA_CLOCKS_PER_SLOT = 1024     # one weight slot of 256 columns: 4 m64n256 MMAs per warpgroup, k16 fp16 or k32 e4m3


def card():
  import torch
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60)
    return r.stdout.strip() or torch.cuda.get_device_name()
  except (OSError, subprocess.SubprocessError):
    return torch.cuda.get_device_name() + " (nvidia-smi unavailable: power limit not read)"


def run(lib_path, reps):
  import torch
  from multiverse_b200 import _lib
  _lib.LIB_PATH = lib_path
  lib = _lib.load()
  probe = lib.mvb_cell_probe
  probe.argtypes = [C.c_void_p, C.c_int]
  buf = (C.c_ulonglong * (len(PHASES) + 3))()
  _lib.check(probe(buf, 1), "mvb_cell_probe")
  from multiverse_b200 import ops
  dev = torch.device("cuda:0")
  rings = os.environ.get("MVB_CELL_FORMAT_RINGS", "1")
  epi_wg = os.environ.get("MVB_CELL_EPI_WG", "1") != "0" and rings != "0"
  print("card: %s; SMs %d; rings: %s; %s" % (
      card(), torch.cuda.get_device_properties(0).multi_processor_count,
      "bf16x2-sized (MVB_CELL_FORMAT_RINGS=0)" if rings == "0" else "format-sized",
      "epilogue warpgroup (128-column tiles)" if epi_wg else "epilogue on the MMA warpgroups (MVB_CELL_EPI_WG=0)"),
        flush=True)
  cols = 128 if epi_wg else 256      # columns of an N tile
  cx = 32
  g = torch.Generator(device=dev)
  g.manual_seed(7)
  kernel = (torch.rand((3, 3, cx + 256, 1024), generator=g, device=dev) * 2 - 1) * 0.02
  bias = torch.randn(1024, generator=g, device=dev) * 0.1
  pk = ops.PackedCell(kernel, bias, ops.PLANES_F16F8)
  xf = ops.XFold(kernel, bias, torch.randn((3, 3, 1, cx), generator=g, device=dev) * 0.5,
                 torch.randn(cx, generator=g, device=dev) * 0.1)
  for tag, h, w, ns in SHAPES:
    xh = ops.alloc_xh(ns, h, w, pk.cpad, ops.PLANES_F16F8, dev)
    ops.nhwc_to_planes(torch.tanh(torch.randn((ns, h, w, 256), generator=g, device=dev)), xh, pk.cxp, h, w)
    ids = torch.randint(0, h * w, (ns,), generator=g, device=dev, dtype=torch.int32)
    row_map = torch.randperm(ns, generator=g, device=dev).to(torch.int32)
    c_in = ops.alloc_state(ns, h, w, dev)
    c_in.normal_(generator=g)
    c_out, h_out = ops.alloc_state(ns, h, w, dev), ops.alloc_state(ns, h, w, dev)
    step = lambda: ops.cell_fwd_onehot(xh, pk, xf, ids, c_in, c_out, h_out, None, h, w, ns, row_map=row_map)
    for _ in range(2):
      step()
    assert ops.cell_last_variant() == ops.PLANES_F16F8 * 2 + 1, "the pair kernel did not run"
    _lib.check(probe(buf, 1), "mvb_cell_probe")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
      step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    _lib.check(probe(buf, 1), "mvb_cell_probe")
    v = dict(zip(PHASES, list(buf)[:len(PHASES)]))
    b_slots, a_stages, a_stage_bytes = list(buf)[len(PHASES):]
    ctas = torch.cuda.get_device_properties(0).multi_processor_count // 2 * 2
    cons, prod = float(v["consumer"]), float(v["producer"])
    ghz = cons / (2 * ctas * reps) / (ms * 1e6)
    wg_tiles = v["tiles"] / (2 * ctas)          # tiles per warpgroup (= per CTA), over the reps
    clk_tile = cons / v["tiles"] * (256 // cols)      # per 128 x 256 of work
    ideal = 8 * 9 * MMA_CLOCKS_PER_SLOT          # x-fold: 4 h chunks x 2 passes x 9 taps
    other_c = cons - sum(v[k] for k in ("full_wait", "afull_wait", "mma_wait", "epilogue", "free_wait"))
    other_p = prod - v["empty_wait"] - v["aempty_wait"]
    pct = lambda x, tot: 100.0 * x / tot
    print("%s: %d sample rows of %dx%d, %d M tiles; rings %d weight slots + %d A stages of %d B; %.2f ms/launch, "
          "%.2f GHz effective SM clock, %.1f tiles per CTA, %.0f clocks per 128x256 of work (%.0f tensor clocks: %.2f)"
          % (tag, ns, h, w, -(-ops.halo_rows(ns, h, w) // 128), b_slots, a_stages, a_stage_bytes, ms, ghz,
             wg_tiles / reps, clk_tile, ideal, ideal / clk_tile))
    print("  MMA warpgroups: full_bar wait %.1f%%, afull_bar wait %.1f%%, wgmma wait %.1f%%, epilogue %.1f%%, "
          "staging-free wait %.1f%%, issue/other %.1f%%"
          % (pct(v["full_wait"], cons), pct(v["afull_wait"], cons), pct(v["mma_wait"], cons), pct(v["epilogue"], cons),
             pct(v["free_wait"], cons), pct(other_c, cons)))
    if epi_wg:
      epi = float(v["staged_wait"] + v["epi_busy"])
      print("  epilogue warpgroup: staged wait %.1f%%, epilogue %.1f%% (%.0f clocks per tile)"
            % (pct(v["staged_wait"], epi), pct(v["epi_busy"], epi), v["epi_busy"] / max(v["tiles"] / 2, 1)))
    print("  TMA producer:   empty_bar wait %.1f%%, aempty_bar wait %.1f%%, issue/other %.1f%%"
          % (pct(v["empty_wait"], prod), pct(v["aempty_wait"], prod), pct(other_p, prod)), flush=True)
    del xh, ids, row_map, c_in, c_out, h_out
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--lib", default=None, help="a library built with MVB_CELL_PROBE (default: build one now)")
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--compare", action="store_true", help="run once per kernel (MVB_CELL_EPI_WG=0, 1), in child processes")
  args = ap.parse_args()
  tmp = None
  if args.lib is None:
    from multiverse_b200 import build
    tmp = tempfile.TemporaryDirectory(prefix="mvb_probe_")
    args.lib = build.build_variant(tmp.name, ["MVB_CELL_PROBE"])
  if args.compare:
    for epi_wg in ("0", "1"):
      env = dict(os.environ, MVB_CELL_EPI_WG=epi_wg)
      r = subprocess.run([sys.executable, "-B", os.path.abspath(__file__), "--lib", args.lib, "--reps",
                          str(args.reps)], env=env, cwd=ROOT)
      if r.returncode:
        sys.exit(r.returncode)
  else:
    run(args.lib, args.reps)
  if tmp is not None:
    tmp.cleanup()


if __name__ == "__main__":
  main()
