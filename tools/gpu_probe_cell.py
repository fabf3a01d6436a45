# coding=utf-8
"""GPU probe: ConvLSTM cell kernel vs the numpy oracle under a set of ablations (debug aid)."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiverse_b200 import ops
from oracle import multiverse_ref as R

dev = torch.device("cuda:0")


def run_case(name, ns, h, w, cx, planes, mask=None, seed=0, zero_c=False):
  rng = np.random.default_rng(seed)
  ch = 256
  lim = np.sqrt(6.0 / (9 * (cx + ch) + 9 * 4 * ch))
  kernel = rng.uniform(-lim, lim, size=(3, 3, cx + ch, 4 * ch)).astype(np.float32)
  biases = (rng.standard_normal(4 * ch) * 0.1).astype(np.float32)
  x = rng.standard_normal((ns, h, w, cx)).astype(np.float32)
  hh = np.tanh(rng.standard_normal((ns, h, w, ch))).astype(np.float32)
  c = rng.standard_normal((ns, h, w, ch)).astype(np.float32)
  if mask is not None:
    kernel = mask(kernel)
  c_ref, h_ref = R.convlstm_cell(x.astype(np.float64), (c * (0 if zero_c else 1)).astype(np.float64),
                                 hh.astype(np.float64), kernel.astype(np.float64), biases.astype(np.float64))
  pk = ops.PackedCell(torch.from_numpy(kernel).to(dev), torch.from_numpy(biases).to(dev), planes)
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  xh2 = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  ops.nhwc_to_planes(torch.from_numpy(x).to(dev), xh, 0, h, w)
  ops.nhwc_to_planes(torch.from_numpy(hh).to(dev), xh, pk.cxp, h, w)
  c_in = ops.alloc_state(ns, h, w, dev)
  ops.nhwc_to_halo(torch.from_numpy(c).to(dev), c_in, h, w)
  c_out = ops.alloc_state(ns, h, w, dev)
  h_out = ops.alloc_state(ns, h, w, dev)
  ops.cell_fwd(xh, pk, None if zero_c else c_in, c_out, h_out, xh2, h, w, ns)
  torch.cuda.synchronize()
  co = torch.empty((ns, h, w, ch), device=dev); ho = torch.empty((ns, h, w, ch), device=dev)
  ops.halo_to_nhwc(c_out, co, h, w); ops.halo_to_nhwc(h_out, ho, h, w)
  co, ho = co.cpu().numpy().astype(np.float64), ho.cpu().numpy().astype(np.float64)
  ec = np.abs(co - c_ref).max() / np.abs(c_ref).max()
  eh = np.abs(ho - h_ref).max() / np.abs(h_ref).max()
  # planes of h' written into xh2's h block must sum back to h'
  hp = xh2[:, :, pk.cxp:].float().sum(0).view(ns, h + 1, w + 1, ch)[:, :h, :w].cpu().numpy()
  ep = np.abs(hp - ho).max()
  halo_clean = float(xh2.float().view(2, ns, h + 1, w + 1, -1)[:, :, h].abs().max() +
                     xh2.float().view(2, ns, h + 1, w + 1, -1)[:, :, :, w].abs().max())
  print("%-28s ns=%d %dx%d cx=%d P=%d  rel_err c=%.3e h=%.3e  plane_sum_err=%.2e halo=%g"
        % (name, ns, h, w, cx, planes, ec, eh, ep, halo_clean), flush=True)
  return ec, eh


def only_tap(t):
  def f(k):
    k2 = np.zeros_like(k); k2[t // 3, t % 3] = k[t // 3, t % 3]; return k2
  return f


def only_x(cx):
  def f(k):
    k2 = k.copy(); k2[:, :, cx:] = 0; return k2
  return f


if __name__ == "__main__":
  print(torch.cuda.get_device_name(0))
  run_case("random", 2, 36, 18, 32, 2)
  run_case("center tap only", 2, 36, 18, 32, 2, only_tap(4))
  run_case("tap 0 only", 2, 36, 18, 32, 2, only_tap(0))
  run_case("tap 8 only", 2, 36, 18, 32, 2, only_tap(8))
  run_case("x part only", 2, 36, 18, 32, 2, only_x(32))
  run_case("zero c", 2, 36, 18, 32, 2, None, zero_c=True)
  run_case("enc class cx=64", 3, 36, 18, 64, 2)
  run_case("enc reg cx=2", 3, 18, 9, 2, 2)
  run_case("native 18x32", 2, 18, 32, 32, 2)
  run_case("multi-tile ns=9", 9, 36, 18, 32, 2)
  # timing at config-2 size
  ns, h, w, cx = 64, 36, 18, 32
  for planes in (2, ops.PLANES_F16F8):
    pk = ops.PackedCell(torch.randn(3, 3, cx + 256, 1024, device=dev) * 0.02, torch.zeros(1024, device=dev), planes)
    xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
    ops.nhwc_to_planes(torch.randn(ns, h, w, cx + 256, device=dev), xh, 0, h, w)
    xh2 = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
    c_in = ops.alloc_state(ns, h, w, dev); c_out = ops.alloc_state(ns, h, w, dev); h_out = ops.alloc_state(ns, h, w, dev)
    for _ in range(3):
      ops.cell_fwd(xh, pk, c_in, c_out, h_out, xh2, h, w, ns)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
      ops.cell_fwd(xh, pk, c_in, c_out, h_out, xh2, h, w, ns)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    fl = 2.0 * ns * h * w * 9 * (cx + 256) * 1024
    print("timing ns=%d P=%d: %.3f ms/step  %.1f algorithmic TFLOP/s" % (ns, planes, ms, fl / ms / 1e9), flush=True)
