# coding=utf-8
"""GPU probe: time of one class-decoder-sized cell launch per operand format (debug / tuning aid).
usage: python tools/gpu_probe_cell_time.py [ns] [planes ...]   (env: MVB_CELL_MULTICAST)"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiverse_b200 import ops
dev = torch.device("cuda:0")
ns = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
planes_list = [int(a) for a in sys.argv[2:]] or [2, 16]
h, w, cx = 36, 18, 32
for planes in planes_list:
  pk = ops.PackedCell(torch.randn(3, 3, cx + 256, 1024, device=dev) * 0.02, torch.zeros(1024, device=dev), planes)
  xf = ops.XFold(torch.randn(3, 3, cx + 256, 1024, device=dev) * 0.02, torch.zeros(1024, device=dev),
                 torch.randn(3, 3, 1, 32, device=dev), torch.zeros(32, device=dev))
  xh = ops.alloc_xh(ns, h, w, pk.cpad, planes, dev)
  hsrc = torch.tanh(torch.randn(ns, h, w, 256, device=dev))
  ops.nhwc_to_planes(hsrc, xh, pk.cxp, h, w)
  ids = torch.randint(0, h * w, (ns,), dtype=torch.int32, device=dev)
  c_in = ops.alloc_state(ns, h, w, dev); c_out = ops.alloc_state(ns, h, w, dev); h_out = ops.alloc_state(ns, h, w, dev)
  for _ in range(3):
    ops.cell_fwd_onehot(xh, pk, xf, ids, c_in, c_out, h_out, None, h, w, ns)
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  reps = 8
  e0.record()
  for _ in range(reps):
    ops.cell_fwd_onehot(xh, pk, xf, ids, c_in, c_out, h_out, None, h, w, ns)
  e1.record(); torch.cuda.synchronize()
  ms = e0.elapsed_time(e1) / reps
  fl = 2.0 * ns * h * w * 9 * (cx + 256) * 1024
  print("ns=%d planes=%d variant=%d mc=%s: %.3f ms/launch  %.1f algorithmic TFLOP/s" %
        (ns, planes, ops.cell_last_variant(), os.environ.get("MVB_CELL_MULTICAST", "1"), ms, fl / ms / 1e9), flush=True)
  del pk, xf, xh, hsrc, c_in, c_out, h_out
