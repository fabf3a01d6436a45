# coding=utf-8
"""Numerics gate for the sliced-int8 ConvLSTM cell (VERDICT r1, item 3a).  CPU only.

Runs the oracle's torch port in fp64 with the cell's contraction replaced by an exact emulation of
each candidate tensor-core scheme, through the 20-step greedy two-scale rollout and the 12-step
K=20 diverse-beam rollout of tests/cases.py, and reports the error of what the caller fetches
(logits, offsets, beam ids / log-probs) against the unmodified fp64 run.

Schemes (operands a = concat[x,h], b = kernel; everything else fp64 so only the scheme shows):
  bf16x2   a=a0+a1, b=b0+b1 (bf16 planes), a0b0+a0b1+a1b0          3 bf16 passes  (round-1 kernel)
  i8x2     16-bit fixed point, q = 256*hi + lo, hi,lo in [-128,127] (signed low digit),
           per-launch activation scale 1/32639 (2/32639 if |a| can reach 2: graph-attended h),
           per-output-column weight scale; hh + (hl + lh), ll dropped   3 int8 passes = 1.5 bf16
  i8x2_15  same with a 7-bit low digit (the judge's 15-bit proposal)
  f16f8    a=a0+a1, b=b0+b1 with a0,b0 fp16 (weights scaled per column by 2^S so that the fp16 and
           e4m3 ranges fit): a0*b0 in fp16 + e4m3(a0)*e4m3(b1) + e4m3(a1*2^12)*e4m3(b0*2^-12) in fp8
           -- all three into ONE fp32 accumulator: 1 + 2*0.5 = 2 bf16-pass equivalents
  fp16x2   a=a0+a1 (fp16), b=b0 only: a0b0 + a1b0                      2 fp16 passes (for the record)
The regression encoder's 2-channel pixel-offset block (+-1.9e3) stays exact in every scheme (the
kernel keeps it on the compensated bf16 path / fp32), and so does the class decoder's folded
one-hot embedding block (exact fp32 table rows in the epilogue).
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
from oracle import multiverse_ref as R  # noqa: E402
from oracle import multiverse_ref_torch as T  # noqa: E402

D = torch.float64


def bf16_split(t):
  p0 = t.to(torch.bfloat16).to(D)
  p1 = (t - p0).to(torch.bfloat16).to(D)
  return p0, p1


def fp16_split(t):
  p0 = t.to(torch.float16).to(D)
  p1 = (t - p0).to(torch.float16).to(D)
  return p0, p1


def fixed_split(t, scale, lo_bits):
  q = torch.round(t / scale)
  base = 1 << lo_bits
  lo = torch.remainder(q + base // 2, base) - base // 2
  hi = (q - lo) / base
  assert float(hi.abs().max()) <= 128 and float(hi.min()) >= -128 and float(hi.max()) <= 127, \
      (float(hi.min()), float(hi.max()))
  return hi, lo, base


def make_cell(scheme, exact_x_kernels):
  conv = T.conv2d_same

  def cell(x, c, h, kernel, biases, forget_bias=1.0):
    cx = x.shape[-1]
    a = torch.cat([x, h], dim=-1)
    if scheme == "exact":
      g = conv(a, kernel)
    else:
      x_exact = kernel.data_ptr() in exact_x_kernels
      gx = conv(x, kernel[:, :, :cx]) if x_exact else 0.0
      aa = h if x_exact else a
      kk = kernel[:, :, cx:] if x_exact else kernel
      if scheme == "bf16x2":
        a0, a1 = bf16_split(aa); b0, b1 = bf16_split(kk)
        g = conv(a0, b0) + conv(a0, b1) + conv(a1, b0)
      elif scheme == "f16f8":
        # per-column power-of-two weight scale: max |w_col| * 2^S in [2^13, 2^14)
        wmax = kk.abs().amax(dim=(0, 1, 2), keepdim=True)
        S = 13 - torch.floor(torch.log2(wmax))
        ks = kk * torch.pow(2.0, S)
        a0 = aa.to(torch.float16).to(D); a1 = aa - a0
        b0 = ks.to(torch.float16).to(D); b1 = ks - b0
        e4 = lambda t: t.to(torch.float32).to(torch.float8_e4m3fn).to(D)
        g = conv(a0, b0) + conv(e4(a0), e4(b1)) + conv(e4(a1 * 4096.0), e4(b0 / 4096.0))
        g = g * torch.pow(2.0, -S).reshape(1, 1, 1, -1)
      elif scheme == "fp16x2":
        a0, a1 = fp16_split(aa); b0, _ = fp16_split(kk)
        g = conv(a0, b0) + conv(a1, b0)
      elif scheme in ("i8x2", "i8x2_15"):
        lo_bits = 8 if scheme == "i8x2" else 7
        amax = float(aa.abs().max())
        qmax = 127 * (1 << lo_bits) + (1 << lo_bits) // 2 - 1      # 32639: largest q with hi <= 127
        sa = (2.0 if amax > 1.0 else 1.0) / qmax
        assert amax <= 2.0
        wmax = kk.abs().amax(dim=(0, 1, 2), keepdim=True)
        sb = wmax / qmax
        ah, al, base = fixed_split(aa, sa, lo_bits)
        bh, bl, _ = fixed_split(kk / sb, 1.0, lo_bits)
        hh = conv(ah, bh)
        cross = conv(ah, bl) + conv(al, bh)
        g = (hh * (base * base) + cross * base) * (sa * sb.reshape(1, 1, 1, -1))
      else:
        raise ValueError(scheme)
      g = g + gx
    g = g + biases
    gi, gj, gf, go = torch.split(g, g.shape[-1] // 4, dim=-1)
    new_c = torch.sigmoid(gf + forget_bias) * c + torch.sigmoid(gi) * torch.tanh(gj)
    return new_c, torch.tanh(new_c) * torch.sigmoid(go)
  return cell


def run(name, scheme):
  over, seed = cases.ROLLOUTS[name]
  cfg = R.default_config(**over)
  w = R.make_weights(cfg, seed)
  f = R.make_inputs(cfg, seed)
  wt = {k: torch.from_numpy(np.ascontiguousarray(v)).to(D) for k, v in w.items()}
  exact = set()
  for k, v in wt.items():
    if "enc_grid_regress" in k and k.endswith("kernel"):
      exact.add(v.data_ptr())
    if "decoder_grid_class" in k and k.endswith("kernel"):
      exact.add(v.data_ptr())
  old = T.convlstm_cell
  T.convlstm_cell = make_cell(scheme, exact)
  try:
    with torch.no_grad():
      out = T._forward(cfg, wt, f, D)
  finally:
    T.convlstm_cell = old
  return cfg, out


def rel(a, b):
  a = a.numpy() if torch.is_tensor(a) else a
  b = b.numpy() if torch.is_tensor(b) else b
  return float(np.abs(a - b).max() / np.abs(b).max())


SCHEMES = tuple(os.environ.get("GATE_SCHEMES", "bf16x2,f16f8,i8x2,i8x2_15,fp16x2").split(","))


def main():
  res = {}
  for name in ("greedy_two_scale", "beam_k20_diverse", "greedy_native_18x32"):
    cfg, ref = run(name, "exact")
    row = {}
    for scheme in SCHEMES:
      _, out = run(name, scheme)
      r = {}
      for i in range(len(cfg.scene_grids)):
        if not cfg.use_grids[i]:
          continue
        r["logits_%d" % i] = rel(out["grid_pred_decoded"][i], ref["grid_pred_decoded"][i])
        r["reg_%d" % i] = rel(out["grid_pred_reg_decoded"][i], ref["grid_pred_reg_decoded"][i])
        a = out["grid_pred_decoded"][i].reshape(cfg.batch_size, cfg.pred_len, -1).argmax(-1)
        b = ref["grid_pred_decoded"][i].reshape(cfg.batch_size, cfg.pred_len, -1).argmax(-1)
        r["argmax_equal_%d" % i] = bool((a == b).all())
      if ref["beam_outputs"] is not None:
        r["beam_ids_equal"] = bool(np.array_equal(out["beam_outputs"][1], ref["beam_outputs"][1]))
        r["beam_logits"] = rel(out["beam_outputs"][0], ref["beam_outputs"][0])
        r["beam_logprob_abs"] = float(np.abs(out["beam_outputs"][2] - ref["beam_outputs"][2]).max())
      row[scheme] = r
      print(name, scheme, json.dumps(r), flush=True)
    res[name] = row
  out = sys.argv[1] if len(sys.argv) > 1 else None          # python tools/numerics_gate.py [RESULT.json]
  if out:
    with open(out, "w") as fh:
      json.dump(res, fh, indent=1)
  else:
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
  torch.set_num_threads(8)
  main()
