# coding=utf-8
"""Thin torch-tensor wrappers over the C ABI (one per entry point of include/multiverse_b200.h).

PyTorch only owns memory and streams here; every computation is a kernel of
libmultiverse_b200.so.  All tensors must be contiguous CUDA tensors on the current device.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib

HIDDEN = 256
# the two operand formats (`planes` codes): two bf16 summands, and MVB_PLANES_F16F8, one fp16 + two e4m3 planes in the
# bytes of two bf16 planes (inference)
PLANES_BF16X2 = 2
PLANES_F16F8 = 16


def planes_of(t):
  """`planes` code of an operand buffer made by alloc_xh (bf16 planes: its leading dimension)."""
  return getattr(t, "mvb_planes", t.shape[0])


def cell_variants_seen(reset=False):
  """Set of (planes, pair) cell-kernel variants launched since the last reset."""
  m = int(_lib.load().mvb_cell_variants_seen(int(bool(reset))))
  return {((PLANES_BF16X2, PLANES_F16F8)[b // 2], bool(b % 2)) for b in range(4) if m >> b & 1}


def cell_last_variant():
  """planes * 2 + multicast of the cell kernel launched last (-1: none yet)."""
  return int(_lib.load().mvb_cell_last_variant())


def _p(t):
  if t is None:
    return None
  assert t.is_cuda and t.is_contiguous(), "expected a contiguous CUDA tensor"
  return C.c_void_p(t.data_ptr())


def _stream():
  return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def halo_rows(ns, h, w):
  """Rows of the halo layout for ns sample rows of an h x w grid."""
  return ns * (h + 1) * (w + 1)


def cell_cpad(cx):
  return (cx + 31) // 32 * 32 + HIDDEN


def launch_count():
  return int(_lib.load().mvb_launch_count())


def reset_launch_count():
  _lib.load().mvb_reset_launch_count()


class PackedCell(object):
  """Device-resident packed weights of one ConvLSTM cell (see mvb_pack_cell_weights)."""

  def __init__(self, kernel, biases, planes=PLANES_BF16X2, comp=False):
    assert kernel.dim() == 4 and kernel.shape[0] == 3 and kernel.shape[1] == 3
    assert kernel.shape[3] == 4 * HIDDEN
    self.cx = int(kernel.shape[2]) - HIDDEN
    self.cpad = cell_cpad(self.cx)
    self.cxp = self.cpad - HIDDEN
    self.planes = planes
    self.comp = bool(comp) and planes == PLANES_BF16X2 and 4 * self.cx <= self.cxp
    kernel = kernel.detach().to(torch.float32).contiguous()
    biases = biases.detach().to(torch.float32).contiguous()
    if planes == PLANES_F16F8:
      # [fp16 1024 x 9cpad][e4m3 2 x 1024 x 9cpad][fp32 1024 column scales]
      self.w = torch.empty((4 * 4 * HIDDEN * 9 * self.cpad + 4 * 4 * HIDDEN,), dtype=torch.uint8,
                           device=kernel.device)
    else:
      self.w = torch.empty((planes, 4 * HIDDEN, 9 * self.cpad), dtype=torch.bfloat16,
                           device=kernel.device)
    self.bias = torch.empty((4 * HIDDEN,), dtype=torch.float32, device=kernel.device)
    _lib.call("mvb_pack_cell_weights", _p(kernel), _p(biases), _p(self.w), _p(self.bias),
              self.cx, planes, int(self.comp), _stream())


def _planes_arg(packed, xh_next):
  """`planes` argument of the cell entry points: format of inputs/weights | (format of hp_out << 8) if it differs."""
  po = packed.planes if xh_next is None else planes_of(xh_next)
  return packed.planes if po == packed.planes else packed.planes | (po << 8)


def _hp_out(xh, packed, xh_next):
  """Checks that `xh` is in the operand format of `packed`, and returns the h-output arguments of the cell entry
  points: the planes xh_next whose h block receives h' (pointer, plane stride, row pitch, channel offset), or none."""
  assert xh.shape[2] == packed.cpad and planes_of(xh) == packed.planes
  if xh_next is None:
    return None, 0, 0, 0
  return _p(xh_next), xh_next.stride(0), xh_next.shape[2], xh_next.shape[2] - HIDDEN


def alloc_xh(ns, h, w, cpad, planes, device):
  """Zeroed operand planes [2, R, cpad] (either format: the same bytes); halo cells and channel padding must stay
  zero."""
  t = torch.zeros((2, halo_rows(ns, h, w), cpad), dtype=torch.bfloat16, device=device)
  if planes == PLANES_F16F8:
    t.mvb_planes = PLANES_F16F8
  return t


def operand_values(xh):
  """fp32 values [R, cpad] an operand buffer represents (sum of its bf16 planes, or a0 + a1 of the f16f8 format),
  plus, for f16f8, the e4m3 copy of a0 (else None).  Diagnostic / test helper: views and casts only."""
  if planes_of(xh) != PLANES_F16F8:
    return xh.float().sum(0), None
    # pylint: disable=unreachable
  r, cpad = xh.shape[1], xh.shape[2]
  raw = xh.view(torch.uint8).reshape(-1)
  n = r * cpad
  a0 = raw[:2 * n].view(torch.float16).reshape(r, cpad).float()
  f8 = raw[2 * n:].view(torch.float8_e4m3fn).reshape(r, 2 * cpad).float()
  # inside an fp8 row, per 64-channel chunk of the x block [e0 (64) | e1 (64)] (a trailing 32-channel chunk:
  # [e0 (32) | e1 (32)]), then per 64 channels of the h block [e0 (64) | e1 (64)] (mvb_common.cuh f8_off)
  cxp = cpad - HIDDEN
  c = torch.arange(cpad, device=xh.device)
  c0 = torch.where(c >= cxp, cxp + (c - cxp) // 64 * 64, c // 64 * 64)     # first channel of c's chunk
  width = torch.where(c >= cxp, 64, (cxp - c0).clamp(max=64))
  off0 = 2 * c0 + (c - c0)
  off1 = off0 + width
  return a0 + f8[:, off1] / 4096.0, f8[:, off0]


def alloc_state(ns, h, w, device, zero=True):
  f = torch.zeros if zero else torch.empty
  return f((halo_rows(ns, h, w), HIDDEN), dtype=torch.float32, device=device)


def cell_fwd(xh, packed, c_in, c_out, h32_out, xh_next, h, w, ns, row_map=None,
             forget_bias=1.0):
  """One ConvLSTM step.  xh_next: operand planes whose h block (channel offset = its cxp)
  receives the bf16 planes of h', or None."""
  hp = _hp_out(xh, packed, xh_next)
  _lib.call("mvb_convlstm_cell_fwd", _p(xh), _p(packed.w), _p(packed.bias), _p(c_in), _p(row_map), _p(c_out),
            _p(h32_out), *hp, ns, h, w, packed.cpad, _planes_arg(packed, xh_next), float(forget_bias), _stream())


class XDense(object):
  """fp32 weights [18, 1024] of the dense x path of a regression-encoder cell (mvb_cell_xdense_weights)."""

  def __init__(self, kernel):
    assert kernel.dim() == 4 and kernel.shape[2] == 2 + HIDDEN, "the dense x path is for 2-channel inputs"
    self.W = torch.empty((18, 4 * HIDDEN), dtype=torch.float32, device=kernel.device)
    _lib.call("mvb_cell_xdense_weights", _p(kernel.detach().float().contiguous()), _p(self.W), _stream())


def cell_fwd_xdense(xh, packed, xdense, x_in, c_in, c_out, h32_out, xh_next, h, w, ns, forget_bias=1.0):
  """One ConvLSTM step of the regression encoder: h block of `xh` through the tensor cores, the raw 2-channel input
  x_in fp32 [ns,h,w,2] added in fp32 in the epilogue (mvb_convlstm_cell_fwd_xdense); the x block of xh is not read."""
  hp = _hp_out(xh, packed, xh_next)
  assert x_in.dtype == torch.float32 and x_in.is_contiguous() and x_in.numel() == ns * h * w * 2
  _lib.call("mvb_convlstm_cell_fwd_xdense", _p(xh), _p(packed.w), _p(packed.bias), _p(x_in), _p(xdense.W), _p(c_in),
            _p(c_out), _p(h32_out), *hp, ns, h, w, packed.cpad, _planes_arg(packed, xh_next), float(forget_bias),
            _stream())


class XSparse(object):
  """fp32 weights [9 * 64, 1024] of the sparse x path of a class-encoder cell (mvb_cell_xsparse_weights)."""

  def __init__(self, kernel):
    assert kernel.dim() == 4 and kernel.shape[2] == 64 + HIDDEN, "the sparse x path is for the 64 scene channels"
    self.W = torch.empty((9 * 64, 4 * HIDDEN), dtype=torch.float32, device=kernel.device)
    _lib.call("mvb_cell_xsparse_weights", _p(kernel.detach().float().contiguous()), 64, _p(self.W), _stream())


def cell_xsparse_table(scene_conv, frame_idx, label, xsparse, table, h, w):
  """table fp32 [ns, 9, 1024] <- the nine x products of every sample row (features at its label cell)."""
  _lib.call("mvb_cell_xsparse_table", _p(scene_conv), _p(frame_idx), _p(label), _p(xsparse.W), _p(table),
            label.shape[0], h, w, _stream())


def cell_fwd_xsparse(xh, packed, table, label, c_in, c_out, h32_out, xh_next, h, w, ns, forget_bias=1.0):
  """One ConvLSTM step of the class encoder: h block of `xh` through the tensor cores, the one-cell scene-feature
  input added from `table` (cell_xsparse_table) in the epilogue; the x block of xh is not read."""
  hp = _hp_out(xh, packed, xh_next)
  _lib.call("mvb_convlstm_cell_fwd_xsparse", _p(xh), _p(packed.w), _p(packed.bias), _p(table), _p(label), _p(c_in),
            _p(c_out), _p(h32_out), *hp, ns, h, w, packed.cpad, _planes_arg(packed, xh_next), float(forget_bias),
            _stream())


class XFold(object):
  """Look-up tables that replace the embedded one-hot input of a class-decoder cell."""

  def __init__(self, kernel, biases, We, be):
    dev = kernel.device
    self.B = torch.empty((9, 4 * HIDDEN), dtype=torch.float32, device=dev)
    self.T2 = torch.empty((9, 25, 4 * HIDDEN), dtype=torch.float32, device=dev)
    _lib.call("mvb_cell_xfold_tables", _p(kernel.detach().float().contiguous()),
              _p(biases.detach().float().contiguous()), _p(We), _p(be), We.shape[3], _p(self.B),
              _p(self.T2), _stream())


def cell_fwd_onehot(xh, packed, xf, ids, c_in, c_out, h32_out, xh_next, h, w, ns, row_map=None,
                    forget_bias=1.0, tiles=None):
  """Class-decoder step with the embedded one-hot input folded into table look-ups.  tiles: (list, count) work list
  of beam_band (only its rows are computed and written), or None (every row)."""
  hp = _hp_out(xh, packed, xh_next)
  tl, tn = tiles if tiles is not None else (None, None)
  _lib.call("mvb_convlstm_cell_fwd_onehot", _p(xh), _p(packed.w), _p(xf.B), _p(xf.T2), _p(ids), _p(c_in),
            _p(row_map), _p(tl), _p(tn), _p(c_out), _p(h32_out), *hp, ns, h, w, packed.cpad,
            _planes_arg(packed, xh_next), float(forget_bias), _stream())


def cell_fwd_onehot_fanout(xh, packed, xf, ids, c_in, c_out, h32_out, h, w, ns, fanout, forget_bias=1.0,
                           workspace=None):
  """First K-row beam step: GEMM on the `ns` parent rows (raw accumulators to `workspace` fp32 [ns*S, 1024]), then
  the children kernel emits ns*fanout child rows (ids [ns*fanout]).  xh None: `workspace` holds the accumulators of
  an earlier call on the same parents; only the children are emitted."""
  assert xh is None and workspace is not None or xh.shape[2] == packed.cpad and planes_of(xh) == packed.planes
  if workspace is None:
    workspace = torch.empty((halo_rows(ns, h, w), 4 * HIDDEN), dtype=torch.float32, device=xh.device)
  assert workspace.numel() >= halo_rows(ns, h, w) * 4 * HIDDEN and workspace.dtype == torch.float32
  _lib.call("mvb_convlstm_cell_fwd_onehot_fanout", _p(xh), _p(packed.w), _p(xf.B), _p(xf.T2), _p(ids), _p(c_in),
            _p(c_out), _p(h32_out), _p(workspace), ns, fanout, h, w, packed.cpad, packed.planes, float(forget_bias),
            _stream())


def nhwc_to_planes(src, xh, ch_off, h, w, comp=False):
  ns, c = src.shape[0], src.shape[-1]
  _lib.call("mvb_nhwc_to_planes", _p(src), _p(xh), xh.stride(0), xh.shape[2], ch_off, ns, h, w,
            c, planes_of(xh), int(comp), _stream())


def traj_to_planes(traj, t, centers, xh, h, w, comp=False):
  """nhwc_to_planes(float32(traj[:, t] - centers), xh, 0, h, w, comp) without the dense offsets: traj fp64 [N,T,2],
  centers fp64 [h,w,2], xh bf16x2 planes."""
  assert planes_of(xh) == PLANES_BF16X2 and 0 <= t < traj.shape[1]
  _, c = _traj_args(traj, centers, h, w)
  _lib.call("mvb_traj_to_planes", C.c_void_p(traj[:, t].data_ptr()), traj.stride(0), c, _p(xh), xh.stride(0),
            xh.shape[2], traj.shape[0], h, w, int(comp), _stream())


def nhwc_to_halo(src, dst, h, w):
  _lib.call("mvb_nhwc_to_halo", _p(src), _p(dst), src.shape[0], h, w, src.shape[-1], _stream())


def halo_to_nhwc(src, dst, h, w):
  _lib.call("mvb_halo_to_nhwc", _p(src), _p(dst), dst.shape[0], h, w, dst.shape[-1], _stream())


def enc_class_input(scene_conv, frame_idx, label, prev_label, xh, h, w):
  _lib.call("mvb_enc_class_input", _p(scene_conv), _p(frame_idx), _p(label), _p(prev_label),
            _p(xh), xh.stride(0), xh.shape[2], label.shape[0], h, w, planes_of(xh), _stream())


def enc_class_input_mix(scene_conv, frame_idx, label, label2, beta, xh, h, w):
  """scene_conv (.) (beta one_hot(label) + (1 - beta) one_hot(label2)) into the (zeroed) x block of xh."""
  _lib.call("mvb_enc_class_input_mix", _p(scene_conv), _p(frame_idx), _p(label), _p(label2), float(beta),
            _p(xh), xh.stride(0), xh.shape[2], label.shape[0], h, w, planes_of(xh), _stream())


def scene_conv_fwd(x, W, b):
  f, ih, iw, cin = x.shape
  cout = W.shape[3]
  out = torch.empty((f, (ih + 1) // 2, (iw + 1) // 2, cout), dtype=torch.float32, device=x.device)
  _lib.call("mvb_scene_conv_fwd", _p(x), _p(W), _p(b), _p(out), f, ih, iw, cin, cout, _stream())
  return out


def scene_time_mean(scene_conv, frame_idx):
  n, t = frame_idx.shape
  hwc = scene_conv[0].numel()
  out = torch.empty((n,) + tuple(scene_conv.shape[1:]), dtype=torch.float32,
                    device=scene_conv.device)
  _lib.call("mvb_scene_time_mean", _p(scene_conv), _p(frame_idx), _p(out), n, t, hwc, _stream())
  return out


def gnn_attend_fwd(h32, scene_mean, xh_next, h, w, ns, beam=1, row_map=None):
  _lib.call("mvb_gnn_attend_fwd", _p(h32), _p(row_map), _p(scene_mean), beam, _p(xh_next),
            xh_next.stride(0), xh_next.shape[2], xh_next.shape[2] - HIDDEN, ns, h, w,
            planes_of(xh_next), _stream())


def head_class_fwd(h32, Wo, logits_out, ids_out, We, be, xh_next, h, w, ns, planes=PLANES_BF16X2):
  e = 0 if We is None else We.shape[3]
  if xh_next is not None:
    stride, cpad, planes = xh_next.stride(0), xh_next.shape[2], planes_of(xh_next)
  else:
    stride, cpad = 0, 0
  _lib.call("mvb_head_class_fwd", _p(h32), _p(Wo), _p(logits_out), _p(ids_out), _p(We), _p(be), e,
            _p(xh_next), stride, cpad, ns, h, w, planes, _stream())


def head_class_fwd_dense(h32, Wo, logits_out, ids_out, We, be, xh_next, h, w, ns, planes=PLANES_BF16X2):
  """head_class_fwd whose feedback embeds the logits map itself (training without --train_w_onehot)."""
  e = 0 if We is None else We.shape[3]
  if xh_next is not None:
    stride, cpad, planes = xh_next.stride(0), xh_next.shape[2], planes_of(xh_next)
  else:
    stride, cpad = 0, 0
  _lib.call("mvb_head_class_fwd_dense", _p(h32), _p(Wo), _p(logits_out), _p(ids_out), _p(We), _p(be), e,
            _p(xh_next), stride, cpad, ns, h, w, planes, _stream())


def head_reg_fwd(h32, Wo, off_out, We, be, xh_next, h, w, ns, planes=PLANES_BF16X2):
  e = 0 if We is None else We.shape[3]
  if xh_next is not None:
    stride, cpad, planes = xh_next.stride(0), xh_next.shape[2], planes_of(xh_next)
  else:
    stride, cpad = 0, 0
  _lib.call("mvb_head_reg_fwd", _p(h32), _p(Wo), _p(off_out), _p(We), _p(be), e, _p(xh_next),
            stride, cpad, ns, h, w, planes, _stream())


def emb_onehot_fwd(ids, We, be, xh_next, h, w):
  _lib.call("mvb_emb_onehot_fwd", _p(ids), _p(We), _p(be), We.shape[3], _p(xh_next),
            xh_next.stride(0), xh_next.shape[2], ids.numel(), h, w, planes_of(xh_next), _stream())


def emb_dense_fwd(x, We, be, xh_next, h, w):
  _lib.call("mvb_emb_dense_fwd", _p(x), _p(We), _p(be), We.shape[3], _p(xh_next),
            xh_next.stride(0), xh_next.shape[2], x.shape[0], h, w, planes_of(xh_next), _stream())


def beam_step(logits, score_in, score_out, ids_out, parents_out, row_map_out, n, b, v,
              first_step, zero_scores, diverse, gamma):
  lg = math.log(gamma) if diverse else 0.0
  _lib.call("mvb_beam_step", _p(logits), _p(score_in), _p(score_out), _p(ids_out),
            _p(parents_out), _p(row_map_out), n, b, v, int(first_step), int(zero_scores),
            int(diverse), float(lg), _stream())


def beam_gather_h(h32, row_map, xh_next, h, w, ns):
  """h block of the f16f8 operand rows of xh_next <- the fp32 h32 rows of each row's parent row_map[s] (the beam
  decoder's state gather without graph attention)."""
  assert planes_of(xh_next) == PLANES_F16F8, "beam_gather_h writes the f16f8 operand format only"
  assert xh_next.shape[1] == halo_rows(ns, h, w) and row_map.dtype == torch.int32 and row_map.numel() == ns
  _lib.call("mvb_beam_gather_h_f16f8", _p(h32), _p(row_map), _p(xh_next), xh_next.stride(0), xh_next.shape[2], ns,
            h, w, _stream())


def beam_band_capacity(ns, h, w):
  """Work-list entries beam_band may write for ns beam rows."""
  return ns * (((h + 1) * (w + 1) + 127) // 128 + 1)


def beam_band(ids, parents, band_in, band_out, tiles, tile_count, k, radius, h, w):
  """Bands band_out int32 [ns, 2] (first, last image row where beam s may differ from its sample's base rollout) from
  the step's ids / parents int32 [N, K] and the parents' bands band_in (None at the fan-out), and the work list of
  the step's cell launch: tiles int32 [beam_band_capacity, 2] (m0, m_end) and tile_count int32 [1]."""
  ns = ids.numel()
  assert band_out.shape == (ns, 2) and band_out.dtype == torch.int32 and tiles.shape[1] == 2
  _lib.call("mvb_beam_band", _p(ids), _p(parents), _p(band_in), _p(band_out), _p(tiles), tiles.shape[0],
            _p(tile_count), ns, k, radius, h, w, _stream())


def beam_band_copy(base_c, base_h32, band, c, h32, k, h, w):
  """Valid rows of beam s outside band[s] <- the rows of sample s // k of the base rollout's state."""
  ns = band.shape[0]
  assert c.shape[0] == halo_rows(ns, h, w) and base_c.shape[0] * k == c.shape[0]
  _lib.call("mvb_beam_band_copy", _p(base_c), _p(base_h32), _p(band), _p(c), _p(h32), ns, k, h, w, _stream())


def beam_backtrace(step_ids, step_parents, step_logits, out_ids, out_logits):
  tp, n, b = step_ids.shape
  v = step_logits.shape[-1]
  _lib.call("mvb_beam_backtrace", _p(step_ids), _p(step_parents), _p(step_logits), _p(out_ids),
            _p(out_logits), n, b, tp, v, _stream())


def beam_backtrace_ragged(step_ids, step_parents, step_logits, lengths, out_ids, out_logits):
  """beam_backtrace of rows that end at their own lengths int32 [N] (1..Tp): row n's trace starts at step
  lengths[n] - 1, and its outputs at the steps after are zeros."""
  tp, n, b = step_ids.shape
  v = step_logits.shape[-1]
  assert lengths.dtype == torch.int32 and lengths.numel() == n
  _lib.call("mvb_beam_backtrace_ragged", _p(step_ids), _p(step_parents), _p(step_logits), _p(lengths), _p(out_ids),
            _p(out_logits), n, b, tp, v, _stream())


# --------------------------------------------------------------------------- training (BPTT) ops
def cell_fwd_train(xh, packed, c_in, c_out, h32_out, xh_next, gates_out, h, w, ns, forget_bias=1.0):
  """cell_fwd that also stores the activated gates [R,1024] for the backward pass."""
  hp = _hp_out(xh, packed, xh_next)
  _lib.call("mvb_convlstm_cell_fwd_train", _p(xh), _p(packed.w), _p(packed.bias), _p(c_in), _p(c_out), _p(h32_out),
            *hp, _p(gates_out), ns, h, w, packed.cpad, packed.planes, float(forget_bias), _stream())


def pack_dgrad(packed, kernel):
  """Operand planes of the dgrad GEMM for a PackedCell (cached on it)."""
  if getattr(packed, "wd", None) is None:
    packed.wd = torch.empty((packed.planes, packed.cpad, 9 * 4 * HIDDEN), dtype=torch.bfloat16,
                            device=kernel.device)
  _lib.call("mvb_pack_cell_weights_dgrad", _p(kernel.detach().float().contiguous()), _p(packed.wd),
            packed.cx, packed.planes, _stream())
  return packed.wd


def lstm_gates_bwd(gates, c_prev, c_new, dh, dc_in, dg_planes, dc_prev, dbias_packed, h, w, ns):
  _lib.call("mvb_lstm_gates_bwd", _p(gates), _p(c_prev), _p(c_new), _p(dh), _p(dc_in),
            _p(dg_planes), dg_planes.stride(0), _p(dc_prev), _p(dbias_packed), ns, h, w,
            dg_planes.shape[0], _stream())


def cell_dgrad(dg_planes, wd, dxh, h, w, ns, need_dx=True):
  _lib.call("mvb_cell_dgrad", _p(dg_planes), _p(wd), _p(dxh), ns, h, w, dxh.shape[1],
            dg_planes.shape[0], int(need_dx), _stream())


def cell_wgrad_direct(dg_planes, xh, dw_packed, h, w, ns):
  """wgrad straight from the row-major planes (MN-major wgmma operands, no transposes)."""
  _lib.call("mvb_cell_wgrad_direct", _p(dg_planes), _p(xh), _p(dw_packed), ns, h, w, xh.shape[2],
            xh.shape[0], _stream())


def wgrad_slabs(cpad):
  return int(_lib.load().mvb_cell_wgrad_slabs(cpad))


def unpack_cell_wgrad(dw_packed, dbias_packed, dkernel, dbiases, cx, comp=False, accumulate=False):
  slabs = dw_packed.shape[0] if dw_packed.dim() == 3 else 1
  _lib.call("mvb_unpack_cell_wgrad", _p(dw_packed), _p(dbias_packed), _p(dkernel), _p(dbiases), cx,
            int(comp), int(accumulate), slabs, _stream())


def loss_fwd_bwd(logits, labels, dlogits, cls_weight, reg, target, dreg, reg_weight, loss_out):
  """loss_out[0] += weighted mean CE, loss_out[1] += weighted mean Huber; gradients written."""
  rows, v = (logits.numel() // logits.shape[-1], logits.shape[-1]) if logits is not None else (0, 0)
  nreg = reg.numel() if reg is not None else 0
  _lib.call("mvb_loss_fwd_bwd", _p(logits), _p(labels), _p(dlogits), rows, v, float(cls_weight),
            _p(reg), _p(target), _p(dreg), nreg, float(reg_weight), _p(loss_out), _stream())


def soft_ce_fwd_bwd(logits, labels, dlogits, cls_weight, loss_out):
  """loss_out[0] += weighted mean soft-label CE of logits fp32 [..., V] against labels fp32 [..., V]; dlogits written."""
  v = logits.shape[-1]
  assert labels.dtype == torch.float32 and labels.numel() == logits.numel()
  _lib.call("mvb_soft_ce_fwd_bwd", _p(logits), _p(labels), _p(dlogits), logits.numel() // v, v, float(cls_weight),
            _p(loss_out), _stream())


def fg_count(labels, v, count):
  """count fp64 [1] += number of foreground cells of labels: fp32 maps [..., V] (> 0) or int32 cells [...]."""
  soft = labels.dtype == torch.float32
  rows = labels.numel() // v if soft else labels.numel()
  _lib.call("mvb_fg_count", _p(labels) if soft else None, None if soft else _p(labels), rows, v, _p(count),
            _stream())


def masked_huber_fwd_bwd(reg, target, dreg, labels, count, reg_weight, loss_out):
  """loss_out[1] += reg_weight * Huber over the foreground cells of `labels` (as fg_count) / (2 * count[0]);
  reg / target / dreg fp32 [..., V, 2]."""
  v = reg.shape[-2]
  soft = labels.dtype == torch.float32
  rows = reg.numel() // (2 * v)
  assert count.dtype == torch.float64 and (labels.numel() == rows * v if soft else labels.numel() == rows)
  _lib.call("mvb_masked_huber_fwd_bwd", _p(reg), _p(target), _p(dreg), _p(labels) if soft else None,
            None if soft else _p(labels), rows, v, _p(count), float(reg_weight), _p(loss_out), _stream())


def _traj_args(traj, centers, h, w):
  assert traj.dtype == torch.float64 and traj.shape[-1] == 2 and traj.is_contiguous()
  assert centers.dtype == torch.float64 and centers.numel() == 2 * h * w
  return _p(traj), _p(centers)


def huber_traj_fwd_bwd(reg, pred_traj, centers, dreg, reg_weight, loss_out):
  """The Huber half of loss_fwd_bwd against the targets float32(pred_traj[n,t] - centers[v]) (fp64 difference),
  computed in the kernel: reg / dreg fp32 [Tp,N,V,2], pred_traj fp64 [N,Tp,2], centers fp64 [h,w,2]."""
  tp, n, v = reg.shape[0], reg.shape[1], reg.shape[2]
  assert tuple(pred_traj.shape) == (n, tp, 2)
  traj, c = _traj_args(pred_traj, centers, 1, v)
  _lib.call("mvb_huber_traj_fwd_bwd", _p(reg), traj, c, _p(dreg), n, tp, v, float(reg_weight), _p(loss_out), _stream())


def soft_ce_label_fwd_bwd(logits, labels, soft_grid, h, w, dlogits, cls_weight, loss_out):
  """soft_ce_fwd_bwd against the --soft_grid label maps of the int32 label cells `labels` [...] (one per logits row),
  computed in the kernel."""
  assert labels.dtype == torch.int32 and labels.numel() * h * w == logits.numel()
  _lib.call("mvb_soft_ce_label_fwd_bwd", _p(logits), _p(labels), int(soft_grid), _p(dlogits), labels.numel(), h, w,
            float(cls_weight), _p(loss_out), _stream())


def fg_count_label(labels, soft_grid, h, w, count):
  """fg_count of the label maps of the int32 label cells `labels` under --soft_grid (0: the sparse labels)."""
  assert labels.dtype == torch.int32
  _lib.call("mvb_fg_count_label", _p(labels), int(soft_grid), labels.numel(), h, w, _p(count), _stream())


def masked_huber_traj_fwd_bwd(reg, pred_traj, centers, dreg, labels, soft_grid, h, w, count, reg_weight, loss_out):
  """masked_huber_fwd_bwd with the targets of huber_traj_fwd_bwd and the foreground of the label maps of
  fg_count_label; labels int32 [Tp,N]."""
  tp, n = reg.shape[0], reg.shape[1]
  assert tuple(pred_traj.shape) == (n, tp, 2) and reg.shape[2] == h * w and tuple(labels.shape) == (tp, n)
  assert count.dtype == torch.float64 and labels.dtype == torch.int32
  traj, c = _traj_args(pred_traj, centers, h, w)
  _lib.call("mvb_masked_huber_traj_fwd_bwd", _p(reg), traj, c, _p(dreg), _p(labels), int(soft_grid), n, tp, h, w,
            _p(count), float(reg_weight), _p(loss_out), _stream())


def head_bwd(h32, dout, Wo, dWo, dh, accumulate_dh, h, w, ns):
  _lib.call("mvb_head_bwd", _p(h32), _p(dout), _p(Wo), Wo.shape[3], _p(dWo), _p(dh),
            int(accumulate_dh), ns, h, w, _stream())


def emb_bwd(dxh, ids, in_map, We, be, dWe, dbe, d_in, accumulate_din, h, w, ns):
  _lib.call("mvb_emb_bwd", _p(dxh), dxh.shape[1], _p(ids), _p(in_map), _p(We), _p(be), We.shape[3],
            We.shape[2], _p(dWe), _p(dbe), _p(d_in), int(accumulate_din), ns, h, w, _stream())


def gnn_bwd(h32, scene_mean, gout, work, dh, accumulate_dh, dscene_mean, h, w, ns):
  _lib.call("mvb_gnn_attend_bwd", _p(h32), _p(scene_mean), _p(gout), _p(work), _p(dh),
            int(accumulate_dh), _p(dscene_mean), ns, h, w, _stream())


def scene_conv_bwd(x, W, out, dout, dW, db, din):
  f, ih, iw, cin = x.shape
  _lib.call("mvb_scene_conv_bwd", _p(x), _p(W), _p(out), _p(dout), _p(dW), _p(db), _p(din), f, ih, iw,
            cin, W.shape[3], _stream())


def enc_class_input_bwd(dxh, frame_idx, label, dscene, h, w):
  _lib.call("mvb_enc_class_input_bwd", _p(dxh), dxh.shape[1], _p(frame_idx), _p(label), _p(dscene),
            label.shape[0], h, w, _stream())


def enc_class_input_mix_bwd(dxh, frame_idx, label, label2, beta, dscene, h, w):
  _lib.call("mvb_enc_class_input_mix_bwd", _p(dxh), dxh.shape[1], _p(frame_idx), _p(label), _p(label2), float(beta),
            _p(dscene), label.shape[0], h, w, _stream())


def scene_time_mean_bwd(dmean, frame_idx, dscene):
  n, t = frame_idx.shape
  _lib.call("mvb_scene_time_mean_bwd", _p(dmean), _p(frame_idx), _p(dscene), n, t, dmean[0].numel(),
            _stream())


def clip_adadelta(w, grad, acc, acc_upd, lr, clip, wd, grad_scale=1.0, rho=0.95, eps=1e-8):
  _lib.call("mvb_clip_adadelta", _p(w), _p(grad), _p(acc), _p(acc_upd), w.numel(), float(lr),
            float(rho), float(eps), float(clip or 0.0), float(wd), float(grad_scale), _stream())


def clip_update(w, grad, s1, s2, kind, lr, p1, p2, eps, clip, wd, grad_scale=1.0):
  """Momentum (kind 1) / Adam (2) / RMSProp (3) update fused with wd, 1/G scaling and the element-wise clip."""
  _lib.call("mvb_clip_update", _p(w), _p(grad), _p(s1), _p(s2), w.numel(), int(kind), float(lr), float(p1), float(p2),
            float(eps), float(clip or 0.0), float(wd), float(grad_scale), _stream())


def decode_trajectories(ids, offs, centers, out):
  """ids int32 [N,K,Tp], offs fp32 [Tp,N,V,2], centers fp32 [V,2] -> out fp32 [N,K,Tp,2]."""
  n, k, tp = ids.shape
  _lib.call("mvb_decode_trajectories", _p(ids), _p(offs), _p(centers), _p(out), n, k, tp, offs.shape[2],
            _stream())


def gather_offsets(ids, offs, lengths):
  """ids int32 [N,K,Tp], offs fp32 [Tp,N,V,2], lengths int32 [N] -> fp32 [N,K,Tp,2]: the offsets of the selected
  cells for t < lengths[n], zeros after."""
  n, k, tp = ids.shape
  assert offs.shape[:2] == (tp, n) and lengths.dtype == torch.int32 and lengths.numel() == n
  out = torch.empty((n, k, tp, 2), dtype=torch.float32, device=ids.device)
  _lib.call("mvb_gather_offsets", _p(ids), _p(offs), _p(lengths), _p(out), n, k, tp, offs.shape[2], _stream())
  return out


def operand_rows(xh, ns, h, w):
  """The operand planes of the first ns sample rows of an alloc_xh buffer, as the kernels address them: a
  [2, halo_rows(ns), cpad] view of its leading bytes (the cell kernels find the second plane halo_rows(ns) rows after
  the first).  Halo cells and padding are zero in every such view: the plane boundary falls on a sample boundary."""
  r, cpad = halo_rows(ns, h, w), xh.shape[2]
  if r == xh.shape[1]:
    return xh
  v = xh.view(-1)[:2 * r * cpad].view(2, r, cpad)
  if planes_of(xh) == PLANES_F16F8:
    v.mvb_planes = PLANES_F16F8
  return v


def operand_shrink(xh, ns_from, ns_to, h, w):
  """Re-lays operand planes written for ns_from sample rows (operand_rows(xh, ns_from)) for their first ns_to rows:
  the second plane's first rows move to their place in operand_rows(xh, ns_to)."""
  if ns_to == ns_from:
    return
  cpad = xh.shape[2]
  r0, r1 = halo_rows(ns_from, h, w), halo_rows(ns_to, h, w)
  flat = xh.view(-1)
  flat[r1 * cpad:2 * r1 * cpad].copy_(flat[r0 * cpad:(r0 + r1) * cpad].clone())


def adv_step(x, adv, grad, out, eps, step):
  """out = clip(adv - step*sign(grad), clip(x-eps,-1,1), clip(x+eps,-1,1)) (SimAug/code/pred_models.py:96-124,142-143)."""
  _lib.call("mvb_adv_step", _p(x), _p(adv), _p(grad), _p(out), float(eps), float(step), x.numel(), _stream())


def mix(a, b, out, w):
  """out = a*w + b*(1-w) (SimAug mixup, SimAug/code/pred_models.py:149-166)."""
  _lib.call("mvb_mix", _p(a), _p(b), _p(out), float(w), a.numel(), _stream())


def ce_rows(logits, labels):
  """Per-row sparse softmax cross entropy [rows] of logits fp32 [..., V] and labels int32 [...] (no gradient)."""
  v = logits.shape[-1]
  rows = logits.numel() // v
  out = torch.empty(logits.shape[:-1], dtype=torch.float32, device=logits.device)
  _lib.call("mvb_ce_rows", _p(logits), _p(labels), _p(out), rows, v, _stream())
  return out


def min_ade_fde(pred, gt, gt_len):
  """pred fp32 [N,K,Tp,2], gt fp32 [N,G,Tg,2], gt_len int32 [N,G] -> (ade_err fp64 [N,G,Tg], ade_idx int32 [N,G],
  fde fp64 [N,G], fde_idx int32 [N,G]): code/multifuture_eval_trajs.py:41-78 on the device."""
  n, k, tp, _ = pred.shape
  g, tg = gt.shape[1], gt.shape[2]
  dev = pred.device
  ade_err = torch.empty((n, g, tg), dtype=torch.float64, device=dev)
  ade_idx = torch.empty((n, g), dtype=torch.int32, device=dev)
  fde = torch.empty((n, g), dtype=torch.float64, device=dev)
  fde_idx = torch.empty((n, g), dtype=torch.int32, device=dev)
  _lib.call("mvb_min_ade_fde", _p(pred), _p(gt), _p(gt_len), _p(ade_err), _p(ade_idx), _p(fde), _p(fde_idx), n, g, k,
            tp, tg, _stream())
  return ade_err, ade_idx, fde, fde_idx


def beam_nll(logits, logprobs, gt_idx, steps):
  """logits fp32 [N,K,Tp,V], logprobs fp32 [N,K], gt_idx int32 [N,J,G] (-1 = absent), steps int32 [J] ->
  (nll fp64 [N,J], count int32 [N,J]): code/multifuture_eval_trajs_prob.py:113-131,170-197 on the device."""
  n, k, tp, v = logits.shape
  j, g = gt_idx.shape[1], gt_idx.shape[2]
  nll = torch.empty((n, j), dtype=torch.float64, device=logits.device)
  cnt = torch.empty((n, j), dtype=torch.int32, device=logits.device)
  _lib.call("mvb_beam_nll", _p(logits), _p(logprobs), _p(gt_idx), _p(steps), _p(nll), _p(cnt), n, k, tp, v, j, g,
            _stream())
  return nll, cnt


def beam_nll_ragged(logits, logprobs, lengths, gt_idx, steps):
  """beam_nll of a ragged decode: logits fp32 [N,K,Tmax,V] and logprobs fp32 [N,K] as forward(pred_lengths=...) returns
  them, lengths int32 [N] (its out["_lengths"]); a step at or past a row's length is not evaluated (count 0)."""
  n, k, tp, v = logits.shape
  j, g = gt_idx.shape[1], gt_idx.shape[2]
  assert lengths.dtype == torch.int32 and lengths.numel() == n
  nll = torch.empty((n, j), dtype=torch.float64, device=logits.device)
  cnt = torch.empty((n, j), dtype=torch.int32, device=logits.device)
  _lib.call("mvb_beam_nll_ragged", _p(logits), _p(logprobs), _p(lengths), _p(gt_idx), _p(steps), _p(nll), _p(cnt), n,
            k, tp, v, j, g, _stream())
  return nll, cnt


def min_ade_fde_cells(ids, offs, centers, lengths, gt, gt_len, center_only=False):
  """ids int32 [N,K,Tp], offs fp32 [N,K,Tp,2] (gather_offsets), centers fp64 [V,2], lengths int32 [N], gt fp64
  [N,G,Tg,2], gt_len int32 [N,G] -> (ade_err fp64 [N,G,Tg], ade_idx, fde fp64 [N,G], fde_idx, err int32 [1]):
  min_ade_fde on the points centre + offset formed in fp64 (centre alone with center_only).  err bit 1: a future
  longer than its row's predictions; bit 2: a cell id outside the centres."""
  n, k, tp = ids.shape
  g, tg = gt.shape[1], gt.shape[2]
  assert offs.shape == (n, k, tp, 2) and centers.dtype == torch.float64 and gt.dtype == torch.float64
  assert lengths.dtype == torch.int32 and gt_len.dtype == torch.int32 and ids.dtype == torch.int32
  dev = ids.device
  ade_err = torch.empty((n, g, tg), dtype=torch.float64, device=dev)
  ade_idx = torch.empty((n, g), dtype=torch.int32, device=dev)
  fde = torch.empty((n, g), dtype=torch.float64, device=dev)
  fde_idx = torch.empty((n, g), dtype=torch.int32, device=dev)
  err = torch.zeros(1, dtype=torch.int32, device=dev)
  _lib.call("mvb_min_ade_fde_cells", _p(ids), _p(offs), _p(centers), int(bool(center_only)), _p(lengths), _p(gt),
            _p(gt_len), _p(ade_err), _p(ade_idx), _p(fde), _p(fde_idx), _p(err), n, g, k, tp, centers.shape[0], tg,
            _stream())
  return ade_err, ade_idx, fde, fde_idx, err


def points_to_cells(points, scene_h, scene_w, video_h, video_w):
  """points fp64 [..., 2] frame pixels -> (cells int32 [...], err int32 [1]): xys_to_indexes of
  code/multifuture_eval_trajs_prob.py:45-63 (err 1: an index numpy would refuse; that cell is -1)."""
  assert points.dtype == torch.float64 and points.shape[-1] == 2
  cells = torch.empty(points.shape[:-1], dtype=torch.int32, device=points.device)
  err = torch.zeros(1, dtype=torch.int32, device=points.device)
  if cells.numel():
    _lib.call("mvb_points_to_cells", _p(points), _p(cells), _p(err), cells.numel(), int(scene_h), int(scene_w),
              int(video_h), int(video_w), _stream())
  return cells, err


def traj_to_grid(traj, centers, h_gap, w_gap, labels, regress, h, w):
  """traj fp64 [...,2], centers fp64 [h*w,2] -> labels int32 [...], regress fp32 [...,h,w,2]."""
  _lib.call("mvb_traj_to_grid", _p(traj), _p(centers), float(h_gap), float(w_gap), _p(labels), _p(regress),
            traj.numel() // 2, h, w, _stream())
