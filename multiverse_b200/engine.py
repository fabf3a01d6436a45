# coding=utf-8
"""Rollout engine: the forward pass of Model.build_forward (code/pred_models.py:123-308) as a
sequence of libmultiverse_b200 kernel launches on one CUDA stream.

Host code only sequences launches and owns the (PyTorch-allocated) device buffers; every
arithmetic step is a kernel of the C-ABI library:

  scene CNN (:146-165)                      -> mvb_scene_conv_fwd x2, mvb_scene_time_mean
  class encoder (:210-215, dynamic_rnn)      -> T x [mvb_enc_class_input, mvb_convlstm_cell_fwd]
    without use_scene_enc (:218-229)         -> T x mvb_convlstm_cell_fwd_onehot (no scene CNN)
  regression encoder (:232-234)              -> T x [mvb_nhwc_to_planes, mvb_convlstm_cell_fwd]
  greedy class decoder (:311-471, raw_rnn)   -> Tp x [mvb_gnn_attend_fwd, mvb_convlstm_cell_fwd_onehot,
                                                     mvb_head_class_fwd (logits+argmax)]
  regression decoder (:298-305)              -> Tp x [mvb_convlstm_cell_fwd, mvb_head_reg_fwd]
  beam decoder (:474-806)                    -> Tp x [mvb_head_class_fwd, mvb_beam_step,
                                                     mvb_gnn_attend_fwd (mvb_beam_gather_h_f16f8
                                                     without use_gnn),
                                                     mvb_convlstm_cell_fwd_onehot] + mvb_beam_backtrace

The (c,h) gather by parent beam (:611-623) is never a copy of c: mvb_beam_step emits a row map that
the next GNN / cell launch reads its state through (without use_gnn, mvb_beam_gather_h_f16f8 reads h
through it into the cell's operands).
"""
from __future__ import annotations

import os

import torch

from . import ops

P_ = "person_pred/"
# the class encoder's input embedding without use_scene_enc (code/pred_models.py:221-225): created under the top scope
# with AUTO_REUSE, so one variable serves every scale
ENC_EMB = (P_ + "grid_emb/W", P_ + "grid_emb/b")


def _names(i):
  """TF variable names of scale i (SURVEY.md §8a; scopes at code/pred_models.py:140,160,193,200,
  215,234,240,247,327,456,446,469,930-950)."""
  return dict(
      enc_class=(P_ + "encoder_grid_class_%d/enc_grid_%d/kernel" % (i, i),
                 P_ + "encoder_grid_class_%d/enc_grid_%d/biases" % (i, i)),
      enc_reg=(P_ + "encoder_grid_reg_%d/enc_grid_regress_%d/kernel" % (i, i),
               P_ + "encoder_grid_reg_%d/enc_grid_regress_%d/biases" % (i, i)),
      dec_class=(P_ + "decoder_grid_class_%d/decoder_rnn/dec_grid_%d/kernel" % (i, i),
                 P_ + "decoder_grid_class_%d/decoder_rnn/dec_grid_%d/biases" % (i, i)),
      dec_reg=(P_ + "decoder_grid_reg_%d/decoder_rnn/dec_grid_reg_%d/kernel" % (i, i),
               P_ + "decoder_grid_reg_%d/decoder_rnn/dec_grid_reg_%d/biases" % (i, i)),
      emb_class=(P_ + "decoder_grid_class_%d/decoder_rnn/grid_emb/W" % i,
                 P_ + "decoder_grid_class_%d/decoder_rnn/grid_emb/b" % i),
      emb_reg=(P_ + "decoder_grid_reg_%d/decoder_rnn/grid_emb/W" % i,
               P_ + "decoder_grid_reg_%d/decoder_rnn/grid_emb/b" % i),
      head_class=P_ + "hidden2grid_decoder_grid_class_%d/out_dec_grid/W" % i,
      head_reg=P_ + "hidden2grid_decoder_grid_reg_%d/out_dec_grid/W" % i)


class ScaleWeights(object):
  """Packed / device-resident weights of one grid scale."""

  def __init__(self, weights, i, planes, fast_class=False, fast=False, scene_enc=True):
    nm = _names(i)
    f = lambda n: weights[n].detach().to(torch.float32).contiguous()
    fp = ops.PLANES_F16F8 if fast else planes
    self.enc_class = ops.PackedCell(f(nm["enc_class"][0]), f(nm["enc_class"][1]), fp)
    self.enc_reg = ops.PackedCell(f(nm["enc_reg"][0]), f(nm["enc_reg"][1]), planes, comp=True)
    # inference: regression encoder with the h block in f16f8 on the tensor cores and the raw 2-channel offsets
    # (+-1.9e3 pixels) added in fp32 in the epilogue (ops.cell_fwd_xdense) - 2 passes instead of 3 and no x chunk
    # inference: class encoder with its one-cell scene-feature input added from per-sample table rows in the epilogue
    # (ops.cell_fwd_xsparse) instead of a K chunk of the GEMM
    self.enc_class_xs = None
    if fast and scene_enc and weights[nm["enc_class"][0]].shape[2] == 64 + ops.HIDDEN:
      self.enc_class_xs = ops.XSparse(f(nm["enc_class"][0]))
    self.enc_reg_fast = self.enc_reg_xd = None
    if fast and weights[nm["enc_reg"][0]].shape[2] == 2 + ops.HIDDEN:
      self.enc_reg_fast = ops.PackedCell(f(nm["enc_reg"][0]), f(nm["enc_reg"][1]), ops.PLANES_F16F8)
      self.enc_reg_xd = ops.XDense(f(nm["enc_reg"][0]))
    # class decoder fed by the graph attention: f16f8 operands (2 instead of 3 bf16-pass equivalents per product)
    self.dec_class = ops.PackedCell(f(nm["dec_class"][0]), f(nm["dec_class"][1]),
                                    ops.PLANES_F16F8 if fast_class else planes)
    self.dec_reg = ops.PackedCell(f(nm["dec_reg"][0]), f(nm["dec_reg"][1]), fp)
    self.emb_class = (f(nm["emb_class"][0]), f(nm["emb_class"][1]))
    self.emb_reg = (f(nm["emb_reg"][0]), f(nm["emb_reg"][1]))
    self.head_class = f(nm["head_class"])
    self.head_reg = f(nm["head_reg"])
    # inference: the class decoder's embedded one-hot input folded into table look-ups
    self.dec_class_xf = ops.XFold(f(nm["dec_class"][0]), f(nm["dec_class"][1]), *self.emb_class)
    # without scene encoding the class encoder's input, grid_emb(one_hot(label)), has the decoder's form: folded the
    # same way at inference (enc_class_fold); training embeds it (emb_onehot_fwd)
    self.enc_emb = self._enc_class_xf = None
    if not scene_enc:
      self.enc_emb = (f(ENC_EMB[0]), f(ENC_EMB[1]))
      self._enc_cell = (f(nm["enc_class"][0]), f(nm["enc_class"][1]))

  def enc_class_fold(self):
    """XFold of the class encoder's embedded one-hot input (models without scene encoding), built on first use: the
    training step, which repacks the weights after every update, never reads it."""
    if self._enc_class_xf is None:
      self._enc_class_xf = ops.XFold(*self._enc_cell, *self.enc_emb)
    return self._enc_class_xf


def beam_band_on():
  """MVB_BEAM_BAND=0 runs every row of the beam cell launches (decode_class_beam); read at every forward."""
  return os.environ.get("MVB_BEAM_BAND", "1") != "0"


class ConvRNNEngine(object):
  """Inference engine for one config (batch size, grids, flags) and one weight set."""
  GRAPH_CACHE = 4             # captured forward graphs kept per engine
  ALLOW_F16F8 = True          # TrainEngine: False (its packed weights also feed the bf16 backward GEMMs)

  def __init__(self, cfg, weights, device=None, planes=ops.PLANES_BF16X2):
    assert planes == ops.PLANES_BF16X2, \
        "planes=%r: the engines run the bf16x2 operand format (planes=2), with f16f8 where inference allows" % (planes,)
    self.cfg = cfg
    self.device = device or torch.device("cuda", torch.cuda.current_device())
    self.planes = planes
    # The class decoder's cell reads only what the graph attention writes (its one-hot input is folded into table
    # look-ups), so that producer/consumer pair switches to the f16f8 operand format as a unit.  Without the attention,
    # the beam decoder's parent gather (ops.beam_gather_h) is that producer.
    self.fast_class = self.ALLOW_F16F8 and bool(cfg.use_gnn or cfg.use_beam_search)
    self.class_planes = ops.PLANES_F16F8 if self.fast_class else self.planes
    # class encoder and regression decoder (inputs in (-1,1): tanh outputs) use the same format; the regression
    # ENCODER keeps bf16 planes: its raw pixel offsets (+-1.9e3) need the compensated x block.
    self.fast = self.ALLOW_F16F8
    self.fast_planes = ops.PLANES_F16F8 if self.fast else self.planes
    assert cfg.enc_hidden_size == ops.HIDDEN and cfg.dec_hidden_size == ops.HIDDEN, \
        "the kernels are specialised for hidden size 256 (every published config)"
    assert cfg.convlstm_kernel == 3 and cfg.scene_conv_kernel == 3
    assert cfg.scene_conv_dim == 64
    assert getattr(cfg, "activation_func", "tanh") in ("tanh",) or \
        getattr(cfg.activation_func, "__name__", "") == "tanh", "kernels implement tanh"
    self.set_weights(weights)
    self._bufs = {}
    self.cell_events = None   # set to [] to record (tag, (h, w, ns), start, end) events per cell launch
    self._graphs = {}         # forward_graph(): feed signature -> (CUDAGraph, static feeds, static outputs)
    self._graph_seen = set()  # signatures seen once (captured at their second occurrence)

  @property
  def gnn_scene_in_greedy(self):
    """False = SimAug's model variant: its gnn_edge (SimAug/code/pred_models.py:1213-1226) concatenates the scene
    features to the node features only under `if tile_to_beam:`, so the greedy class decoder (training, test.py)
    attends over h alone; the Multiverse file (code/pred_models.py:824-838) always uses them (default)."""
    return bool(self.scene_enc and getattr(self.cfg, "gnn_scene_in_greedy", True))

  @property
  def scene_enc(self):
    """use_scene_enc (code/pred_models.py:146, :184-229, :824): the scene CNN feeds the class encoder and the graph
    attention; without it the class encoder reads grid_emb(one_hot(label))."""
    return bool(getattr(self.cfg, "use_scene_enc", True))

  # ------------------------------------------------------------------ weights
  def set_weights(self, weights):
    dev = self.device
    if getattr(self, "_graphs", None) is not None:
      self._graphs.clear()      # captured graphs point at the previous weight buffers
      self._graph_seen.clear()
    w = {k: (v if torch.is_tensor(v) else torch.as_tensor(v)).to(dev) for k, v in weights.items()}
    scene_enc = self.scene_enc
    self.scene_w = [(w[P_ + "scene_conv%d/W" % (i + 1)].float().contiguous(),
                     w[P_ + "scene_conv%d/b" % (i + 1)].float().contiguous())
                    for i in range(len(self.cfg.scene_grid_strides))] if scene_enc else []
    self.scales = [ScaleWeights(w, i, self.planes, self.fast_class, self.fast, scene_enc) if self.cfg.use_grids[i]
                   else None for i in range(len(self.cfg.scene_grids))]

  # ------------------------------------------------------------------ buffers
  def _buf(self, key, maker):
    b = self._bufs.get(key)
    if b is None:
      b = maker()
      self._bufs[key] = b
    return b

  def _xh(self, tag, ns, h, w, cpad, planes=None):
    planes = planes or self.planes
    return [self._buf((tag, j, ns, h, w, cpad, planes),
                      lambda: ops.alloc_xh(ns, h, w, cpad, planes, self.device))
            for j in range(2)]

  def _state(self, tag, ns, h, w):
    return self._buf((tag, ns, h, w), lambda: ops.alloc_state(ns, h, w, self.device))

  def _cell(self, tag, shape, launch, *args, **kw):
    """launch(*args, **kw): one cell launch of shape (h, w, ns).  With cell_events a list, it is bracketed by CUDA
    events on the launching stream and (tag, shape, start, end) is appended (bench.py's live roofline measurement of
    the dominant kernel)."""
    if self.cell_events is None:
      return launch(*args, **kw)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    launch(*args, **kw)
    e1.record()
    self.cell_events.append((tag, shape, e0, e1))

  # ------------------------------------------------------------------ pieces
  def scene_cnn(self, scene_feat, obs_scene):
    """code/pred_models.py:146-165 on the unique frames; returns per-scale [F,h,w,64] maps and
    the per-sample time means used by the graph attention (:826-828).  Without use_scene_enc nothing reads the scene
    (:146, :824): None per scale."""
    if not self.scene_enc:
      return [None] * len(self.cfg.scene_grids), [None] * len(self.cfg.scene_grids)
    x = scene_feat
    convs, means = [], []
    for (W, b) in self.scene_w:
      x = ops.scene_conv_fwd(x, W, b)
      convs.append(x)
      means.append(ops.scene_time_mean(x, obs_scene))
    return convs, means

  def encode_class(self, i, scene_conv, obs_scene_t, labels_t, xh_out):
    """Class encoder (:210-215; without use_scene_enc :218-229, scene_conv None).  obs_scene_t / labels_t: int32
    [T,N].  Writes the planes of the last h into the h block of xh_out (if given) and returns (c, h32) halo
    buffers."""
    h, w = self.cfg.scene_grids[i]
    n = labels_t.shape[1]
    t_len = labels_t.shape[0]
    sw = self.scales[i]
    xh = self._xh("enc_class", n, h, w, sw.enc_class.cpad, self.fast_planes)
    c = [self._state("enc_c0", n, h, w), self._state("enc_c1", n, h, w)]
    h32 = self._state("enc_h32", n, h, w)
    if sw.enc_emb is not None:
      # the embedded one_hot(label_t) input is folded into table look-ups: nobody writes the x blocks
      xf = sw.enc_class_fold()
      xh[0][:, :, sw.enc_class.cxp:].zero_()   # h_0 = 0
      for t in range(t_len):
        cur, nxt = xh[t % 2], xh[(t + 1) % 2]
        last = t == t_len - 1
        self._cell("enc_class", (h, w, n), ops.cell_fwd_onehot, cur, sw.enc_class, xf, labels_t[t],
                   None if t == 0 else c[t % 2], c[(t + 1) % 2], h32 if last else None, xh_out if last else nxt,
                   h, w, n)
      return c[t_len % 2], h32
    if sw.enc_class_xs is not None:
      # (one table per scale: the chains of different scales run concurrently under forward_graph)
      table = self._buf(("enc_class_xtab", n, h, w), lambda: torch.empty((n, 9, 4 * ops.HIDDEN), dtype=torch.float32,
                                                                  device=self.device))
      xh[0][:, :, sw.enc_class.cxp:].zero_()   # h_0 = 0 (the x blocks are neither written nor read)
      for t in range(t_len):
        cur, nxt = xh[t % 2], xh[(t + 1) % 2]
        last = t == t_len - 1
        ops.cell_xsparse_table(scene_conv, obs_scene_t[t], labels_t[t], sw.enc_class_xs, table, h, w)
        self._cell("enc_class", (h, w, n), ops.cell_fwd_xsparse, cur, sw.enc_class, table, labels_t[t],
                   None if t == 0 else c[t % 2], c[(t + 1) % 2], h32 if last else None, xh_out if last else nxt,
                   h, w, n)
      return c[t_len % 2], h32
    # a previous call left the label pixels of its last two steps in the x blocks: clear them
    for j in range(2):
      xh[j][:, :, :sw.enc_class.cxp].zero_()
    xh[0][:, :, sw.enc_class.cxp:].zero_()   # h_0 = 0
    for t in range(t_len):
      cur, nxt = xh[t % 2], xh[(t + 1) % 2]
      ops.enc_class_input(scene_conv, obs_scene_t[t], labels_t[t],
                          labels_t[t - 2] if t >= 2 else None, cur, h, w)
      last = t == t_len - 1
      self._cell("enc_class", (h, w, n), ops.cell_fwd, cur, sw.enc_class, None if t == 0 else c[t % 2],
                 c[(t + 1) % 2], h32 if last else None, xh_out if last else nxt, h, w, n)
    return c[t_len % 2], h32

  def encode_reg(self, i, obs_reg_t, xh_out):
    """Regression encoder (:232-234).  obs_reg_t fp32 [T,N,h,w,2]."""
    h, w = self.cfg.scene_grids[i]
    t_len, n = obs_reg_t.shape[0], obs_reg_t.shape[1]
    sw = self.scales[i]
    if sw.enc_reg_fast is not None:
      pk = sw.enc_reg_fast
      xh = self._xh("enc_reg_f", n, h, w, pk.cpad, ops.PLANES_F16F8)
      c = [self._state("encr_c0", n, h, w), self._state("encr_c1", n, h, w)]
      h32 = self._state("encr_h32", n, h, w)
      xh[0][:, :, pk.cxp:].zero_()            # h_0 = 0 (the x blocks are never written nor read)
      for t in range(t_len):
        cur, nxt = xh[t % 2], xh[(t + 1) % 2]
        last = t == t_len - 1
        self._cell("enc_reg", (h, w, n), ops.cell_fwd_xdense, cur, pk, sw.enc_reg_xd, obs_reg_t[t],
                   None if t == 0 else c[t % 2], c[(t + 1) % 2], h32 if last else None, xh_out if last else nxt,
                   h, w, n)
      return c[t_len % 2], h32
    xh = self._xh("enc_reg", n, h, w, sw.enc_reg.cpad)
    c = [self._state("encr_c0", n, h, w), self._state("encr_c1", n, h, w)]
    h32 = self._state("encr_h32", n, h, w)
    xh[0][:, :, sw.enc_reg.cxp:].zero_()
    for t in range(t_len):
      cur, nxt = xh[t % 2], xh[(t + 1) % 2]
      ops.nhwc_to_planes(obs_reg_t[t], cur, 0, h, w, comp=sw.enc_reg.comp)
      last = t == t_len - 1
      self._cell("enc_reg", (h, w, n), ops.cell_fwd, cur, sw.enc_reg, None if t == 0 else c[t % 2],
                 c[(t + 1) % 2], h32 if last else None, xh_out if last else nxt, h, w, n)
    return c[t_len % 2], h32

  def decode_class_greedy(self, i, c_enc, h32_enc, first_ids, scene_mean, pred_len, act=None):
    """Greedy class decoder (:311-471, appendix A.1).  Returns logits [Tp,N,HW], ids [Tp,N].
    act: ragged rollout (forward(pred_lengths=...)): step t runs the first act[t] rows only, the rest stay zero."""
    cfg = self.cfg
    h, w = cfg.scene_grids[i]
    n = first_ids.shape[0]
    sw = self.scales[i]
    xh = self._xh("dec_class", n, h, w, sw.dec_class.cpad, self.class_planes)
    c = [self._state("dec_c0", n, h, w), self._state("dec_c1", n, h, w)]
    h32 = self._state("dec_h32", n, h, w)
    alloc = torch.empty if act is None else torch.zeros
    logits = alloc((pred_len, n, h * w), dtype=torch.float32, device=self.device)
    ids = alloc((pred_len, n), dtype=torch.int32, device=self.device)
    h_src, c_src, ids_prev, m = h32_enc, c_enc, first_ids, n
    for t in range(pred_len):
      cur, nxt = xh[t % 2], xh[(t + 1) % 2]
      if act is not None:     # operand planes as the kernels address them for the running rows (ops.operand_rows)
        if not cfg.use_gnn:   # cur holds the previous step's h for its m rows
          ops.operand_shrink(cur, m, act[t], h, w)
        m = act[t]
        cur, nxt = ops.operand_rows(cur, m, h, w), ops.operand_rows(nxt, m, h, w)
      if cfg.use_gnn:
        ops.gnn_attend_fwd(h_src, scene_mean if self.gnn_scene_in_greedy else None, cur, h, w, m)
      # (no attention: the planes of the previous h already sit in cur's h block)
      # the embedded one_hot(ids_prev) input is folded into table look-ups: nobody writes the x block
      self._cell("dec_class", (h, w, m), ops.cell_fwd_onehot, cur, sw.dec_class, sw.dec_class_xf, ids_prev, c_src,
                 c[(t + 1) % 2], h32, None if cfg.use_gnn else nxt, h, w, m)
      c_src, h_src = c[(t + 1) % 2], h32
      ops.head_class_fwd(h32, sw.head_class, logits[t], ids[t], None, None, None, h, w, m,
                         planes=self.planes)
      ids_prev = ids[t]
    return logits, ids

  def decode_reg(self, i, c_enc, first_input, pred_len, xh, act=None):
    """Regression decoder (:298-305): greedy, no attention, raw 2-channel feedback.  `xh` are
    the decoder operand buffers whose xh[0] h block already holds the encoder state planes.  act: as
    decode_class_greedy."""
    h, w = self.cfg.scene_grids[i]
    n = first_input.shape[0]
    sw = self.scales[i]
    c = [self._state("decr_c0", n, h, w), self._state("decr_c1", n, h, w)]
    h32 = self._state("decr_h32", n, h, w)
    offs = (torch.empty if act is None else torch.zeros)((pred_len, n, h * w, 2), dtype=torch.float32,
                                                          device=self.device)
    We, be = sw.emb_reg
    ops.emb_dense_fwd(first_input, We, be, xh[0], h, w)
    c_src, m = c_enc, n
    for t in range(pred_len):
      cur, nxt = xh[t % 2], xh[(t + 1) % 2]
      if act is not None:     # cur holds the previous step's h and fed-back offsets for its m rows
        ops.operand_shrink(cur, m, act[t], h, w)
        m = act[t]
        cur, nxt = ops.operand_rows(cur, m, h, w), ops.operand_rows(nxt, m, h, w)
      self._cell("dec_reg", (h, w, m), ops.cell_fwd, cur, sw.dec_reg, c_src, c[(t + 1) % 2], h32, nxt, h, w, m)
      c_src = c[(t + 1) % 2]
      last = t == pred_len - 1
      ops.head_reg_fwd(h32, sw.head_reg, offs[t], None if last else We, None if last else be,
                       None if last else nxt, h, w, m, planes=self.planes)
    return offs

  def decode_class_beam(self, i, c_enc, h32_enc, first_ids, scene_mean, pred_len, act=None, lengths=None):
    """K-way beam decoder (:474-806, appendix A.2).  Returns (out_logits [N,B,Tp,V],
    out_ids [N,B,Tp] int32, scores [N,B]).
    Ragged rollout (forward(pred_lengths=...)): rows sorted by length, longest first; lengths int32 [N] on the device
    and act[t] = number of rows longer than t.  The selection at time t runs the rows whose length is at least t,
    the cell of time t (which feeds the selection at t + 1) only those longer than t: every launch takes a prefix of
    the rows, and a row's outputs are those of a rollout of its own length.  Its scores are those after its own last
    selection, its outputs after its length zeros."""
    cfg = self.cfg
    h, w = cfg.scene_grids[i]
    n, b, v = first_ids.shape[0], cfg.beam_size, h * w
    ns = n * b
    dev = self.device
    sw = self.scales[i]
    xh = self._xh("beam", ns, h, w, sw.dec_class.cpad, self.class_planes)
    c = [self._state("beam_c0", ns, h, w), self._state("beam_c1", ns, h, w)]
    h32 = self._state("beam_h32", ns, h, w)
    step_logits = torch.empty((pred_len, n, b, v), dtype=torch.float32, device=dev)
    step_ids = torch.empty((pred_len, n, b), dtype=torch.int32, device=dev)
    step_par = torch.empty((pred_len, n, b), dtype=torch.int32, device=dev)
    scores = [torch.zeros((n, b), dtype=torch.float32, device=dev) for _ in range(2)]
    row_map = torch.empty((ns,), dtype=torch.int32, device=dev)
    xf = sw.dec_class_xf
    # time = 0 (:497-502, :527-531): the reference tiles the encoder state and the last observed cell K times, so
    # all K beams carry identical rows until the first selection (which looks at beam 0 only, :569-573).  That
    # step - graph attention, cell, and the time-1 head - is therefore evaluated once per sample (N rows, not
    # N*K) and the first selection's children read it through row_map = sample index: same values, 1/K of
    # the work for 1 of the Tp steps.  The embedded one-hot input of every step is folded into table
    # look-ups (ops.cell_fwd_onehot).
    # Without the graph attention (use_gnn off) the state goes straight into the cell: the encoder has written its
    # last h into xh1[0] (forward()), the time-0 cell writes its h into xh1[1] for the fan-out, and from time 2 on
    # ops.beam_gather_h copies the parents' h rows into the children's operand rows.
    assert cfg.use_gnn or self.class_planes == ops.PLANES_F16F8, \
        "beam search without use_gnn runs on f16f8 operands (inference engine)"
    xh1 = self._xh("beam_t0", n, h, w, sw.dec_class.cpad, self.class_planes)
    c_t0 = self._state("beam_c_t0", n, h, w)
    h32_t0 = self._state("beam_h32_t0", n, h, w)
    logits_t0 = torch.empty((n, v), dtype=torch.float32, device=dev)
    if cfg.use_gnn:
      ops.gnn_attend_fwd(h32_enc, scene_mean, xh1[0], h, w, n, beam=1, row_map=None)
    self._cell("beam_t0", (h, w, n), ops.cell_fwd_onehot, xh1[0], sw.dec_class, xf, first_ids.contiguous(), c_enc,
               c_t0, h32_t0, None if cfg.use_gnn else xh1[1], h, w, n)
    ops.head_class_fwd(h32_t0, sw.head_class, logits_t0, None, None, None, None, h, w, n, planes=self.planes)
    step_logits[0].copy_(logits_t0.unsqueeze(1).expand(n, b, v))
    # Image-row bands (ops.beam_band, DESIGN.md 3.2): outside rows band[k], beam k's c and h are bit for bit those of
    # its sample's base rollout - the same recurrence, through the same kernels, fed the no-selection input (ids
    # outside the grid) - so the beam cell computes only the bands' rows and the rest is copied from the base.
    # MVB_BEAM_BAND=0 runs every row.
    band = pred_len > 2 and beam_band_on()
    # samples in the selection (sel) and in the cell step (ncell) of each time, and the operand planes of ns rows as
    # the kernels address them (ops.operand_rows)
    sel = (lambda time: n) if act is None else (lambda time: act[time - 1])
    ncell = (lambda time: n) if act is None else (lambda time: act[time])
    rows_of = (lambda t, ns_: t) if act is None else (lambda t, ns_: ops.operand_rows(t, ns_, h, w))
    if band:
      bands = [self._buf(("beam_band", j, ns), lambda: torch.empty((ns, 2), dtype=torch.int32, device=dev))
               for j in range(2)]
      tiles = self._buf(("beam_band_tiles", ns, h, w), lambda: torch.empty(
          (ops.beam_band_capacity(ns, h, w), 2), dtype=torch.int32, device=dev))
      tile_count = torch.empty((pred_len,), dtype=torch.int32, device=dev)
      base_xh = self._xh("beam_base", n, h, w, sw.dec_class.cpad, self.class_planes)[0]
      base_c = [self._state("beam_base_c0", n, h, w), self._state("beam_base_c1", n, h, w)]
      base_h32 = self._state("beam_base_h32", n, h, w)
      no_ids = self._buf(("beam_base_ids", n, h, w), lambda: torch.full((n,), (h + 3) * w, dtype=torch.int32,
                                                                        device=dev))
      rows = self._buf(("beam_base_rows", n), lambda: torch.arange(n, dtype=torch.int32, device=dev))
      radius = 2 if cfg.use_gnn else 1      # the graph attention spreads a difference by one more row per step
    h_src, c_src, cur_c = h32_t0, c_t0, 1
    for time in range(1, pred_len + 1):
      ms = sel(time)
      if time > 1:
        ops.head_class_fwd(h32, sw.head_class, step_logits[time - 1], None, None, None, None, h, w,
                           ms * b, planes=self.planes)
      s_in, s_out = scores[(time - 1) % 2], scores[time % 2]
      ops.beam_step(step_logits[time - 1], s_in, s_out, step_ids[time - 1], step_par[time - 1],
                    row_map, ms, b, v, first_step=(time <= 1),
                    zero_scores=(time <= cfg.fix_num_timestep), diverse=cfg.diverse_beam,
                    gamma=cfg.diverse_gamma)
      if time == pred_len:
        break
      m = ncell(time)
      if band:
        ops.beam_band(step_ids[time - 1][:m], step_par[time - 1][:m], None if time == 1 else bands[time % 2],
                      bands[1 - time % 2][:m * b], tiles, tile_count[time:time + 1], b, radius, h, w)
      nxt = rows_of(xh[time % 2], m * b)
      if time == 1:
        # every child's parent is its sample's single t0 row: the K children share the graph-attended h and c and
        # differ only in the selected cell, i.e. in the folded table rows -> attention and GEMM once per sample,
        # the cell epilogue fans the K children out (ops.cell_fwd_onehot_fanout; 1/K of the step's MMAs)
        if not cfg.use_gnn and act is not None:     # the time-0 cell wrote h for all rows
          ops.operand_shrink(xh1[1], n, m, h, w)
        x_t1 = rows_of(xh1[1], m)
        if cfg.use_gnn:
          ops.gnn_attend_fwd(h32_t0, scene_mean, x_t1, h, w, m, beam=1, row_map=None)
        ws = self._buf(("beam_fanout_ws", n, h, w), lambda: torch.empty(
            (ops.halo_rows(n, h, w), 4 * ops.HIDDEN), dtype=torch.float32, device=dev))
        self._cell("beam_fanout", (h, w, m), ops.cell_fwd_onehot_fanout, x_t1, sw.dec_class, xf,
                   step_ids[0].view(-1), c_t0, c[1 - cur_c], h32, h, w, m, b, workspace=ws)
        if band:      # the base's first step: the same accumulators, no selection
          ops.cell_fwd_onehot_fanout(None, sw.dec_class, xf, no_ids, c_t0, base_c[1], base_h32, h, w, m, 1,
                                     workspace=ws)
      else:
        if band:
          x_base = rows_of(base_xh, m)
          if cfg.use_gnn:
            ops.gnn_attend_fwd(base_h32, scene_mean, x_base, h, w, m, beam=1, row_map=None)
          else:
            ops.beam_gather_h(base_h32, rows[:m], x_base, h, w, m)
          self._cell("beam_base", (h, w, m), ops.cell_fwd_onehot, x_base, sw.dec_class, xf, no_ids,
                     base_c[(time - 1) % 2], base_c[time % 2], base_h32, None, h, w, m)
        if cfg.use_gnn:
          ops.gnn_attend_fwd(h_src, scene_mean, nxt, h, w, m * b, beam=b, row_map=row_map)
        else:
          ops.beam_gather_h(h_src, row_map[:m * b], nxt, h, w, m * b)
        self._cell("beam", (h, w, m * b), ops.cell_fwd_onehot, nxt, sw.dec_class, xf, step_ids[time - 1].view(-1),
                   c_src, c[1 - cur_c], h32, None, h, w, m * b, row_map=row_map,
                   tiles=(tiles, tile_count[time:time + 1]) if band else None)
        if band:
          hr, hr_base = ops.halo_rows(m * b, h, w), ops.halo_rows(m, h, w)
          ops.beam_band_copy(base_c[time % 2][:hr_base], base_h32[:hr_base], bands[1 - time % 2][:m * b],
                             c[1 - cur_c][:hr], h32[:hr], b, h, w)
      cur_c = 1 - cur_c
      h_src, c_src = h32, c[cur_c]
    out_ids = torch.empty((n, b, pred_len), dtype=torch.int32, device=dev)
    out_logits = torch.empty((n, b, pred_len, v), dtype=torch.float32, device=dev)
    if act is None:
      ops.beam_backtrace(step_ids, step_par, step_logits, out_ids, out_logits)
      final = scores[pred_len % 2]
    else:
      ops.beam_backtrace_ragged(step_ids, step_par, step_logits, lengths, out_ids, out_logits)
      # row j's last selection (time lengths[j]) wrote scores[lengths[j] % 2]; later selections skip it
      final = torch.where((lengths % 2 == 0).unsqueeze(1), scores[0], scores[1])
    return out_logits, out_ids, final, dict(ids=step_ids, parents=step_par, logits=step_logits)

  # ------------------------------------------------------------------ whole forward
  def branches(self):
    """The independent chains of one forward: ("class", i) and ("reg", i) per used scale (they share only the feeds;
    the scene CNN belongs to the class chains)."""
    return [(kind, i) for i in range(len(self.cfg.scene_grids)) if self.cfg.use_grids[i] for kind in ("class", "reg")]

  def forward(self, feeds, pred_len=None, on_output=None, branches=None, pred_lengths=None):
    """feeds: device tensors
         scene_feat fp32 [F,SH,SW,SC], obs_scene int32 [N,T],
         grid_obs_labels[i] int32 [N,T], grid_obs_regress[i] fp32 [N,T,h,w,2]
    Returns a dict shaped like the reference fetches: grid_pred_decoded[i] [N,Tp,h,w,1],
    grid_pred_reg_decoded[i] [N,Tp,h,w,2] ([] for unused scales, :170-171) and
    beam_outputs = [logits [N,B,Tp,V], ids [N,B,Tp], logprobs [N,B]] or None (:276).
    on_output(name, index, tensor) is called as soon as a fetched tensor is complete on the current stream, so a
    caller can start its device->host copy on another stream while the remaining branches still run.
    `branches`: subset of self.branches() to run (forward_graph captures one graph per chain); the outputs of the
    others are None.
    `pred_lengths`: int [N], every L_i >= 1 (host array or tensor), decodes each row to its own length: the rollout
    runs T = max L_i steps (pred_len is ignored), and row i's outputs at t < L_i are byte for byte those of a forward
    of row i alone with pred_len = L_i, zeros at t >= L_i; beam_outputs[2][i] holds the scores after row i's own last
    selection.  The rows are sorted by length, longest first, and every step launches only the rows still running
    (the rollout of code/multifuture_inference.py, which decodes every trajectory alone to its own length, :311).
    With all lengths equal this is forward(pred_len=T).  out["_lengths"]: the lengths, int32 on the device."""
    cfg = self.cfg
    emit = on_output if on_output is not None else (lambda *a: None)
    run = set(self.branches() if branches is None else branches)
    # raw_rnn runs until `time >= pred_length` (code/pred_models.py:347,:520): the rollout length is the
    # FED pred_length (multifuture_inference.py feeds max_pred_lengths[idx], :311), not config.pred_len
    tp = int(pred_len) if pred_len else cfg.pred_len
    obs_scene = feeds["obs_scene"].to(torch.int32).contiguous()
    n = obs_scene.shape[0]
    act = lengths = perm = inv = None
    if pred_lengths is not None:
      import numpy as np
      lens = np.asarray(pred_lengths.cpu() if torch.is_tensor(pred_lengths) else pred_lengths).astype(np.int64)
      lens = lens.reshape(-1)
      if lens.size != n or lens.min() < 1:
        raise ValueError("pred_lengths: one length >= 1 per row (%d rows), got %s" % (n, lens))
      tp = int(lens.max())
      if (lens != tp).any():
        order = np.argsort(-lens, kind="stable")
        act = [int((lens > t).sum()) for t in range(tp)]
        perm = torch.from_numpy(order).to(self.device)
        inv = torch.from_numpy(np.argsort(order)).to(self.device)
        lengths = torch.from_numpy(lens[order].astype(np.int32)).to(self.device)
        obs_scene = obs_scene.index_select(0, perm)
    # rows back in the caller's order (ragged: they run sorted by length)
    unsort = (lambda t, dim=0: t) if inv is None else (lambda t, dim=0: t.index_select(dim, inv))
    sort = (lambda t: t) if perm is None else (lambda t: t.index_select(0, perm))
    obs_scene_t = obs_scene.t().contiguous()
    convs = means = None
    if any(kind == "class" for kind, _ in run):
      convs, means = self.scene_cnn(feeds["scene_feat"].float().contiguous(), obs_scene)
    out = dict(grid_pred_decoded=[], grid_pred_reg_decoded=[], beam_outputs=None)
    for i, (h, w) in enumerate(cfg.scene_grids):
      if not cfg.use_grids[i]:
        out["grid_pred_decoded"].append([])
        out["grid_pred_reg_decoded"].append([])
        continue
      sw = self.scales[i]
      dec = reg = None
      if ("class", i) in run:
        labels = sort(feeds["grid_obs_labels"][i].to(torch.int32))
        labels_t = labels.t().contiguous()
        # without the graph attention the encoder writes its last h straight into the decoder's first operands
        xh_dec = self._xh("beam_t0" if cfg.use_beam_search and not cfg.use_gnn else "dec_class", n, h, w,
                          sw.dec_class.cpad, self.class_planes)
        c_e, h_e = self.encode_class(i, convs[i], obs_scene_t, labels_t,
                                     None if cfg.use_gnn else xh_dec[0])
        if cfg.use_beam_search:
          logits, ids, logprobs, _ = self.decode_class_beam(i, c_e, h_e, labels_t[-1].contiguous(),
                                                            means[i], tp, act, lengths)
          out["beam_outputs"] = [unsort(logits), unsort(ids), unsort(logprobs)]
          dec = out["beam_outputs"][0][:, 0].reshape(n, tp, h, w, 1)     # :799-803
          for j, t in enumerate(out["beam_outputs"]):
            emit("beam_outputs", j, t)
        else:
          lg, _ = self.decode_class_greedy(i, c_e, h_e, labels_t[-1].contiguous(), means[i], tp, act)
          dec = unsort(lg, 1).permute(1, 0, 2).reshape(n, tp, h, w, 1)
        emit("grid_pred_decoded", i, dec)
      if ("reg", i) in run:
        obs_reg = sort(feeds["grid_obs_regress"][i].float())
        obs_reg_t = obs_reg.transpose(0, 1).contiguous()
        xh_reg = self._xh("dec_reg", n, h, w, sw.dec_reg.cpad, self.fast_planes)
        c_r, _ = self.encode_reg(i, obs_reg_t, xh_reg[0])
        offs = unsort(self.decode_reg(i, c_r, obs_reg_t[-1], tp, xh_reg, act), 1)
        reg = offs.permute(1, 0, 2, 3).reshape(n, tp, h, w, 2)
        emit("grid_pred_reg_decoded", i, reg)
        out.setdefault("_offs", {})[i] = offs           # engine layout [Tp,N,HW,2], for decode_trajectories
      out["grid_pred_decoded"].append(dec)
      out["grid_pred_reg_decoded"].append(reg)
    if pred_lengths is not None:
      out["_lengths"] = torch.full((n,), tp, dtype=torch.int32, device=self.device) if lengths is None \
          else unsort(lengths)
    return out

  # ------------------------------------------------------------------ CUDA-graph replay of forward()
  @staticmethod
  def _flat_feeds(feeds):
    items = [("scene_feat", feeds["scene_feat"]), ("obs_scene", feeds["obs_scene"])]
    for name in ("grid_obs_labels", "grid_obs_regress"):
      for i, t in enumerate(feeds[name]):
        if t is not None:
          items.append(("%s/%d" % (name, i), t))
    return items

  def forward_graph(self, feeds, pred_len=None, on_output=None):
    """forward() captured per feed signature (shapes, dtypes, rollout length) into CUDA graphs and replayed:
    a forward is 120-950 kernel launches with no host-side data dependence (the beam loop has a fixed trip count and
    parents travel as device row maps), so at small batches - where the ~20 us the host spends per launch exceeds
    the kernels' run time - graph launches replace them.  Bit-identical to forward().  The returned tensors
    are the graphs' static outputs: they are overwritten by the next replay of the same signature.
    ONE GRAPH PER CHAIN (self.branches(): class / regression x scale), each with its own memory pool, replayed on
    its own stream: the chains share nothing but the feeds, and at these batch sizes a launch of one chain leaves SMs
    idle (64 rows of 36x18 = 2.4 waves of tiles) that the launches of another chain fill.  `on_output(name, index,
    tensor)` is called inside the chain's stream right after its graph has been launched, so a caller can start the
    device->host copy of the beam logits (87 % of the fetched bytes) while the other chains still run."""
    tp = int(pred_len) if pred_len else self.cfg.pred_len
    # The number of unique scene frames F changes from batch to batch in the reference's loops (scene_feat is
    # re-compacted per batch, code/pred_utils.py:680-704), so the graph is captured for F rounded up to a multiple
    # of 64: the scene CNN also runs on the padding frames, which no obs_scene index ever points at.
    sf = feeds["scene_feat"]
    f_pad = -(-int(sf.shape[0]) // 64) * 64
    flat = self._flat_feeds(feeds)
    key = (tp, f_pad) + tuple((k, tuple(t.shape[1:] if k == "scene_feat" else t.shape), t.dtype) for k, t in flat) + \
        (("MVB_BEAM_BAND", beam_band_on()),)     # a graph holds one of the two beam paths
    ent = self._graphs.get(key)
    main = torch.cuda.current_stream(self.device)
    if ent is None:
      if self.cell_events is not None:
        raise RuntimeError("forward_graph: per-launch event recording (cell_events) is an eager-mode feature")
      # A signature is captured the second time it is seen, and at most GRAPH_CACHE graphs are kept (each owns
      # the memory of its temporaries): callers whose feed shapes keep changing just run launch by launch.
      if key not in self._graph_seen:
        if len(self._graph_seen) >= 64:
          self._graph_seen.clear()
        self._graph_seen.add(key)
        return self.forward(feeds, tp, on_output=on_output)
      static = dict(scene_feat=torch.zeros((f_pad,) + tuple(sf.shape[1:]), dtype=sf.dtype, device=sf.device),
                    obs_scene=feeds["obs_scene"].clone(),
                    grid_obs_labels=[None if t is None else t.clone() for t in feeds["grid_obs_labels"]],
                    grid_obs_regress=[None if t is None else t.clone() for t in feeds["grid_obs_regress"]])
      static["scene_feat"][:sf.shape[0]].copy_(sf)
      self.forward(static, tp)        # eager pass: persistent buffers, kernel attributes, lazy caches
      torch.cuda.synchronize(self.device)
      chains = []
      for bi, br in enumerate(self.branches()):
        # the class chains are the long ones: their stream gets the higher priority (lower number)
        stream = self._buf(("graph_stream", bi), lambda: torch.cuda.Stream(device=self.device,
                                                                          priority=-1 if br[0] == "class" else 0))
        done = []
        stream.wait_stream(main)
        with torch.cuda.stream(stream):
          graph = torch.cuda.CUDAGraph()
          # thread_local: calls made by other threads (NCCL watchdog, profilers) must not invalidate the capture
          graph.capture_begin(capture_error_mode="thread_local")
          try:
            part = self.forward(static, tp, branches=[br], on_output=lambda *a: done.append(a))
          finally:
            graph.capture_end()
        main.wait_stream(stream)
        chains.append((br, stream, graph, done, part))
      out = dict(grid_pred_decoded=[[] for _ in self.cfg.scene_grids],
                 grid_pred_reg_decoded=[[] for _ in self.cfg.scene_grids], beam_outputs=None)
      for (kind, i), _, _, _, part in chains:
        if kind == "class":
          out["grid_pred_decoded"][i] = part["grid_pred_decoded"][i]
          if part["beam_outputs"] is not None:
            out["beam_outputs"] = part["beam_outputs"]
        else:
          out["grid_pred_reg_decoded"][i] = part["grid_pred_reg_decoded"][i]
          out.setdefault("_offs", {})[i] = part["_offs"][i]
      ent = (chains, static, out)
      while len(self._graphs) >= self.GRAPH_CACHE:
        self._graphs.pop(next(iter(self._graphs)))      # oldest first (dicts keep insertion order)
      self._graphs[key] = ent
    chains, static, out = ent
    for (name, dst), (_, src) in zip(self._flat_feeds(static), flat):
      (dst[:src.shape[0]] if name == "scene_feat" else dst).copy_(src, non_blocking=True)
    fed = main.record_event()
    # short chains first: their launches are in flight when the long chain starts and fill its partial waves
    for br, stream, graph, done, _ in sorted(chains, key=lambda c: c[0][0] != "reg"):
      stream.wait_event(fed)
      with torch.cuda.stream(stream):
        graph.replay()
        if on_output is not None:
          for name, index, t in done:
            on_output(name, index, t)
    for _, stream, _, _, _ in chains:
      main.wait_stream(stream)
    return out

  def grid_feeds_from_traj(self, obs_traj, centers=None, video_h=1080, video_w=1920):
    """Feed generation on the device (SURVEY.md §8 row f-1): the observed trajectories fp64 [N,T,2] (frame
    pixels; numpy or tensor) -> (grid_obs_labels, grid_obs_regress) lists per scale, i.e. what get_grid_input
    builds per trajectory on the host (code/multifuture_inference.py:115-156) and what 99 % of the fed bytes are.
    `centers[i]` fp64 [h,w,2]: the caller's args.scene_grid_centers; default = the reference's formula (:101-113).
    The returned tensors are per-engine buffers, overwritten by the next call with the same shapes."""
    import numpy as np
    cfg = self.cfg
    vh, vw = getattr(cfg, "video_h", video_h), getattr(cfg, "video_w", video_w)
    if torch.is_tensor(obs_traj):
      traj = obs_traj.to(self.device, torch.float64).contiguous()
    else:      # host array: through a pinned staging block, asynchronously on the current stream
      a = np.ascontiguousarray(obs_traj, dtype=np.float64)
      stage = self._buf(("traj_stage", a.shape), lambda: torch.empty(a.shape, dtype=torch.float64).pin_memory())
      ev = self._bufs.get(("traj_stage_event", a.shape))
      if ev is not None:
        ev.synchronize()                  # the previous call's copy out of the staging block has finished
      stage.copy_(torch.from_numpy(a))
      traj = stage.to(self.device, non_blocking=True)
      ev = torch.cuda.Event()
      ev.record(torch.cuda.current_stream(self.device))
      self._bufs[("traj_stage_event", a.shape)] = ev
    n, t = traj.shape[0], traj.shape[1]
    labels, regress = [], []
    for i, (h, w) in enumerate(cfg.scene_grids):
      if not cfg.use_grids[i]:
        labels.append(None); regress.append(None)
        continue
      h_gap, w_gap = vh * 1.0 / h, vw * 1.0 / w
      if centers is not None and centers[i] is not None:
        c = np.asarray(centers[i], dtype=np.float64).reshape(h * w, 2)
      else:
        cx = np.cumsum([w_gap] * w) - w_gap / 2.0
        cy = np.cumsum([h_gap] * h) - h_gap / 2.0
        c = np.stack((np.tile(cx[None], (h, 1)), np.tile(cy[:, None], (1, w))), axis=-1).reshape(h * w, 2)
      # the centres are a per-model constant: uploaded once per distinct array (keyed by its bytes)
      ckey = ("centers", i, hash(np.ascontiguousarray(c).tobytes()))
      c_dev = self._buf(ckey, lambda: torch.from_numpy(np.ascontiguousarray(c)).to(self.device))
      lab = self._buf(("traj_lab", i, n, t), lambda: torch.empty((n, t), dtype=torch.int32, device=self.device))
      reg = self._buf(("traj_reg", i, n, t), lambda: torch.empty((n, t, h, w, 2), dtype=torch.float32,
                                                                  device=self.device))
      ops.traj_to_grid(traj, c_dev, h_gap, w_gap, lab, reg, h, w)
      labels.append(lab); regress.append(reg)
    return labels, regress

  def grid_centers(self, i, video_h=1080, video_w=1920):
    """Cell centres of scale i in frame pixels (code/multifuture_inference.py:101-113)."""
    h, w = self.cfg.scene_grids[i]
    vh, vw = getattr(self.cfg, "video_h", video_h), getattr(self.cfg, "video_w", video_w)
    ys = (torch.arange(h, device=self.device, dtype=torch.float64) + 0.5) * (vh * 1.0 / h)
    xs = (torch.arange(w, device=self.device, dtype=torch.float64) + 0.5) * (vw * 1.0 / w)
    return torch.stack(torch.meshgrid(xs, ys, indexing="xy"), dim=-1).reshape(h * w, 2).float().contiguous()

  def decode_trajectories(self, out, i, centers=None):
    """Post-decode of a forward() result on the device (SURVEY.md §8 f-3): [N,K,Tp,2] pixel trajectories
    = centre + offset of the selected cells (beam ids, or the greedy arg-max with K = 1).  `centers`
    [h,w,2] / [HW,2]: the caller's args.scene_grid_centers[i]; default = grid_centers(i)."""
    offs = out["_offs"][i]
    tp, n = offs.shape[0], offs.shape[1]
    if out["beam_outputs"] is not None:
      ids = out["beam_outputs"][1].contiguous()
    else:
      ids = out["grid_pred_decoded"][i].reshape(n, tp, -1).argmax(-1).to(torch.int32).unsqueeze(1).contiguous()
    res = torch.empty(ids.shape + (2,), dtype=torch.float32, device=self.device)
    if centers is None:
      centers = self.grid_centers(i)
    else:
      centers = torch.as_tensor(centers).to(self.device, torch.float32).reshape(-1, 2).contiguous()
    ops.decode_trajectories(ids, offs.contiguous(), centers, res)
    return res
