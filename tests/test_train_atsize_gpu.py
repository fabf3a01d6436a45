# coding=utf-8
"""Every kernel of the training step around the ConvLSTM cell, element by element, at the micro-batch the training
workload runs (128 trajectories on the 36x18 and 18x9 grids), and the whole-model gradient at that micro-batch.

The unit tests of test_train_gpu.py run these kernels on 3 samples of toy grids.  Three kinds of code run only at
size:
  - grid-stride loops after their first pass (huber_loss, scene_time_mean[_bwd], clip_adadelta, clip_update launch
    at most 16 x SMs blocks);
  - reductions over many blocks: head_bwd / emb_bwd flush dWo / dWe / dbe with one atomic per element per block,
    scene_conv_bwd sums its dW terms over all the output pixels of its block (at most 8 x SMs blocks);
  - frames shared between trajectories: several trajectories per frame, windows of frames that overlap, labels
    that share a cell, so the scatters of enc_class_input[_mix]_bwd, scene_time_mean_bwd and the din of
    scene_conv_bwd collide across samples.
Every output is compared on the full tensors with a plain fp64 torch reference on the same device (the ref_*
functions below; gradients by torch autograd through them, no multiverse_b200 kernel involved), which the CPU test
of this file pins to the oracle's torch restatement.  Forward kernels that write the next step's bf16 x 2 operand
planes are checked through the values the planes sum back to.

Bars (max|diff| / max|ref| per tensor, as in the unit tests): FTOL 1e-5 for the fp32 kernels, ATOL 2e-5 for the
graph attention and the scene CNN, PTOL 3e-5 for values read back from bf16 x 2 planes, 2e-4 / 1e-4 for the
whole-model gradients / losses.  The GPU tests are marked one by one so that the CPU test runs under -m "not gpu"."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from test_kernels_atsize_gpu import _taps, halo_bits, halo_rows, inner, rel, to_halo
from oracle import multiverse_ref as R
from oracle import multiverse_ref_torch as RT

FTOL = 1e-5      # fp32 kernels (test_loss_kernel, test_head_and_emb_backward, test_clip_adadelta_matches_tf_formula)
ATOL = 2e-5      # graph attention and scene CNN (test_gnn_backward, test_scene_backward)
PTOL = 3e-5      # read back from bf16 x 2 operand planes (test_parity_gpu.py)
GTOL = 2e-4      # whole-model gradients (test_train_gpu.py)
LTOL = 1e-4      # whole-model losses
HID = 256
E = 32           # grid embedding size
NS = 128         # the training micro-batch
T_OBS, T_PRED = 8, 12
GRIDS = [(36, 18), (18, 9)]
SENTINEL = 1234.5


# --------------------------------------------------------------------------- fp64 reference (plain torch)
def _taps_s2(x):
  """[f, ih, iw, C] -> [f*oh*ow, 9*C]: im2col rows of the 3x3 stride-2 SAME convolution (TF padding: the extra row /
  column of padding goes after), tap-major."""
  f, ih, iw, c = x.shape
  oh, pt, pb = R.same_pad(ih, 3, 2)
  ow, pl, pr = R.same_pad(iw, 3, 2)
  p = F.pad(x, (0, 0, pl, pr, pt, pb))
  return torch.cat([p[:, dy:dy + 2 * oh - 1:2, dx:dx + 2 * ow - 1:2] for dy in range(3) for dx in range(3)],
                   -1).reshape(f * oh * ow, 9 * c)


def ref_scene_conv(x, W, b):
  """tanh(conv3x3 stride 2 SAME + b) (the scene CNN layer, code/pred_models.py:157-160) -> [f, oh, ow, Cout]."""
  f, ih, iw, _ = x.shape
  return torch.tanh(_taps_s2(x) @ W.reshape(-1, W.shape[-1]) + b).reshape(f, -(-ih // 2), -(-iw // 2), -1)


def ref_head(h, Wo):
  """hidden2grid: conv3x3 SAME of h [n, h, w, 256] with Wo [3,3,256,P], no bias -> [n, h*w, P]."""
  n, hh, ww, c = h.shape
  return (_taps(h) @ Wo.reshape(9 * c, -1)).reshape(n, hh * ww, -1)


def ref_emb(x, We, be):
  """grid_emb: tanh(conv3x3 SAME of x [n, h, w, P] + be) -> [n, h, w, E]."""
  n, hh, ww, p = x.shape
  return torch.tanh(_taps(x) @ We.reshape(9 * p, -1) + be).reshape(n, hh, ww, -1)


def ref_onehot(ids, h, w, dtype=torch.float64):
  """one_hot(ids) as an [n, h, w, 1] map."""
  return F.one_hot(ids.long(), h * w).to(dtype).reshape(-1, h, w, 1)


def ref_gnn(h, sm):
  """Graph attention + residual over the 3x3 band (what gnn_edge / gnn_mask_edge / gnn_node compute: the masked
  entries of the dense softmax are exactly zero): h [n, hh, ww, 256], sm the scene mean [n, hh, ww, 64] or None."""
  n, hh, ww, _ = h.shape
  f = h if sm is None else torch.cat([h, sm], -1)
  fn = f * torch.rsqrt(torch.clamp((f * f).sum(-1, keepdim=True), min=1e-12))
  pf = F.pad(fn, (0, 0, 1, 1, 1, 1))
  ph = F.pad(h, (0, 0, 1, 1, 1, 1))
  inside = F.pad(torch.ones((1, hh, ww), dtype=torch.bool, device=h.device), (1, 1, 1, 1))
  offs = [(dy, dx) for dy in range(3) for dx in range(3)]
  e = torch.stack([(fn * pf[:, dy:dy + hh, dx:dx + ww]).sum(-1) for dy, dx in offs], -1)
  ok = torch.stack([inside[:, dy:dy + hh, dx:dx + ww] for dy, dx in offs], -1)
  a = torch.softmax(e.masked_fill(~ok, float("-inf")), -1)
  return h + sum(a[..., k:k + 1] * ph[:, dy:dy + hh, dx:dx + ww] for k, (dy, dx) in enumerate(offs))


def ref_ce(logits, labels):
  """Mean sparse softmax cross entropy over the rows of logits [..., V]."""
  lg = logits.reshape(-1, logits.shape[-1])
  return (torch.logsumexp(lg, -1) - lg.gather(1, labels.reshape(-1, 1).long())[:, 0]).mean()


def ref_ce_rows(logits, labels):
  lg = logits.reshape(-1, logits.shape[-1])
  return torch.logsumexp(lg, -1) - lg.gather(1, labels.reshape(-1, 1).long())[:, 0]


def ref_huber(pred, target):
  """Mean Huber loss, delta 1."""
  a = (pred - target).abs()
  return torch.where(a <= 1.0, 0.5 * a * a, a - 0.5).mean()


def vjp(fn, inputs, upstream):
  """fn(*inputs) in fp64 and the gradients of sum(fn(*inputs) * upstream) with respect to every input."""
  xs = [x.detach().double().requires_grad_(True) for x in inputs]
  out = fn(*xs)
  gr = torch.autograd.grad(out, xs, upstream.double())
  return out.detach(), list(gr)


# --------------------------------------------------------------------------- CPU: the reference against the oracle
def test_reference_helpers_match_the_oracle():
  """ref_head / ref_emb / ref_gnn / ref_scene_conv / ref_ce / ref_huber (the reference of the GPU tests below) and
  their autograd gradients equal the oracle's torch restatement (conv2d_same, grid_emb, gnn_dense, F.cross_entropy,
  F.huber_loss as RT.loss_and_grads uses them) to 1e-12 on the unit-test shapes."""
  d64 = lambda a: torch.from_numpy(np.asarray(a)).double()
  rng = np.random.default_rng(7)
  hd = cases.head_case()
  ns, h, w, _ = hd["h"].shape
  for pout in (1, 2):
    Wo = d64(hd["Wo%d" % pout])
    up = d64(rng.standard_normal((ns, h * w, pout)))
    mine, g_mine = vjp(ref_head, [d64(hd["h"]), Wo], up)
    theirs, g_theirs = vjp(lambda a, b: RT.conv2d_same(a, b).reshape(ns, h * w, pout), [d64(hd["h"]), Wo], up)
    assert rel(mine, theirs) < 1e-12 and all(rel(a, b) < 1e-12 for a, b in zip(g_mine, g_theirs)), pout
    We, be = d64(hd["We%d" % pout]), d64(hd["be"])
    if pout == 1:
      ids = torch.from_numpy(rng.integers(0, h * w, size=ns))
      ids[0] = h * w - 1
      x = ref_onehot(ids, h, w)
      assert torch.equal(x, RT.one_hot_map(ids, h, w, torch.float64))
    else:
      x = d64(rng.standard_normal((ns, h, w, 2)) * 3)
    up = d64(rng.standard_normal((ns, h, w, E)))
    mine, g_mine = vjp(ref_emb, [x, We, be], up)
    theirs, g_theirs = vjp(RT.grid_emb, [x, We, be], up)
    assert rel(mine, theirs) < 1e-12 and all(rel(a, b) < 1e-12 for a, b in zip(g_mine, g_theirs)), pout
  gc = cases.gnn_case()
  ns, h, w, _ = gc["h"].shape
  hh = gc["h"].copy()
  sc = gc["scene"].copy()
  hh[0, 0, 0] = 0.0                          # zero norm (with the scene: the scene channels too)
  sc[0, 0, 0] = 0.0
  hh[1, 2, 1] = 1e-8 * np.sign(rng.standard_normal(256))     # |F|^2 = 2.6e-14: below the 1e-12 clamp
  sc[1, 2, 1] = 0.0
  mask = RT.neighbour_mask(h, w, torch.float64)
  up = d64(rng.standard_normal((ns, h, w, 256)))
  mine, g_mine = vjp(ref_gnn, [d64(hh), d64(sc)], up)
  theirs, g_theirs = vjp(lambda a, b: RT.gnn_dense(a, b, mask), [d64(hh), d64(sc)], up)
  assert rel(mine, theirs) < 1e-12 and all(rel(a, b) < 1e-12 for a, b in zip(g_mine, g_theirs))
  mine, g_mine = vjp(lambda a: ref_gnn(a, None), [d64(hh)], up)
  theirs, g_theirs = vjp(lambda a: RT.gnn_dense(a, None, mask), [d64(hh)], up)
  assert rel(mine, theirs) < 1e-12 and rel(g_mine[0], g_theirs[0]) < 1e-12
  s = cases.scene_case()
  x = d64(s["scene_feat"])
  for W, b in ((s["W1"], s["b1"]), (s["W2"], s["b2"])):
    W, b = d64(W), d64(b)
    out = ref_scene_conv(x, W, b)
    up = d64(rng.standard_normal(tuple(out.shape)))
    mine, g_mine = vjp(ref_scene_conv, [x, W, b], up)
    theirs, g_theirs = vjp(lambda a, k, c: torch.tanh(RT.conv2d_same(a, k, 2) + c), [x, W, b], up)
    assert mine.shape == theirs.shape and rel(mine, theirs) < 1e-12
    assert all(rel(a, b) < 1e-12 for a, b in zip(g_mine, g_theirs))
    x = out
  lg = d64(rng.standard_normal((7, 3, 50)) * 3)
  lab = torch.from_numpy(rng.integers(0, 50, size=(7, 3)))
  one = torch.ones((), dtype=torch.float64)
  mine, g_mine = vjp(lambda a: ref_ce(a, lab), [lg], one)
  theirs, g_theirs = vjp(lambda a: F.cross_entropy(a.reshape(-1, 50), lab.reshape(-1)), [lg], one)
  assert rel(mine, theirs) < 1e-12 and rel(g_mine[0], g_theirs[0]) < 1e-12
  pr, tg = d64(rng.standard_normal((7, 3, 50, 2)) * 2), d64(rng.standard_normal((7, 3, 50, 2)) * 2)
  mine, g_mine = vjp(lambda a: ref_huber(a, tg), [pr], one)
  theirs, g_theirs = vjp(lambda a: F.huber_loss(a, tg, delta=1.0), [pr], one)
  assert rel(mine, theirs) < 1e-12 and rel(g_mine[0], g_theirs[0]) < 1e-12


# --------------------------------------------------------------------------- shared-frame feeds
def shared_frame_feeds(cfg, n, frames, seed):
  """Feeds of n trajectories (synthetic.make_feeds: random walks, labels and offsets per scale) over `frames`
  distinct segmentation frames, as real batches see them: trajectory s observes the window of frames
  start_s .. start_s + 7, windows overlap, and pairs of trajectories share a frame window and the label cell of
  their first four observed steps."""
  from multiverse_b200 import synthetic
  f = synthetic.make_feeds(cfg, n, seed, with_pred=True)
  rng = np.random.default_rng(seed + 1)
  blocks = rng.integers(0, cfg.scene_class, size=(frames, -(-cfg.scene_h // 6), -(-cfg.scene_w // 3)))
  seg = np.repeat(np.repeat(blocks, 6, axis=1), 3, axis=2)[:, :cfg.scene_h, :cfg.scene_w]
  f["scene_feat"] = np.eye(cfg.scene_class, dtype=np.float32)[seg]
  start = rng.integers(0, frames - cfg.obs_len + 1, size=n)
  spread = np.concatenate([np.arange(2, n, 4), np.arange(3, n, 4)])[:frames - cfg.obs_len + 1]
  start[spread] = np.arange(spread.size)         # every frame is observed
  pairs = np.arange(0, n - 1, 4)                 # trajectories 4k and 4k+1
  start[pairs + 1] = start[pairs]
  f["obs_scene"] = (start[:, None] + np.arange(cfg.obs_len)[None]).astype(np.int32)
  for lab in f["grid_obs_labels"]:
    lab[pairs + 1, :4] = lab[pairs, :4]
  return f


def on(dev, a, dtype=None):
  t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
  return t if dtype is None else t.to(dtype)


@pytest.fixture(scope="module")
def dev():
  from multiverse_b200 import build
  build.build()
  return torch.device("cuda:0")


def gen(dev, seed):
  g = torch.Generator(device=dev)
  g.manual_seed(seed)
  return g


def interior_fill(t, ns, h, w, vals):
  """Write vals [ns, h, w, C] into the grid cells of the halo-layout buffer t [R, C], leaving the halo as it is."""
  t.view(ns, h + 1, w + 1, -1)[:, :h, :w] = vals


def halo_untouched(t, ns, h, w, value=SENTINEL):
  v = t.view(ns, h + 1, w + 1, -1)
  return bool((v[:, h] == value).all()) and bool((v[:, :, w] == value).all())


def report(tag, errs):
  print("%s: %s" % (tag, " ".join("%s %.2e" % kv for kv in errs.items())))


# --------------------------------------------------------------------------- loss
@pytest.mark.gpu
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_loss_at_size(dev, grid):
  """CE over [12, 128, V] logits and Huber over [12, 128, HW, 2] offsets (about 4 grid-stride passes of the Huber
  kernel at 36x18), errors on both sides of |e| = 1; then the mixed-label path as TrainEngine._backward_scale chains
  it (ce_rows, two CE launches with weights beta and 1 - beta summed into one gradient)."""
  from multiverse_b200 import ops
  h, w = grid
  v = h * w
  g = gen(dev, 200 + h)
  lg = torch.randn((T_PRED, NS, v), generator=g, device=dev) * 3
  lab = torch.randint(0, v, (T_PRED, NS), generator=g, device=dev, dtype=torch.int32)
  tgt = torch.randn((T_PRED, NS, v, 2), generator=g, device=dev) * 200
  pr = tgt + torch.randn((T_PRED, NS, v, 2), generator=g, device=dev) * 1.5
  e = (pr - tgt).abs()
  assert float((e < 1).float().mean()) > 0.3 and float((e > 1).float().mean()) > 0.3
  cw, rw = 1.0 * 0.5, 0.1 * 0.5                  # loss weights times a micro-batch scale
  one = torch.ones((), dtype=torch.float64, device=dev)
  ce, (dce,) = vjp(lambda a: ref_ce(a, lab) * cw, [lg], one)
  hb, (dhb,) = vjp(lambda a: ref_huber(a, tgt.double()) * rw, [pr], one)
  dl = torch.full_like(lg, SENTINEL)
  dp = torch.full_like(pr, SENTINEL)
  out = torch.zeros(2, device=dev)
  ops.loss_fwd_bwd(lg, lab, dl, cw, pr, tgt, dp, rw, out)
  errs = {"ce": abs(float(out[0]) - float(ce)) / abs(float(ce)), "huber": abs(float(out[1]) - float(hb)) / abs(float(hb)),
          "dlogits": rel(dl, dce), "doffsets": rel(dp, dhb)}
  # mixed labels
  beta = 0.7
  lab2 = torch.randint(0, v, (T_PRED, NS), generator=g, device=dev, dtype=torch.int32)
  lab2[:, ::5] = lab[:, ::5]                     # both views in the same cell on some rows
  rows1, rows2 = ops.ce_rows(lg, lab), ops.ce_rows(lg, lab2)
  mixed, (dmix,) = vjp(lambda a: (beta * ref_ce_rows(a, lab) + (1 - beta) * ref_ce_rows(a, lab2)).mean() * cw,
                       [lg], one)
  scratch = torch.zeros(2, device=dev)
  dl1, dl2 = torch.full_like(lg, SENTINEL), torch.full_like(lg, SENTINEL)
  ops.loss_fwd_bwd(lg, lab, dl1, cw * beta, None, None, None, 0.0, scratch)
  ops.loss_fwd_bwd(lg, lab2, dl2, cw * (1.0 - beta), None, None, None, 0.0, scratch)
  got_mixed = float((beta * rows1.double() + (1 - beta) * rows2.double()).mean()) * cw
  errs.update({"ce_rows": rel(rows1.reshape(-1), ref_ce_rows(lg.double(), lab)), "mixed": abs(got_mixed - float(mixed)) / float(mixed),
               "mixed scratch": abs(float(scratch[0]) - float(mixed)) / float(mixed), "dlogits mixed": rel(dl1 + dl2, dmix)})
  report("loss %dx%d" % grid, errs)
  for k, err in errs.items():
    assert err < FTOL, (k, err)


# --------------------------------------------------------------------------- heads
def head_inputs(dev, h, w, seed, steps=1):
  """h32 halo states of `steps` steps (tanh of normal), the class / regression head weights at the scale of
  synthetic.make_weights (he-normal x 4), the grid embeddings."""
  g = gen(dev, seed)
  hs = [torch.tanh(torch.randn((NS, h, w, HID), generator=g, device=dev)) for _ in range(steps)]
  he = lambda *s: torch.randn(s, generator=g, device=dev).clamp(-2, 2) * math.sqrt(2.0 / (9 * s[2]))
  return dict(h=hs, Wo1=he(3, 3, HID, 1) * 4, Wo2=he(3, 3, HID, 2) * 4, We1=he(3, 3, 1, E), We2=he(3, 3, 2, E),
              be=torch.randn((E,), generator=g, device=dev) * 0.05, g=g)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_heads_forward_at_size(dev, grid):
  """head_class_fwd (logits, arg-max ids, the embedded one-hot of the ids as the next step's x planes) and
  head_reg_fwd (offsets, their dense embedding as x planes), planes = 2, 128 samples."""
  from multiverse_b200 import ops
  h, w = grid
  d = head_inputs(dev, h, w, 210 + h)
  h32 = to_halo(d["h"][0])
  cpad = ops.cell_cpad(E)
  # class head
  logits = torch.empty((NS, h * w), device=dev)
  ids = torch.empty((NS,), dtype=torch.int32, device=dev)
  xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
  ops.head_class_fwd(h32, d["Wo1"], logits, ids, d["We1"], d["be"], xh, h, w, NS, planes=2)
  ref = ref_head(d["h"][0].double(), d["Wo1"].double())[..., 0]
  err_abs = float((logits.double() - ref).abs().max())
  srt = ref.sort(-1, descending=True).values
  clear = (srt[:, 0] - srt[:, 1]) > 10 * err_abs
  assert torch.equal(ids.long(), logits.argmax(-1)), "ids are not the arg-max of the kernel's logits"
  assert bool((ids.long() == ref.argmax(-1))[clear].all()) and int(clear.sum()) > NS // 2
  vals, _ = ops.operand_values(xh)
  emb = ref_emb(ref_onehot(ids, h, w), d["We1"].double(), d["be"].double())
  errs = {"logits": rel(logits, ref), "emb planes": rel(inner(vals, NS, h, w)[..., :E], emb)}
  assert float(vals[:, E:].abs().max()) == 0.0 and halo_bits(xh, NS, h, w) == 0
  # regression head
  offs = torch.empty((NS, h * w, 2), device=dev)
  xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
  ops.head_reg_fwd(h32, d["Wo2"], offs, d["We2"], d["be"], xh, h, w, NS, planes=2)
  ref = ref_head(d["h"][0].double(), d["Wo2"].double())
  vals, _ = ops.operand_values(xh)
  emb = ref_emb(offs.double().view(NS, h, w, 2), d["We2"].double(), d["be"].double())
  errs.update({"offsets": rel(offs, ref), "dense emb planes": rel(inner(vals, NS, h, w)[..., :E], emb)})
  assert float(vals[:, E:].abs().max()) == 0.0 and halo_bits(xh, NS, h, w) == 0
  report("heads fwd %dx%d (%d of %d arg-max rows clear of fp32 error)" % (h, w, int(clear.sum()), NS), errs)
  for k in ("logits", "offsets"):
    assert errs[k] < FTOL, (k, errs[k])
  for k in ("emb planes", "dense emb planes"):
    assert errs[k] < PTOL, (k, errs[k])


@pytest.mark.gpu
@pytest.mark.parametrize("pout", [1, 2])
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_head_backward_chained_at_size(dev, grid, pout):
  """head_bwd over the 12 decoder steps into one dWo (128 blocks x 12 launches of atomics), dh as the engine passes
  it: overwritten at the last step, added to what the graph attention left there at the others.  The halo rows of
  dh hold a sentinel that must survive."""
  from multiverse_b200 import ops
  h, w = grid
  d = head_inputs(dev, h, w, 220 + 3 * h + pout, steps=T_PRED)
  g = d["g"]
  Wo = d["Wo%d" % pout]
  dWo = torch.zeros_like(Wo)
  dWo_ref = torch.zeros_like(Wo, dtype=torch.float64)
  dh = torch.full((halo_rows(NS, h, w), HID), SENTINEL, device=dev)
  worst = 0.0
  for t in range(T_PRED - 1, -1, -1):
    dout = torch.randn((NS, h * w, pout), generator=g, device=dev)
    carry = torch.randn((NS, h, w, HID), generator=g, device=dev)
    interior_fill(dh, NS, h, w, carry)
    ops.head_bwd(to_halo(d["h"][t]), dout, Wo, dWo, dh, t < T_PRED - 1, h, w, NS)
    _, (gh, gW) = vjp(ref_head, [d["h"][t], Wo], dout)
    want = gh + carry.double() if t < T_PRED - 1 else gh
    worst = max(worst, rel(inner(dh, NS, h, w), want))
    dWo_ref += gW
  errs = {"dh (worst step)": worst, "dWo (12 steps)": rel(dWo, dWo_ref)}
  report("head_bwd P_out %d %dx%d" % (pout, h, w), errs)
  assert halo_untouched(dh, NS, h, w), "head_bwd wrote a halo row of dh"
  for k, err in errs.items():
    assert err < FTOL, (k, err)


# --------------------------------------------------------------------------- embeddings
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["onehot", "dense", "mixup_pad"])
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_emb_backward_at_size(dev, grid, mode):
  """emb_bwd, 12 launches accumulating into dWe / dbe.  onehot: P_out = 1, ids in the corners and on the edges
  (taps cut off by the border);  dense: P_out = 2 on an offset map, d_in accumulating;  mixup_pad: the mixed
  two-cell first input of the class decoder (channel 0 = beta at l1 + (1 - beta) at l2, l1 == l2 on some rows)
  through the embedding padded with a zero second channel."""
  from multiverse_b200 import ops
  h, w = grid
  hw = h * w
  g = gen(dev, 240 + h + len(mode))
  pout = 1 if mode == "onehot" else 2
  We = torch.randn((3, 3, pout, E), generator=g, device=dev) * 0.5
  be = torch.randn((E,), generator=g, device=dev) * 0.2
  if mode == "mixup_pad":
    We[:, :, 1:] = 0.0
  cpad = ops.cell_cpad(E)
  dWe, dbe = torch.zeros_like(We), torch.zeros_like(be)
  dWe_ref, dbe_ref = torch.zeros_like(We, dtype=torch.float64), torch.zeros_like(be, dtype=torch.float64)
  worst_din = 0.0
  for step in range(T_PRED):
    dxh = torch.randn((halo_rows(NS, h, w), cpad), generator=g, device=dev)
    dx = inner(dxh, NS, h, w)[..., :E]
    if mode == "onehot":
      ids = torch.randint(0, hw, (NS,), generator=g, device=dev, dtype=torch.int32)
      ids[:6] = torch.tensor([0, w - 1, hw - w, hw - 1, w, 2 * w - 1], dtype=torch.int32)
      ops.emb_bwd(dxh, ids, None, We, be, dWe, dbe, None, False, h, w, NS)
      _, (gW, gb) = vjp(lambda a, b: ref_emb(ref_onehot(ids, h, w), a, b), [We, be], dx)
    else:
      if mode == "dense":
        in_map = torch.randn((NS, hw, 2), generator=g, device=dev) * 3
      else:
        beta = 0.7
        l1 = torch.randint(0, hw, (NS,), generator=g, device=dev)
        l2 = torch.randint(0, hw, (NS,), generator=g, device=dev)
        l2[::3] = l1[::3]
        l1[:4] = torch.tensor([0, w - 1, hw - w, hw - 1], device=dev)
        in_map = torch.zeros((NS, hw, 2), device=dev)
        rows = torch.arange(NS, device=dev)
        in_map[:, :, 0].index_put_((rows, l1), torch.full((NS,), beta, device=dev), accumulate=True)
        in_map[:, :, 0].index_put_((rows, l2), torch.full((NS,), 1.0 - beta, device=dev), accumulate=True)
      din = torch.randn((NS, hw, 2), generator=g, device=dev) if mode == "dense" else None
      din0 = None if din is None else din.clone()
      ops.emb_bwd(dxh, None, in_map, We, be, dWe, dbe, din, mode == "dense", h, w, NS)
      _, (gx, gW, gb) = vjp(ref_emb, [in_map.view(NS, h, w, 2), We, be], dx)
      if din is not None:
        worst_din = max(worst_din, rel(din.double() - din0.double(), gx.reshape(NS, hw, 2)))
    dWe_ref += gW
    dbe_ref += gb
  if mode == "mixup_pad":          # the engine keeps the first channel: the class embedding has one input channel
    errs = {"dWe": rel(dWe[:, :, :1], dWe_ref[:, :, :1]), "dbe": rel(dbe, dbe_ref)}
  else:
    errs = {"dWe": rel(dWe, dWe_ref), "dbe": rel(dbe, dbe_ref)}
  if mode == "dense":
    errs["d_in (worst step)"] = worst_din
  report("emb_bwd %s %dx%d, 12 launches" % (mode, h, w), errs)
  for k, err in errs.items():
    assert err < FTOL, (k, err)


# --------------------------------------------------------------------------- graph attention
CLAMPED = [(0, 0, 0, 0.0), (1, 0.5, 0.5, 1e-8), (2, 0.5, 0.0, 4.4e-8)]   # sample, y / h, x / w, |h_c|


def gnn_inputs(dev, h, w, seed, with_scene):
  """h (tanh of normal) and the scene mean, with three cells under the 1e-12 clamp of l2_normalize's squared norm:
  a zero-norm cell in a corner, a squared norm of 2.6e-14 and one of 5e-13 (between 1e-12 / 2 and 1e-12 the kernel
  sees the clamp only through rsqrtf(1e-12f) >= 1e6f).  Returns h, the scene mean (or None), the generator and the
  mask of those cells."""
  g = gen(dev, seed)
  hs = torch.tanh(torch.randn((NS, h, w, HID), generator=g, device=dev))
  sm = torch.tanh(torch.randn((NS, h, w, 64), generator=g, device=dev)) if with_scene else None
  clamped = torch.zeros((NS, h, w), dtype=torch.bool, device=dev)
  for s, fy, fx, mag in CLAMPED:
    y, x = int(fy * (h - 1)), int(fx * (w - 1))
    hs[s, y, x] = mag * torch.sign(torch.randn((HID,), generator=g, device=dev))
    if sm is not None:
      sm[s, y, x] = 0.0
    clamped[s, y, x] = True
  return hs, sm, g, clamped


@pytest.mark.gpu
@pytest.mark.parametrize("with_scene", [True, False], ids=["scene", "h_only"])
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_gnn_forward_at_size(dev, grid, with_scene):
  """gnn_attend_fwd into the h block of the class decoder's operand planes (planes = 2)."""
  from multiverse_b200 import ops
  h, w = grid
  hs, sm, _, _ = gnn_inputs(dev, h, w, 260 + h, with_scene)
  cpad = ops.cell_cpad(E)
  xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
  ops.gnn_attend_fwd(to_halo(hs), sm, xh, h, w, NS)
  vals, _ = ops.operand_values(xh)
  err = rel(inner(vals, NS, h, w)[..., E:], ref_gnn(hs.double(), None if sm is None else sm.double()))
  report("gnn fwd %dx%d %s" % (h, w, "scene" if with_scene else "h only"), {"h' planes": err})
  assert float(vals[:, :E].abs().max()) == 0.0 and halo_bits(xh, NS, h, w) == 0
  assert err < PTOL


@pytest.mark.gpu
@pytest.mark.parametrize("with_scene", [True, False], ids=["scene", "h_only"])
@pytest.mark.parametrize("grid", GRIDS, ids=["36x18", "18x9"])
def test_gnn_backward_at_size(dev, grid, with_scene):
  """gnn_bwd over the 12 decoder steps: dh of every step, d(scene mean) accumulated over the 12 launches; the halo
  rows of dh hold a sentinel that must survive.  The gradient at a clamped cell is about 1e6 x larger than
  elsewhere (l2_normalize divides by 1e-6 there), so the clamped cells and the others are compared separately."""
  from multiverse_b200 import ops
  h, w = grid
  _, sm, g, cl = gnn_inputs(dev, h, w, 270 + h, with_scene)
  work = torch.empty((19 * NS * h * w,), device=dev)
  dh = torch.full((halo_rows(NS, h, w), HID), SENTINEL, device=dev)
  dsm = torch.zeros_like(sm) if with_scene else None
  dsm_ref = torch.zeros_like(sm, dtype=torch.float64) if with_scene else None
  worst = {"dh (worst step)": 0.0, "dh clamped cells": 0.0}
  for t in range(T_PRED):
    hs, _, _, _ = gnn_inputs(dev, h, w, 280 + 7 * t + h, False)
    gout = torch.randn((NS, h, w, HID), generator=g, device=dev)
    ops.gnn_bwd(to_halo(hs), sm, to_halo(gout), work, dh, False, dsm, h, w, NS)
    if with_scene:
      _, (gh, gs) = vjp(ref_gnn, [hs, sm], gout)
      dsm_ref += gs
    else:
      _, (gh,) = vjp(lambda a: ref_gnn(a, None), [hs], gout)
    got = inner(dh, NS, h, w)
    worst["dh (worst step)"] = max(worst["dh (worst step)"], rel(got[~cl], gh[~cl]))
    worst["dh clamped cells"] = max(worst["dh clamped cells"], rel(got[cl], gh[cl]))
  errs = dict(worst)
  if with_scene:
    errs["dscene_mean (12 steps)"] = rel(dsm[~cl], dsm_ref[~cl])
    errs["dscene_mean clamped cells"] = rel(dsm[cl], dsm_ref[cl])
  report("gnn_bwd %dx%d %s" % (h, w, "scene" if with_scene else "h only"), errs)
  assert halo_untouched(dh, NS, h, w), "gnn_bwd wrote a halo row of dh"
  for k, err in errs.items():
    assert err < ATOL, (k, err)


# --------------------------------------------------------------------------- scene CNN on shared frames
FRAMES = 48


@pytest.fixture(scope="module")
def scene(dev):
  """The shared-frame feeds of 128 trajectories over 48 frames, the scene CNN weights (synthetic.make_weights) and
  the kernels' forward outputs."""
  from multiverse_b200 import ops, synthetic
  cfg = synthetic.make_config()
  f = shared_frame_feeds(cfg, NS, FRAMES, 300)
  wts = synthetic.make_weights(cfg, 300)
  W = [on(dev, wts["person_pred/scene_conv%d/W" % k]) for k in (1, 2)]
  b = [on(dev, wts["person_pred/scene_conv%d/b" % k]) for k in (1, 2)]
  x = on(dev, f["scene_feat"])
  conv1 = ops.scene_conv_fwd(x, W[0], b[0])
  conv2 = ops.scene_conv_fwd(conv1, W[1], b[1])
  return dict(f=f, x=x, W=W, b=b, convs=[conv1, conv2], obs=on(dev, f["obs_scene"]),
              labels=[on(dev, a, torch.int32) for a in f["grid_obs_labels"]])


def test_shared_frame_feeds_share_frames_and_cells():
  """The feeds the scene tests run on do share what they claim to (CPU)."""
  from multiverse_b200 import synthetic
  cfg = synthetic.make_config()
  f = shared_frame_feeds(cfg, NS, FRAMES, 300)
  obs = f["obs_scene"]
  assert obs.min() >= 0 and obs.max() < FRAMES and np.all(np.diff(obs, axis=1) == 1)
  uses = np.bincount(obs.reshape(-1), minlength=FRAMES)
  assert uses.max() >= 20 and (uses > 0).sum() == FRAMES          # every frame is used, some by many trajectories
  for lab in f["grid_obs_labels"]:
    key = obs * 10000 + lab                                      # (frame, cell) of every observed step
    same = [len(set(key[:, t])) < NS for t in range(cfg.obs_len)]
    assert all(same[:4])


@pytest.mark.gpu
def test_scene_forward_on_shared_frames(dev, scene):
  """scene_conv_fwd (both layers), scene_time_mean over overlapping windows (about 10 grid-stride passes at 36x18),
  enc_class_input and enc_class_input_mix into the class encoder's x planes, on both grids."""
  from multiverse_b200 import ops
  x64 = scene["x"].double()
  c1 = ref_scene_conv(x64, scene["W"][0].double(), scene["b"][0].double())
  c2 = ref_scene_conv(scene["convs"][0].double(), scene["W"][1].double(), scene["b"][1].double())
  errs = {"conv1": rel(scene["convs"][0], c1), "conv2": rel(scene["convs"][1], c2)}
  obs = scene["obs"]
  cpad = ops.cell_cpad(64)
  worst = {"mean": 0.0, "input planes": 0.0, "mix planes": 0.0}
  for i, (h, w) in enumerate(GRIDS):
    conv = scene["convs"][i]
    mean = ops.scene_time_mean(conv, obs)
    worst["mean"] = max(worst["mean"], rel(mean, conv.double()[obs.long()].mean(1)))
    lab = scene["labels"][i]
    lab2 = lab.flip(0).contiguous()
    lab2[::3] = lab[::3]
    for t in range(T_OBS):
      fr = obs[:, t].contiguous()
      sel = torch.zeros((NS, h * w, 64), dtype=torch.float64, device=dev)
      rows = torch.arange(NS, device=dev)
      sel[rows, lab[:, t].long()] = conv.double().view(-1, h * w, 64)[fr.long(), lab[:, t].long()]
      xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
      ops.enc_class_input(conv, fr, lab[:, t].contiguous(), None, xh, h, w)
      vals, _ = ops.operand_values(xh)
      worst["input planes"] = max(worst["input planes"], rel(inner(vals, NS, h, w)[..., :64], sel.view(NS, h, w, 64)))
      assert float(vals[:, 64:].abs().max()) == 0.0 and halo_bits(xh, NS, h, w) == 0
      beta = 0.7
      mix = torch.zeros((NS, h * w), dtype=torch.float64, device=dev)
      mix.index_put_((rows, lab[:, t].long()), torch.full((NS,), beta, dtype=torch.float64, device=dev), accumulate=True)
      mix.index_put_((rows, lab2[:, t].long()), torch.full((NS,), 1 - beta, dtype=torch.float64, device=dev),
                     accumulate=True)
      xh = ops.alloc_xh(NS, h, w, cpad, 2, dev)
      ops.enc_class_input_mix(conv, fr, lab[:, t].contiguous(), lab2[:, t].contiguous(), beta, xh, h, w)
      vals, _ = ops.operand_values(xh)
      want = conv.double()[fr.long()].view(NS, h * w, 64) * mix[..., None]
      worst["mix planes"] = max(worst["mix planes"], rel(inner(vals, NS, h, w)[..., :64], want.view(NS, h, w, 64)))
  errs.update(worst)
  report("scene fwd, %d trajectories over %d frames" % (NS, FRAMES), errs)
  for k in ("conv1", "conv2", "mean"):
    assert errs[k] < ATOL, (k, errs[k])
  for k in ("input planes", "mix planes"):
    assert errs[k] < PTOL, (k, errs[k])


@pytest.mark.gpu
def test_scene_backward_on_shared_frames(dev, scene):
  """The scene-feature gradient as the training step assembles it, on shared frames: enc_class_input_bwd over the 8
  observed steps and scene_time_mean_bwd scatter into d(conv) of each scale (enc_class_input_mix_bwd alongside);
  then scene_conv_bwd of layer 2 (the KPG 144 instantiation, din added into d(conv1)) and of layer 1 (KPG 25, din
  into d(scene_feat)).  Each kernel is compared with the fp64 reference on the kernel's own inputs."""
  from multiverse_b200 import ops
  g = gen(dev, 310)
  obs = scene["obs"]
  cpad = ops.cell_cpad(64)
  errs = {}
  dconv = []
  for i, (h, w) in enumerate(GRIDS):
    conv = scene["convs"][i]
    lab = scene["labels"][i]
    lab2 = lab.flip(0).contiguous()
    lab2[::3] = lab[::3]
    beta = 0.7
    dc = torch.zeros_like(conv)
    dmix = torch.zeros_like(conv)
    ref = torch.zeros_like(conv, dtype=torch.float64)
    ref_mix = torch.zeros_like(conv, dtype=torch.float64)
    rows = torch.arange(NS, device=dev)
    for t in range(T_OBS):
      dxh = torch.randn((halo_rows(NS, h, w), cpad), generator=g, device=dev)
      fr, l1, l2 = obs[:, t].contiguous(), lab[:, t].contiguous(), lab2[:, t].contiguous()
      ops.enc_class_input_bwd(dxh, fr, l1, dc, h, w)
      ops.enc_class_input_mix_bwd(dxh, fr, l1, l2, beta, dmix, h, w)
      dx = inner(dxh, NS, h, w)[..., :64].double().reshape(NS, h * w, 64)
      flat, flat_mix = ref.view(-1, h * w, 64), ref_mix.view(-1, h * w, 64)
      flat.index_put_((fr.long(), l1.long()), dx[rows, l1.long()], accumulate=True)
      flat_mix.index_put_((fr.long(), l1.long()), dx[rows, l1.long()] * beta, accumulate=True)
      flat_mix.index_put_((fr.long(), l2.long()), dx[rows, l2.long()] * (1 - beta), accumulate=True)
    dmean = torch.randn((NS, h, w, 64), generator=g, device=dev)
    ops.scene_time_mean_bwd(dmean, obs, dc)
    for t in range(T_OBS):
      ref.index_add_(0, obs[:, t].long(), dmean.double() / T_OBS)
    errs["dconv%d" % (i + 1)] = rel(dc, ref)
    errs["dconv%d mix" % (i + 1)] = rel(dmix, ref_mix)
    dconv.append(dc)
  conv1, conv2 = scene["convs"]
  dW2, db2 = torch.zeros_like(scene["W"][1]), torch.zeros_like(scene["b"][1])
  dconv1_in = dconv[0].clone()
  ops.scene_conv_bwd(conv1, scene["W"][1], conv2, dconv[1], dW2, db2, dconv[0])
  _, (gx, gW, gb) = vjp(ref_scene_conv, [conv1, scene["W"][1], scene["b"][1]], dconv[1])
  errs.update({"dW2": rel(dW2, gW), "db2": rel(db2, gb), "din2 (into dconv1)": rel(dconv[0].double() - dconv1_in.double(), gx)})
  dW1, db1 = torch.zeros_like(scene["W"][0]), torch.zeros_like(scene["b"][0])
  dx = torch.zeros_like(scene["x"])
  ops.scene_conv_bwd(scene["x"], scene["W"][0], conv1, dconv[0], dW1, db1, dx)
  _, (gx, gW, gb) = vjp(ref_scene_conv, [scene["x"], scene["W"][0], scene["b"][0]], dconv[0])
  errs.update({"dW1": rel(dW1, gW), "db1": rel(db1, gb), "din1": rel(dx, gx)})
  report("scene bwd, %d trajectories over %d frames" % (NS, FRAMES), errs)
  for k, err in errs.items():
    assert err < ATOL, (k, err)


# --------------------------------------------------------------------------- optimizer
OPTS = {
    # name: (clip_update kind or 0 for clip_adadelta, lr, p1, p2, eps)
    "adadelta": (0, 1.0, 0.95, 0.0, 1e-8),
    "momentum": (1, 0.05, 0.9, 0.0, 0.0),
    "adam": (2, 0.05, 0.9, 0.999, 1e-8),
    "rmsprop": (3, 0.05, 0.9, 0.0, 1e-10),
}


def ref_update(name, w, g, s1, s2, lr, p1, p2, eps, clip, wd, gs):
  """One step of the fp64 formulas of test_clip_adadelta_matches_tf_formula / test_other_optimizers_match_tf_semantics
  -> (w, s1, s2).  The hyper-parameters are the fp32 values the kernel receives (TF casts them to the variable's
  dtype as well): 1 - float32(0.999) differs from 0.001 by 1.3e-5 relative."""
  gg = torch.clamp(g * gs + wd * w, -clip, clip)
  if name == "adadelta":
    a = p1 * s1 + (1 - p1) * gg * gg
    u = torch.sqrt(s2 + eps) / torch.sqrt(a + eps) * gg
    return w - lr * u, a, p1 * s2 + (1 - p1) * u * u
  if name == "momentum":
    a = p1 * s1 + gg
    return w - lr * a, a, s2
  if name == "adam":          # lr: the bias-corrected rate of TrainEngine.apply_gradients
    m, v = p1 * s1 + (1 - p1) * gg, p2 * s2 + (1 - p2) * gg * gg
    return w - lr * m / (torch.sqrt(v) + eps), m, v
  ms = p1 * s1 + (1 - p1) * gg * gg
  mom = p2 * s2 + lr * gg / torch.sqrt(ms + eps)
  return w - mom, ms, mom


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(OPTS))
def test_optimizer_on_every_variable(dev, name):
  """clip_adadelta / clip_update on tensors shaped like every variable of the two-scale config (21.3 M elements:
  about 5 grid-stride passes on one ConvLSTM kernel), two steps, grad_scale 1/8, weight decay on .../W only,
  gradients on both sides of +-clip.  The weight is compared through its update w' - w (relative to the reference
  update), the slots directly."""
  from multiverse_b200 import ops, synthetic
  kind, lr, p1, p2, eps = OPTS[name]
  clip, wdc, gs = 10.0, 0.001, 1.0 / 8
  cfg = synthetic.make_config()
  wts = synthetic.make_weights(cfg, 320)
  g = gen(dev, 320 + kind)
  worst = {"dw": 0.0, "s1": 0.0, "s2": 0.0}
  n_el, n_clipped = 0, 0
  for k, shp in sorted(synthetic.weight_shapes(cfg).items()):
    wd = wdc if k.endswith("/W") else 0.0
    w = on(dev, wts[k])
    if name == "adadelta":
      s1 = torch.randn(shp, generator=g, device=dev).abs()
      s2 = torch.randn(shp, generator=g, device=dev).abs() * 1e-3
    else:
      s1 = torch.ones_like(w) if name == "rmsprop" else torch.zeros_like(w)
      s2 = torch.zeros_like(w)
    r = [w.double(), s1.double(), s2.double()]
    for t in (1, 2):
      grad = torch.randn(shp, generator=g, device=dev) * 80
      gg = grad.double() * gs + wd * w.double()
      n_el += gg.numel()
      n_clipped += int((gg.abs() > clip).sum())
      w_old = w.clone()
      lr_t = lr * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) if name == "adam" else lr
      if kind == 0:
        ops.clip_adadelta(w, grad, s1, s2, lr_t, clip, wd, grad_scale=gs, rho=p1, eps=eps)
      else:
        ops.clip_update(w, grad, s1, s2, kind, lr_t, p1, p2, eps, clip, wd, grad_scale=gs)
      # the reference step starts from the kernel's fp32 state of the previous step
      f32 = lambda v: float(np.float32(v))
      w_ref, a_ref, b_ref = ref_update(name, w_old.double(), grad.double(), r[1], r[2], f32(lr_t), f32(p1), f32(p2),
                                       f32(eps), clip, f32(wd), gs)
      worst["dw"] = max(worst["dw"], rel(w.double() - w_old.double(), w_ref - w_old.double()))
      worst["s1"] = max(worst["s1"], rel(s1, a_ref))
      if name != "momentum":
        worst["s2"] = max(worst["s2"], rel(s2, b_ref))
      r = [w.double(), s1.double(), s2.double()]
  report("%s on %d variables, %.1f M elements per step, %.0f %% clipped" % (
      name, len(synthetic.weight_shapes(cfg)), n_el / 2e6, 100.0 * n_clipped / n_el), worst)
  assert 0.05 < n_clipped / n_el < 0.95
  assert worst["dw"] < 2e-5 and worst["s1"] < FTOL, worst
  assert worst["s2"] < (1e-4 if name == "adadelta" else FTOL), worst


# --------------------------------------------------------------------------- whole model at the micro-batch
WM_SEED = 337       # seeds 330-336 put some decoded arg-max of the fp64 reference within 1e-4 x max|logit| of a tie
MARGIN = 1e-4        # smallest top-2 logit gap the class decoder's arg-max may have, relative to max|logit| (the
                     # engine's logit error at this size measures 1.3e-5 at 36x18, 2.1e-5 at 18x9)


def wm_configs(n, chunk):
  from multiverse_b200 import synthetic
  loss = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.1, wd=0.001)
  return synthetic.make_config(batch_size=n, clip_gradient_norm=10.0, **loss), R.default_config(batch_size=chunk, **loss)


def chunk_feeds(f, sl):
  """Trajectories `sl` of the feeds, with the whole frame table (the reference indexes it with obs_scene)."""
  out = dict(scene_feat=f["scene_feat"], obs_scene=f["obs_scene"][sl])
  for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    out[k] = [a[sl] for a in f[k]]
  return out


@pytest.mark.gpu
def test_reference_on_cuda_equals_reference_on_cpu(dev):
  """RT.loss_and_grads on the GPU (im2col convolutions) equals the CPU path to 1e-10: losses, every gradient and the
  decoded logits, batch 2, both scales."""
  from multiverse_b200 import synthetic
  cfg, rcfg = wm_configs(2, 2)
  w = synthetic.make_weights(cfg, 31)
  f = synthetic.make_feeds(cfg, 2, 31, with_pred=True)
  tot_c, l_c, wd_c, g_c, lg_c = RT.loss_and_grads(rcfg, w, f, return_logits=True)
  tot_g, l_g, wd_g, g_g, lg_g = RT.loss_and_grads(rcfg, w, f, device=dev, return_logits=True)
  assert abs(tot_g - tot_c) <= 1e-10 * abs(tot_c) and abs(wd_g - wd_c) <= 1e-10 * wd_c
  assert np.abs(np.array(l_g) - np.array(l_c)).max() <= 1e-10 * max(l_c)
  worst = max(rel(g_g[k], g_c[k]) for k in g_c if np.abs(g_c[k]).max() > 0)
  assert worst < 1e-10, worst
  for a, b in zip(lg_g, lg_c):
    assert rel(a, b) < 1e-10


@pytest.mark.gpu
def test_whole_model_gradient_at_micro_batch(dev):
  """TrainEngine.loss_and_grads_chunked on 256 trajectories of shared frames (frames shared across the micro-batch
  boundary) with micro_batch = 128 - the pair cell kernel runs - against RT.loss_and_grads on the GPU over chunks of
  16 trajectories, gradients summed with weight 16/256 (every loss is a batch mean) minus the weight-decay term the
  engine leaves to the optimizer.  The class decoder feeds one_hot(arg-max) forward, so the comparison is
  well-posed only if no arg-max of the reference lies within the engine's logit error of a tie: asserted as a
  precondition: every top-2 gap lies above MARGIN x max|logit|, and MARGIN is at least 4 x the measured logit error
  of the last micro-batch (a flip needs the errors of the two logits to differ by the gap, at most 2 x the error).
  The engine's ids of the last micro-batch must equal the reference's."""
  from multiverse_b200 import ops
  from multiverse_b200.train_engine import TrainEngine
  from multiverse_b200 import synthetic
  n, mb, chunk = 256, NS, 16
  cfg, rcfg = wm_configs(n, chunk)
  w = synthetic.make_weights(cfg, WM_SEED)
  f = shared_frame_feeds(cfg, n, FRAMES, WM_SEED)
  last = f["obs_scene"][n - mb:]
  assert np.intersect1d(f["obs_scene"][:n - mb], last).size > 0, "no frame shared across the micro-batch boundary"
  # ---- reference
  grads = {k: np.zeros(v.shape) for k, v in w.items()}
  losses = np.zeros(4)
  logits = [[], []]
  for lo in range(0, n, chunk):
    _, l, _, gr, lg = RT.loss_and_grads(rcfg, w, chunk_feeds(f, slice(lo, lo + chunk)), device=dev, return_logits=True)
    losses += np.array(l) * chunk / n
    for k in grads:
      grads[k] += gr[k] * chunk / n
    for i in range(2):
      logits[i].append(lg[i])
  for k in grads:
    if k.endswith("/W"):
      grads[k] -= cfg.wd * w[k]
  # ---- engine
  eng = TrainEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev, 2)
  feeds = dict(scene_feat=on(dev, f["scene_feat"]), obs_scene=on(dev, f["obs_scene"]))
  for k in ("grid_obs_labels", "grid_obs_regress", "grid_pred_labels", "grid_pred_regress"):
    feeds[k] = [on(dev, a) for a in f[k]]
  ops.cell_variants_seen(reset=True)
  got, _ = eng.loss_and_grads_chunked(feeds, mb)
  torch.cuda.synchronize()
  assert (2, True) in ops.cell_variants_seen(), "the P=2 pair cell kernel did not run: %s" % sorted(ops.cell_variants_seen())
  # ---- well-posedness of the arg-max feedback, and the ids / logits of the last micro-batch
  fwd_err = {}
  for i, (h, ww) in enumerate(cfg.scene_grids):
    ref = np.concatenate(logits[i]).reshape(n, T_PRED, h * ww)
    srt = np.sort(ref, -1)
    gap = (srt[..., -1] - srt[..., -2]).min() / np.abs(ref).max()
    mine = eng.last_logits[i].cpu().numpy().transpose(1, 0, 2)          # [Tp, mb, HW] -> [mb, Tp, HW]
    fwd_err[i] = rel(mine, ref[n - mb:])
    print("scale %d: smallest top-2 gap %.2e x max|logit|, logit error of the last micro-batch %.2e"
          % (i, gap, fwd_err[i]))
    assert fwd_err[i] * 4 < MARGIN, "the engine's logit error leaves no room for the arg-max margin"
    assert gap > MARGIN, "degenerate seed: a decoded arg-max lies within %.0e of a tie" % MARGIN
    ids = eng._store[("ids", i, mb)][0].cpu().numpy().T                  # [Tp, mb] -> [mb, Tp]
    assert np.array_equal(ids, ref[n - mb:].argmax(-1))
  got = got.cpu().numpy()
  assert np.abs(got - losses).max() < LTOL * np.abs(losses).max(), (got, losses)
  worst = {k: rel(eng.grads[k], grads[k]) for k in sorted(grads)}
  print("whole model, 256 trajectories in micro-batches of 128: losses %s, worst gradient errors %s"
        % (np.abs(got - losses).max() / np.abs(losses).max(), sorted(worst.items(), key=lambda kv: -kv[1])[:4]))
  bad = {k: v for k, v in worst.items() if v > GTOL}
  assert not bad, bad
