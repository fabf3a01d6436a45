# coding=utf-8
"""The reference's `pred_models` call surface on top of the H100 engine.

Mirrors code/pred_models.py of JunweiLiang/Multiverse: `get_model` (:19), `Model` (:32) with the
same placeholder / fetch attribute names, `get_feed_dict` (:1042-1194), `Trainer` (:1636) and
`Tester` (:1745) with the same `step` return conventions, so code/train.py, code/test.py,
code/multifuture_inference.py (which subclasses Model, :301) and code/pred_utils.py run with
their source unchanged once `multiverse_b200/dropin` is first on sys.path (it provides
`pred_models` and the `tensorflow`-named shim).  north_star's enc_cell / dec_cell / decode are
exposed as methods for unit testing.

Host code here only packs numpy feeds and sequences kernel launches (multiverse_b200.engine);
there is no graph and no CPU compute path.
"""
from __future__ import annotations

import os
import sys
import weakref

import numpy as np

_DROPIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")


def _shim():
  m = sys.modules.get("tensorflow")
  if m is not None:
    if not hasattr(m, "_GRAPH"):
      raise RuntimeError("a real `tensorflow` module is imported; multiverse_b200.pred_models "
                         "needs its shim (multiverse_b200/dropin) first on sys.path")
    return m
  if _DROPIN not in sys.path:
    sys.path.insert(0, _DROPIN)
  import tensorflow  # noqa: F401  (the shim)
  return sys.modules["tensorflow"]


tf = _shim()


class Handle(object):
  """Placeholder or fetch handle owned by a Model (what `sess.run` receives).  The owner is held weakly: the model
  holds its handles, and a strong back-reference would keep a dropped model - and the device memory of its engine -
  alive until Python's cycle collector happens to run."""

  def __init__(self, owner, kind, name, index=None):
    self._owner = weakref.ref(owner)
    self.kind, self.name, self.index = kind, name, index

  @property
  def owner(self):
    return self._owner()

  def __repr__(self):
    return "<%s %s%s>" % (self.kind, self.name, "" if self.index is None else "[%d]" % self.index)


def get_model(config, gpuid):
  """code/pred_models.py:19-30."""
  with tf.name_scope(config.modelname), tf.device("/gpu:%d" % gpuid):
    model = Model(config, "%s" % config.modelname)
  model.gpuid = gpuid
  return model


def _glorot(shape, rng):
  fan_in, fan_out = shape[0] * shape[1] * shape[2], shape[0] * shape[1] * shape[3]
  lim = np.sqrt(6.0 / (fan_in + fan_out))
  return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def _he(shape, rng):
  # tf.variance_scaling_initializer(scale=2.0): truncated normal, stddev sqrt(2/fan_in)/.8796
  fan_in = shape[0] * shape[1] * shape[2]
  std = np.sqrt(2.0 / fan_in) / 0.87962566103423978
  return (np.clip(rng.standard_normal(shape), -2, 2) * std).astype(np.float32)


class Model(object):
  """code/pred_models.py:32-121.  Reads the same `config.*` attributes."""

  def __init__(self, config, scope):
    self.scope = scope
    self.config = config
    self.gpuid = 0
    self._engine = None
    self._stale = True
    self._device_newer = False
    self._rng = np.random.default_rng(getattr(config, "seed", 0) or 0)
    self._own_vars = []

    self.global_step = self._var("global_step", (), dtype="int32", trainable=False)
    N = self.N = config.batch_size
    self.SH, self.SW, self.SC = config.scene_h, config.scene_w, config.scene_class
    self.beam_size = config.beam_size
    ph = lambda name, idx=None: Handle(self, "placeholder", name, idx)
    self.obs_length = ph("obs_length")
    self.pred_length = ph("pred_length")
    self.is_train = ph("is_train")
    self.obs_scene = ph("obs_scene")
    self.obs_scene_mask = ph("obs_scene_mask")
    self.scene_feat = ph("scene_feat")
    (self.grid_pred_labels, self.grid_pred_targets, self.grid_obs_labels, self.grid_obs_targets,
     self.grid_obs_regress, self.grid_pred_labels_T, self.grid_pred_regress) = [[] for _ in range(7)]
    for i, _ in enumerate(config.scene_grids):
      self.grid_pred_labels.append(ph("grid_pred_labels", i))
      self.grid_pred_targets.append(ph("grid_pred_targets", i))
      self.grid_obs_labels.append(ph("grid_obs_labels", i))
      self.grid_obs_targets.append(ph("grid_obs_targets", i))
      self.grid_obs_regress.append(ph("grid_obs_regress", i))
      self.grid_pred_labels_T.append(ph("grid_pred_labels_T", i))
      self.grid_pred_regress.append(ph("grid_pred_regress", i))
    # Extension placeholders (SURVEY.md section 8 row f-1): the observed trajectories [N,T,2] float64 and the cell
    # centres [h,w,2] float64 of a scale.  Fed INSTEAD of grid_obs_regress, they make the engine build the dense
    # per-cell offsets on the device (mvb_traj_to_grid, bit-identical to get_grid_input,
    # code/multifuture_inference.py:115-156 == code/preprocess.py:436-475): 128 bytes per trajectory on the PCIe
    # bus instead of 41 KB per trajectory and scale.  get_feed_dict uses them when the batch carries both.
    self.obs_traj = ph("obs_traj")
    self.grid_centers = [ph("grid_centers", i) for i, _ in enumerate(config.scene_grids)]
    # Training batches also feed the future trajectories [N,Tp,2] float64 and int32 label cells in grid_pred_labels_T,
    # instead of grid_obs_regress, grid_pred_regress and (--use_soft_grid_class) the soft label maps: the training
    # step's kernels compute the offsets, regression targets and label maps where they read them.
    self.pred_traj = ph("pred_traj")
    # SimAug's Model (SimAug/code/pred_models.py:225-267): the other camera views of every sample
    if getattr(config, "multiview_train", False):
      self.obs_scene_extra = ph("obs_scene_extra")
      self.grid_obs_labels_extra = [ph("grid_obs_labels_extra", i) for i, _ in enumerate(config.scene_grids)]
      self.grid_pred_labels_T_extra = [ph("grid_pred_labels_T_extra", i) for i, _ in enumerate(config.scene_grids)]
      self.grid_pred_regress_extra = [ph("grid_pred_regress_extra", i) for i, _ in enumerate(config.scene_grids)]
      self.grid_obs_regress_extra = [ph("grid_obs_regress_extra", i) for i, _ in enumerate(config.scene_grids)]
    self.beam_outputs = None
    self.loss = None
    self.build_forward()
    if config.is_train:
      self.build_loss()

  # ---------------------------------------------------------------- variables
  def _var(self, name, shape, dtype="float32", init=None, trainable=True):
    fn = None
    if init is not None:
      fn = lambda shp, init=init, rng=self._rng: init(tuple(shp), rng)     # no reference back to the model
    v = tf.Variable(name, shape, dtype=dtype, initializer=fn, trainable=trainable, owner=self)
    tf._GRAPH.add(v)
    self._own_vars.append(v)
    return v

  def _var_names(self):
    return {v.name.split(":")[0] for v in self._own_vars}

  def _variables_changed(self):
    self._stale = True

  def _sync_to_host(self):
    """Pull trained parameters back into the host copies (Saver.save, Variable.eval)."""
    eng = self._engine
    if eng is not None and getattr(eng, "params", None) is not None and self._device_newer:
      for v in self._own_vars:
        key = v.name.split(":")[0]
        if key in eng.params:
          v.value = eng.params[key].cpu().numpy()
      self._device_newer = False

  def weights(self):
    return {v.name.split(":")[0]: v.value for v in self._own_vars if v.dtype == "float32"}

  # ---------------------------------------------------------------- graph
  def build_forward(self):
    """code/pred_models.py:123-308: declares the variables under the reference's names and the
    fetch handles; the computation itself is ConvRNNEngine.forward."""
    cfg = self.config
    zeros = lambda shp, rng: np.zeros(shp, dtype=np.float32)
    cin = cfg.scene_class
    for i in range(len(cfg.scene_grid_strides) if cfg.use_scene_enc else 0):
      self._var("person_pred/scene_conv%d/W" % (i + 1), (3, 3, cin, cfg.scene_conv_dim), init=_he)
      self._var("person_pred/scene_conv%d/b" % (i + 1), (cfg.scene_conv_dim,), init=zeros)
      cin = cfg.scene_conv_dim
    ch, e, k = cfg.enc_hidden_size, cfg.emb_size, cfg.convlstm_kernel
    self.grid_pred_decoded, self.grid_pred_reg_decoded = [], []
    p = "person_pred/"
    for i, _ in enumerate(cfg.scene_grids):
      if not cfg.use_grids[i]:
        self.grid_pred_decoded.append([])            # :170-171
        self.grid_pred_reg_decoded.append([])
        continue
      cell = lambda name, cx: (self._var(name + "/kernel", (k, k, cx + ch, 4 * ch), init=_glorot),
                               self._var(name + "/biases", (4 * ch,), init=zeros))
      if not cfg.use_scene_enc and p + "grid_emb/W" not in self._var_names():
        # the class encoder's embedding of one_hot(label): created under the top scope with AUTO_REUSE (:221-225,
        # :1339), so every scale shares it
        self._var(p + "grid_emb/W", (3, 3, 1, e), init=_he)
        self._var(p + "grid_emb/b", (e,), init=zeros)
      cell(p + "encoder_grid_class_%d/enc_grid_%d" % (i, i), cfg.scene_conv_dim if cfg.use_scene_enc else e)
      cell(p + "encoder_grid_reg_%d/enc_grid_regress_%d" % (i, i), 2)
      for kind, cname, pdim in (("class", "dec_grid_%d" % i, 1), ("reg", "dec_grid_reg_%d" % i, 2)):
        d = p + "decoder_grid_%s_%d/decoder_rnn/" % (kind, i)
        cell(d + cname, e)
        self._var(d + "grid_emb/W", (3, 3, pdim, e), init=_he)
        self._var(d + "grid_emb/b", (e,), init=zeros)
        self._var(p + "hidden2grid_decoder_grid_%s_%d/out_dec_grid/W" % (kind, i), (3, 3, ch, pdim), init=_he)
      self.grid_pred_decoded.append(Handle(self, "fetch", "grid_pred_decoded", i))
      self.grid_pred_reg_decoded.append(Handle(self, "fetch", "grid_pred_reg_decoded", i))
    if cfg.use_beam_search:
      assert not cfg.is_train                        # :261-262
      assert sum(cfg.use_grids) == 1, "only one scale test at a time"
      self.beam_outputs = [Handle(self, "fetch", "beam_outputs", j) for j in range(3)]   # :276

  def build_loss(self):
    """code/pred_models.py:961-1040 (handles; evaluated by the training path)."""
    self.pred_grid_loss = []
    for i, _ in enumerate(self.config.scene_grids):
      if self.config.use_grids[i]:
        self.pred_grid_loss.extend([Handle(self, "fetch", "classification_loss", i),
                                    Handle(self, "fetch", "regression_loss", i)])
    self.wd_loss = Handle(self, "fetch", "wd_loss")
    self.loss = Handle(self, "fetch", "loss")

  # ---------------------------------------------------------------- feeds
  def get_feed_dict(self, batch, is_train=False, train_traj=False):
    """code/pred_models.py:1042-1194, vectorised.  `batch` is a pred_utils.Dataset whose
    `.data` holds obs_grid_class / pred_grid_class [num_scale,T], obs/pred_grid_target_all_<j>
    [T,h,w,2], batch_scene_feat [F,SH,SW,SC] and batch_obs_scene [[idx],...].
    train_traj (Trainer.step): a training batch that carries its trajectories and grid centres is fed as those
    (_train_traj_feeds) - no dense offset, target or soft label map is built; without it a training feed dict is
    the reference's."""
    cfg = self.config
    N, T_in, T_pred = self.N, cfg.obs_len, cfg.pred_len
    data = batch.data
    fd = {self.obs_length: np.full((N,), T_in, dtype="int32"),
          self.pred_length: np.full((N,), T_pred, dtype="int32"),
          self.is_train: is_train}
    n_have = len(data["obs_grid_class"])
    traj = self._train_traj_feeds(batch, n_have) if is_train and train_traj else None
    for j, (h, w) in enumerate(cfg.scene_grids):
      labels = np.zeros((N, T_in), dtype="int32")
      if n_have:
        labels[:n_have] = np.stack([np.asarray(a)[j, :] for a in data["obs_grid_class"]])
      fd[self.grid_obs_labels[j]] = labels           # :1186-1191 (every scale, used or not)
      if not cfg.use_grids[j]:
        continue
      if traj is not None:
        fd[self.grid_pred_labels_T[j]] = np.stack([np.asarray(a)[j, :] for a in data["pred_grid_class"]]).astype("int32")
        fd[self.grid_centers[j]] = traj[2][j]
        continue
      obs_reg = np.zeros((N, T_in, h, w, 2), dtype="float32")
      obs_reg[:n_have] = np.stack(data["obs_grid_target_all_%d" % j])
      fd[self.grid_obs_regress[j]] = obs_reg
      if is_train or cfg.use_gt_grid:
        pred_reg = np.zeros((N, T_pred, h, w, 2), dtype="float32")
        pred_reg[:n_have] = np.stack(data["pred_grid_target_all_%d" % j])
        cls = np.stack([np.asarray(a)[j, :] for a in data["pred_grid_class"]])
        if cfg.use_soft_grid_class:
          pred_lab = np.zeros((N, T_pred, h, w, 1), dtype="float32")
          pred_lab[:n_have] = _soft_labels(cls, h, w, cfg.soft_grid)
        else:
          pred_lab = np.zeros((N, T_pred), dtype="float32")
          pred_lab[:n_have] = cls
        fd[self.grid_pred_regress[j]] = pred_reg
        fd[self.grid_pred_labels_T[j]] = pred_lab
      else:
        fd[self.grid_pred_regress[j]] = np.zeros((N, T_pred, h, w, 2), dtype="float32")
        fd[self.grid_pred_labels_T[j]] = (np.zeros((N, T_pred, h, w, 1), dtype="int32")
                                          if cfg.use_soft_grid_class else
                                          np.zeros((N, T_pred), dtype="int32"))
    obs_scene = np.zeros((N, T_in), dtype="int32")
    mask = np.zeros((N, T_in), dtype="bool")
    for i, row in enumerate(data["batch_obs_scene"]):
      idx = np.asarray(row).reshape(len(row), -1)[:, 0]
      obs_scene[i, :len(idx)] = idx
      mask[i, :len(idx)] = True
    fd[self.obs_scene] = obs_scene
    fd[self.obs_scene_mask] = mask
    fd[self.scene_feat] = data["batch_scene_feat"]
    if is_train and getattr(cfg, "multiview_train", False):
      # SimAug/code/pred_models.py:1517-1541, :1553-1555: the M other camera views of every sample
      M = cfg.multiview_max_num
      for j, (h, w) in enumerate(cfg.scene_grids):
        if not cfg.use_grids[j]:
          continue
        obs_lab = np.zeros((N, M, T_in), dtype="int32")
        pred_lab = np.zeros((N, M, T_pred), dtype="float32")
        obs_reg = np.zeros((N, M, T_in, h, w, 2), dtype="float32")
        pred_reg = np.zeros((N, M, T_pred, h, w, 2), dtype="float32")
        for i, ex in enumerate(data["extra"]):
          for k in range(len(ex["obs_grid_class"])):
            obs_lab[i, k] = np.asarray(ex["obs_grid_class"][k])[j, :]
            pred_lab[i, k] = np.asarray(ex["pred_grid_class"][k])[j, :]
            obs_reg[i, k] = ex["obs_grid_target_all_%d" % j][k]
            pred_reg[i, k] = ex["pred_grid_target_all_%d" % j][k]
        fd[self.grid_obs_labels_extra[j]] = obs_lab
        fd[self.grid_pred_labels_T_extra[j]] = pred_lab
        fd[self.grid_pred_regress_extra[j]] = pred_reg
        fd[self.grid_obs_regress_extra[j]] = obs_reg
      fd[self.obs_scene_extra] = np.squeeze(data["batch_extra_obs_scene"])
    if traj is not None:
      fd[self.obs_traj], fd[self.pred_traj] = traj[0], traj[1]
    self._compact_grid_feeds(fd, batch, n_have, is_train)
    return fd

  def _train_traj_feeds(self, batch, n_have):
    """Row f-1 for training: (obs_traj [N,T,2], pred_traj [N,Tp,2], {scale: centres [h,w,2]}, all float64) when a
    training batch can be fed as trajectories, else None and the batch keeps the dense feeds.  That needs a full batch
    (pred_utils pads the last one with its last item; padded rows of a dense feed are zeros no trajectory gives),
    data["obs_traj"] / data["pred_traj"] and shared["grid_center_<j>"] of every used scale (pred_utils.read_data puts
    them there), label cells that index the grid under --use_soft_grid_class (as _soft_labels' numpy indexing needs),
    and dense offsets that agree with float32(trajectory - centre) on 32 sampled cells per scale, observed and future,
    as in _compact_grid_feeds.  SimAug's adversarial and multiview training keep the dense feeds."""
    cfg = self.config
    N, T, Tp = self.N, cfg.obs_len, cfg.pred_len
    if not getattr(cfg, "device_grid_feeds", True) or n_have != N:
      return None
    if getattr(cfg, "multiview_train", False) or getattr(cfg, "adv_train", False):
      return None
    data, shared = batch.data, getattr(batch, "shared", None)
    if shared is None or "obs_traj" not in data or "pred_traj" not in data:
      return None
    soft = bool(getattr(cfg, "use_soft_grid_class", False))
    if soft and getattr(cfg, "soft_grid", None) not in range(1, 8):
      return None
    try:
      obs = np.stack([np.asarray(t, dtype=np.float64) for t in data["obs_traj"]])[:, :T]
      pred = np.stack([np.asarray(t, dtype=np.float64) for t in data["pred_traj"]])[:, :Tp]
    except Exception:
      return None
    if obs.shape != (N, T, 2) or pred.shape != (N, Tp, 2):
      return None
    rng = np.random.default_rng(0)
    centers = {}
    for j, (h, w) in enumerate(cfg.scene_grids):
      if not cfg.use_grids[j]:
        continue
      c = shared.get("grid_center_%d" % j)
      if c is None or np.shape(c) != (h, w, 2):
        return None
      centers[j] = np.ascontiguousarray(c, dtype=np.float64)
      cls = np.stack([np.asarray(a)[j, :] for a in data["pred_grid_class"]])
      if soft and not ((cls >= -h * w) & (cls < h * w)).all():
        return None
      for key, tr, steps in (("obs_grid_target_all_%d" % j, obs, T), ("pred_grid_target_all_%d" % j, pred, Tp)):
        ii, tt = rng.integers(0, N, 32), rng.integers(0, steps, 32)
        yy, xx = rng.integers(0, h, 32), rng.integers(0, w, 32)
        try:
          dense = np.array([np.asarray(data[key][i][t, y, x], dtype=np.float32) for i, t, y, x in zip(ii, tt, yy, xx)])
        except Exception:
          return None
        if not np.array_equal(dense, (tr[ii, tt] - centers[j][yy, xx]).astype(np.float32)):
          return None
    return obs, pred, centers

  def _compact_grid_feeds(self, fd, batch, n_have, is_train):
    """Row f-1: when the batch carries the observed trajectories and the grid centres the dense offsets were
    computed from (pred_utils.read_data puts both there: data["obs_traj"], shared["grid_center_<j>"]), feed those
    instead of the dense [N,T,h,w,2] arrays; the engine regenerates the arrays on the device.  Guarded by a
    sampled consistency check - dense == float32(trajectory - centre) on 32 random cells per scale - so a batch
    whose dense targets were edited independently keeps the dense path.  config.device_grid_feeds=False turns it
    off.  Training batches are decided before any dense array is built (_train_traj_feeds)."""
    cfg = self.config
    if is_train or not getattr(cfg, "device_grid_feeds", True) or not n_have:
      return
    data, shared = batch.data, getattr(batch, "shared", None)
    if shared is None or "obs_traj" not in data:
      return
    used = [j for j in range(len(cfg.scene_grids)) if cfg.use_grids[j]]
    if any(("grid_center_%d" % j) not in shared for j in used):
      return
    traj = np.zeros((self.N, cfg.obs_len, 2), dtype=np.float64)
    try:
      traj[:n_have] = np.stack([np.asarray(t, dtype=np.float64) for t in data["obs_traj"]])[:, :cfg.obs_len]
    except Exception:
      return
    rng = np.random.default_rng(0)
    for j in used:
      h, w = cfg.scene_grids[j]
      centers = np.asarray(shared["grid_center_%d" % j], dtype=np.float64)
      if centers.shape != (h, w, 2):
        return
      dense = fd[self.grid_obs_regress[j]]
      ii, tt = rng.integers(0, n_have, 32), rng.integers(0, cfg.obs_len, 32)
      yy, xx = rng.integers(0, h, 32), rng.integers(0, w, 32)
      want = (traj[ii, tt] - centers[yy, xx]).astype(np.float32)
      if not np.array_equal(dense[ii, tt, yy, xx], want):
        return
    for j in used:
      del fd[self.grid_obs_regress[j]]
      fd[self.grid_centers[j]] = np.asarray(shared["grid_center_%d" % j], dtype=np.float64)
    fd[self.obs_traj] = traj

  # ---------------------------------------------------------------- execution
  def _ensure_engine(self):
    import torch
    from . import build, engine
    if self._engine is None:
      build.build()
      dev = torch.device("cuda", self.gpuid)
      torch.cuda.set_device(dev)
      w = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in self.weights().items()}
      if self.config.is_train:
        from . import train_engine
        self._engine = train_engine.TrainEngine(_engine_config(self.config), w, dev)
      else:
        self._engine = engine.ConvRNNEngine(_engine_config(self.config), w, dev)
      self._stale = False
    elif self._stale:
      w = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in self.weights().items()}
      if getattr(self._engine, "params", None) is not None:      # restored checkpoint while training
        for k, v in w.items():
          self._engine.params[k].copy_(v)
        self._engine._repack()
      else:
        self._engine.set_weights(w)
      self._stale = False
    return self._engine

  def _device_feeds(self, feed, train_traj=False):
    """The feeds of the engine on its device.  train_traj: a training feed of trajectories (obs_traj, pred_traj,
    grid_centers): they go to the device as feeds["traj"] (TrainEngine.loss_and_grads) and no dense offset is built."""
    import torch
    eng = self._ensure_engine()
    dev = eng.device
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev, non_blocking=True)
    cfg = self.config
    scene = up(feed[self.scene_feat], np.float32)
    if getattr(cfg, "norm_input", False):      # SimAug/code/pred_models.py:282-284: features to [-1, 1]
      scene = scene * 2.0 - 1.0
    out = dict(scene_feat=scene,
               obs_scene=up(feed[self.obs_scene], np.int32),
               grid_obs_labels=[None] * len(cfg.scene_grids),
               grid_obs_regress=[None] * len(cfg.scene_grids))
    regress = None
    if train_traj:
      out["traj"] = dict(obs=up(feed[self.obs_traj], np.float64), pred=up(feed[self.pred_traj], np.float64),
                         centers=[up(feed[self.grid_centers[i]], np.float64) if cfg.use_grids[i] else None
                                  for i in range(len(cfg.scene_grids))],
                         soft_grid=int(cfg.soft_grid) if getattr(cfg, "use_soft_grid_class", False) else 0)
    elif self.obs_traj in feed:     # row f-1: dense offsets built on the device from the trajectories
      centers = [feed.get(self.grid_centers[i]) for i in range(len(cfg.scene_grids))]
      _, regress = eng.grid_feeds_from_traj(np.asarray(feed[self.obs_traj], dtype=np.float64), centers=centers)
    for i in range(len(cfg.scene_grids)):
      if cfg.use_grids[i]:
        out["grid_obs_labels"][i] = up(feed[self.grid_obs_labels[i]], np.int32)
        if self.grid_obs_regress[i] in feed:
          out["grid_obs_regress"][i] = up(feed[self.grid_obs_regress[i]], np.float32)
        elif regress is not None:
          out["grid_obs_regress"][i] = regress[i]
        elif not train_traj:
          raise KeyError("feed neither grid_obs_regress[%d] nor obs_traj + grid_centers[%d]" % (i, i))
    return out

  def _run(self, handles, feed):
    """What `sess.run(fetches, feed_dict)` does for this model: one engine forward per call,
    numpy arrays out in the reference's shapes."""
    need_fwd = any(isinstance(h, Handle) and h.kind == "fetch" and
                   h.name in ("grid_pred_decoded", "grid_pred_reg_decoded", "beam_outputs")
                   for h in handles)
    train_names = ("loss", "wd_loss", "classification_loss", "regression_loss", "train_op")
    tr = None
    if any(isinstance(h, Handle) and h.name in train_names for h in handles):
      tr = self._train_step(feed, apply=any(isinstance(h, Handle) and h.name == "train_op" for h in handles))
    fwd_names = ("grid_pred_decoded", "grid_pred_reg_decoded", "beam_outputs")
    host = self._engine_forward(feed, {(h.name, h.index) for h in handles if isinstance(h, Handle)
                                        and h.kind == "fetch" and h.name in fwd_names}) if need_fwd else None
    out = []
    for h in handles:
      if isinstance(h, tf.Variable):
        out.append(h.eval())
      elif h.name in train_names:
        out.append(tr[h.name] if h.index is None else tr[h.name][h.index])
      elif h.kind == "fetch":
        out.append(host[(h.name, h.index)])
      else:
        raise ValueError("cannot fetch %r" % (h,))
    return out

  def _engine_forward(self, feed, wanted):
    """One engine forward; every requested fetch is copied to pinned host memory on a side stream as soon as the
    engine reports it complete (the beam logits, 90 % of the fetched bytes, travel while the regression branch
    still computes), and comes back as a numpy array that owns its pinned block."""
    import torch
    eng = self._ensure_engine()
    dev = eng.device
    if getattr(self, "_copy_stream", None) is None:
      self._copy_stream = torch.cuda.Stream(device=dev)
    side, host, busy = self._copy_stream, {}, set()

    def on_output(name, index, t):
      if (name, index) not in wanted or not torch.is_tensor(t):
        return
      t = t.contiguous()
      side.wait_event(torch.cuda.current_stream(dev).record_event())
      with torch.cuda.stream(side):
        dst = self._pinned_block(tuple(t.shape), t.dtype, busy)
        dst.copy_(t, non_blocking=True)
      t.record_stream(side)
      host[(name, index)] = dst

    with torch.cuda.device(dev):
      feeds, tp = self._device_feeds(feed), self._fed_pred_len(feed)
      if self._launch_bound(feeds):
        # small batch: the host cannot launch ~10^3 kernels as fast as the GPU runs them -> graph replay
        # (captured in segments cut after every class branch: the fetches of a finished branch travel while the next
        # segment runs; the static outputs are consumed before the next replay)
        eng.forward_graph(feeds, pred_len=tp, on_output=on_output)
      else:
        eng.forward(feeds, pred_len=tp, on_output=on_output)
      side.synchronize()
    res = {k: v.numpy() for k, v in host.items()}
    for k in wanted:
      if k not in res:
        if k[0] in ("grid_pred_decoded", "grid_pred_reg_decoded"):
          res[k] = []                                   # unused scale (:170-171)
        else:
          raise ValueError("fetch %s[%s] is not produced by this configuration" % k)
    return res

  def _pinned_block(self, shape, dtype, busy, keep=4):
    """A pinned host tensor for one fetch.  Blocks are kept per (shape, dtype) and handed out again once the numpy
    array that wrapped them (and every view of it) is gone (`busy`: ids of the blocks already handed out during
    the current call, which have no array yet): a fresh 40 MB pinned allocation per Session.run costs tens of ms of
    host time, which torch's own host allocator would pay on every call here."""
    import torch
    use_count = getattr(torch._C, "_storage_Use_Count", None)
    if use_count is None:                   # no way to tell whether a block is still referenced: do not pool
      return torch.empty(shape, dtype=dtype, pin_memory=True)
    if getattr(self, "_pinned", None) is None:
      self._pinned = {}
    blocks = self._pinned.setdefault((shape, dtype), [])
    for t, idle in blocks:
      # Tensor.numpy() wraps an alias of the tensor: the storage's use count is back at its idle value once the
      # array and every view / from_numpy of it are gone
      if id(t) not in busy and use_count(t.untyped_storage()._cdata) <= idle:
        busy.add(id(t))
        return t
    t = torch.empty(shape, dtype=dtype, pin_memory=True)
    busy.add(id(t))
    if len(blocks) < keep:                  # callers that hold many results get unpooled blocks beyond `keep`
      blocks.append((t, use_count(t.untyped_storage()._cdata)))
    return t

  def _launch_bound(self, feeds):
    """CUDA-graph replay (ConvRNNEngine.forward_graph) when a forward is host-launch bound: fewer than
    MVB_GRAPH_MAX_ROWS (default 2000) sample rows x beams; MVB_CUDA_GRAPH=0/1 forces eager / graph."""
    mode = os.environ.get("MVB_CUDA_GRAPH", "")
    if mode in ("0", "1"):
      return mode == "1"
    rows = int(feeds["obs_scene"].shape[0]) * (self.config.beam_size if self.config.use_beam_search else 1)
    return rows <= int(os.environ.get("MVB_GRAPH_MAX_ROWS", "2000"))

  def _fed_pred_len(self, feed):
    """Rollout length = the fed pred_length (raw_rnn's stop condition, :347/:520)."""
    pl = feed.get(self.pred_length)
    if pl is None:
      return self.config.pred_len
    pl = np.asarray(pl).reshape(-1)
    if pl.size == 0:
      return self.config.pred_len
    if not (pl == pl[0]).all():
      raise NotImplementedError("per-row pred_length is not implemented (every reference feed uses one value)")
    return int(pl[0])

  def learning_rate(self, step):
    """Trainer's schedule (code/pred_models.py:1645-1665): init_lr, optionally cosine or staircase
    exponential decay every num_epoch_per_decay epochs; times emb_lr (:1672)."""
    import math
    cfg = self.config
    lr = cfg.init_lr
    if getattr(cfg, "use_cosine_lr", False):
      max_steps = int(cfg.train_num_examples / cfg.batch_size * cfg.num_epochs)
      lr = cfg.init_lr * 0.5 * (1 + math.cos(math.pi * min(step, max_steps) / max(max_steps, 1)))
    elif getattr(cfg, "learning_rate_decay", None) is not None:
      decay_steps = int(cfg.train_num_examples / cfg.batch_size * cfg.num_epoch_per_decay)
      lr = cfg.init_lr * cfg.learning_rate_decay ** (step // max(decay_steps, 1))
    return lr * getattr(cfg, "emb_lr", 1.0)

  def _train_step(self, feed, apply=True):
    """What sess.run([loss, train_op, wd_loss, pred_grid_loss]) does (Trainer.step, :1719-1742)."""
    import torch
    cfg = self.config
    if getattr(cfg, "optimizer", "adadelta") not in ("adadelta", "momentum", "adam", "rmsprop"):
      raise Exception("Optimizer not implemented")            # code/pred_models.py:1681
    soft = bool(getattr(cfg, "use_soft_grid_class", False))
    options = [name for name, on in (("use_soft_grid_class", soft),
                                     ("mask_grid_regression", getattr(cfg, "mask_grid_regression", False)),
                                     ("no train_w_onehot", not getattr(cfg, "train_w_onehot", True))) if on]
    augment = [k for k in ("adv_train", "multiview_train") if getattr(cfg, k, False)]
    if options and augment:
      raise NotImplementedError("%s combined with SimAug's --%s is not implemented"
                                % (" / ".join(options), " / --".join(augment)))
    if soft and any(hasattr(cfg, k) for k in ("adv_train", "multiview_train")):
      raise NotImplementedError("SimAug's model ignores --use_soft_grid_class; this combination is not implemented")
    eng = self._ensure_engine()
    dev = eng.device
    train_traj = self.pred_traj in feed          # get_feed_dict's trajectory feeds (_train_traj_feeds)
    feeds = self._device_feeds(feed, train_traj)
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev, non_blocking=True)
    feeds["grid_pred_labels"] = [None] * len(cfg.scene_grids)
    feeds["grid_pred_regress"] = [None] * len(cfg.scene_grids)
    for i in range(len(cfg.scene_grids)):
      if cfg.use_grids[i]:
        feeds["grid_pred_labels"][i] = up(feed[self.grid_pred_labels_T[i]],
                                          np.float32 if soft and not train_traj else np.int32)
        if not train_traj:
          feeds["grid_pred_regress"][i] = up(feed[self.grid_pred_regress[i]], np.float32)
    feeds = self._simaug_feeds(eng, feeds, feed)
    step = int(self.global_step.value)
    if apply:
      # under torchrun (an initialised NCCL process group) the drop-in train.py is data parallel: every rank feeds its
      # own batches and the gradients are all-reduced (SURVEY.md section 8e); a single process trains alone
      import torch.distributed as dist
      group = dist if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None
      losses, wd = eng.train_step(feeds, self.learning_rate(step), group)
      self.global_step.value = np.asarray(step + 1, dtype="int32")
      self._device_newer = True
    else:
      losses, wd = eng.loss_and_grads(feeds)
    losses = losses.cpu().numpy()
    wd = float(wd)
    cls = {}
    reg = {}
    used = [i for i in range(len(cfg.scene_grids)) if cfg.use_grids[i]]
    for j, i in enumerate(used):
      cls[i], reg[i] = losses[2 * j], losses[2 * j + 1]
    return dict(loss=np.float32(losses.sum() + wd), wd_loss=np.float32(wd), train_op=None,
                classification_loss=cls, regression_loss=reg)

  def _simaug_feeds(self, eng, feeds, feed):
    """The training-time input augmentations of SimAug's Model (SimAug/code/pred_models.py:286-325), applied to the
    scene semantics before the training tower runs: `adv_train` (white_box_attack, :289-301), `multiview_train`
    (multiview_augmentation, :304-310) and `standard_aug` (uniform pixel jitter, :312-325).  Like the reference they
    work on one private frame per (sample, step) row: the batch's unique frames are expanded first."""
    import torch
    cfg = self.config
    adv = getattr(cfg, "adv_train", False)
    multi = getattr(cfg, "multiview_train", False)
    jitter = getattr(cfg, "standard_aug", False)
    if not (adv or multi or jitter):
      return feeds
    from . import simaug
    if getattr(self, "_aug_rng", None) is None:
      self._aug_rng = np.random.default_rng(getattr(cfg, "seed", None))
    dev = eng.device
    n, t_obs = feeds["obs_scene"].shape
    rows = dict(feeds)
    rows["scene_feat"] = feeds["scene_feat"].float()[feeds["obs_scene"].long()].reshape(
        (n * t_obs,) + tuple(feeds["scene_feat"].shape[1:])).contiguous()
    rows["obs_scene"] = torch.arange(n * t_obs, device=dev, dtype=torch.int32).reshape(n, t_obs)
    if adv or multi:
      assert sum(cfg.use_grids) == 1, "only one scale for adv / multiview train"        # :290, :305
      i = list(cfg.use_grids).index(True)
    if adv:
      label = np.asarray(feed[self.grid_pred_labels_T[i]]).astype(np.int64)
      rows["scene_feat"], _ = simaug.white_box_attack(eng, rows, label, cfg, self._aug_rng,
                                                      norm_feat=getattr(cfg, "norm_feat", False))
    elif multi:
      src = dict(feeds)       # the unique frames: obs_scene_extra indexes them
      src["grid_pred_labels_extra"] = [None if not cfg.use_grids[j] else
                                       np.asarray(feed[self.grid_pred_labels_T_extra[j]]).astype(np.int32)
                                       for j in range(len(cfg.scene_grids))]
      src["obs_scene_extra"] = np.asarray(feed[self.obs_scene_extra]).astype(np.int32)
      rows["scene_feat"], self.multiview_info = simaug.multiview_augmentation(eng, src, cfg, self._aug_rng)
      if int(cfg.multiview_exp) == 3:
        # the label side of experiment 3 (SimAug/code/pred_models.py:616-638, :1371-1405): the observed class maps
        # and the loss labels are mixed with those of the selected other view, weight beta; the per-sample focal
        # weights multiply the classification loss under --double_weighting
        info = self.multiview_info
        sel = info["selected_extra_indices"].long()
        pick = lambda a: torch.as_tensor(np.asarray(a), device=dev).to(torch.int32)[torch.arange(n, device=dev), sel]
        ns = len(cfg.scene_grids)
        rows["mixup"] = dict(
            beta=float(info["beta_weight"]),
            obs_labels2=[pick(feed[self.grid_obs_labels_extra[j]]) if cfg.use_grids[j] else None for j in range(ns)],
            pred_labels2=[pick(feed[self.grid_pred_labels_T_extra[j]]) if cfg.use_grids[j] else None for j in range(ns)],
            focal=info["focal_loss_weight"] if getattr(cfg, "double_weighting", False) else None)
    if jitter:
      eps = float(cfg.adv_epsilon)
      noise = self._aug_rng.uniform(-eps, eps, size=tuple(rows["scene_feat"].shape)).astype(np.float32)
      rows["scene_feat"] = rows["scene_feat"] + torch.from_numpy(noise).to(dev)
    return rows

  # ---------------------------------------------------------------- unit-test surface
  def enc_cell(self, x, state, scale=0, kind="class"):
    """One encoder ConvLSTM step (enc_cell_obs_grid / enc_cell_obs_grid_reg, :189-202) on NHWC
    numpy inputs: x [N,h,w,Cx], state=(c,h) [N,h,w,256] -> (c', h')."""
    return self._cell_step("enc_" + kind, x, state, scale)

  def dec_cell(self, x, state, scale=0, kind="class"):
    """One decoder ConvLSTM step (dec_cell_grid / dec_cell_grid_reg, :236-249); x is the
    embedded input [N,h,w,emb_size]."""
    return self._cell_step("dec_" + kind, x, state, scale)

  def _cell_step(self, which, x, state, scale):
    import torch
    from . import ops
    eng = self._ensure_engine()
    dev = eng.device
    pk = getattr(eng.scales[scale], which)
    n, h, w, _ = x.shape
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    xh = ops.alloc_xh(n, h, w, pk.cpad, pk.planes, dev)
    ops.nhwc_to_planes(up(x), xh, 0, h, w, comp=pk.comp)
    ops.nhwc_to_planes(up(state[1]), xh, pk.cxp, h, w)
    c_in = ops.alloc_state(n, h, w, dev)
    ops.nhwc_to_halo(up(state[0]), c_in, h, w)
    c_out, h_out = ops.alloc_state(n, h, w, dev), ops.alloc_state(n, h, w, dev)
    ops.cell_fwd(xh, pk, c_in, c_out, h_out, None, h, w, n)
    co = torch.empty((n, h, w, 256), device=dev)
    ho = torch.empty((n, h, w, 256), device=dev)
    ops.halo_to_nhwc(c_out, co, h, w)
    ops.halo_to_nhwc(h_out, ho, h, w)
    return co.cpu().numpy(), ho.cpu().numpy()

  def decode(self, feed):
    """Whole rollout for a feed dict (grid_decoder / grid_decoder_beam_search, :311-806):
    returns (grid_pred_decoded, grid_pred_reg_decoded, beam_outputs) as numpy."""
    ns = len(self.config.scene_grids)
    wanted = {(nm, i) for nm in ("grid_pred_decoded", "grid_pred_reg_decoded") for i in range(ns)}
    if self.config.use_beam_search:
      wanted |= {("beam_outputs", j) for j in range(3)}
    res = self._engine_forward(feed, wanted)
    return ([res[("grid_pred_decoded", i)] for i in range(ns)], [res[("grid_pred_reg_decoded", i)] for i in range(ns)],
            [res[("beam_outputs", j)] for j in range(3)] if self.config.use_beam_search else None)


def _engine_config(config):
  """The subset of `config` the engine reads, with the activation token normalised."""
  from types import SimpleNamespace
  act = config.activation_func
  name = act if isinstance(act, str) else getattr(act, "__name__", "tanh")
  if name != "tanh":
    raise NotImplementedError("activation %r: the kernels implement tanh (every published config)" % name)
  keys = ("batch_size scene_h scene_w scene_class scene_conv_dim scene_conv_kernel scene_grid_strides "
          "scene_grids use_grids enc_hidden_size dec_hidden_size emb_size convlstm_kernel use_scene_enc "
          "use_gnn use_beam_search beam_size diverse_beam diverse_gamma fix_num_timestep "
          "pred_len").split()
  d = {k: getattr(config, k) for k in keys}
  if not (d["emb_size"] % 8 == 0 and 8 <= d["emb_size"] <= 256):
    raise NotImplementedError("--emb_size %r: the kernels take a multiple of 8 from 8 to 256 (the reference's default "
                              "is 128, the published commands pass 32)" % (d["emb_size"],))
  d["obs_len"] = getattr(config, "obs_len", None)    # multifuture_inference.py's Namespace has none (:419-452)
  d["activation_func"] = "tanh"
  for k, default in (("grid_loss_weight", 1.0), ("grid_reg_loss_weight", 0.1), ("wd", 0.0),
                     ("clip_gradient_norm", None), ("is_train", False), ("optimizer", "adadelta"),
                     ("mask_grid_regression", False), ("train_w_onehot", True)):
    d[k] = getattr(config, k, default)
  # SimAug's pred_models.py differs from Multiverse's in one line of gnn_edge (scene features only under
  # tile_to_beam): a config that carries SimAug's flags selects that variant unless it says otherwise
  simaug = any(hasattr(config, k) for k in ("multiview_train", "adv_train"))
  d["gnn_scene_in_greedy"] = bool(getattr(config, "gnn_scene_in_greedy", not simaug))
  aug = [k for k in ("adv_train", "multiview_train", "standard_aug", "norm_input") if getattr(config, k, False)]
  if not config.use_scene_enc and aug:
    raise NotImplementedError("--%s without --use_scene_enc: SimAug's model always encodes the scene, and its "
                              "augmentations act on the scene input" % " / --".join(aug))
  for flag in ("use_single_decoder", "use_teacher_forcing"):
    if getattr(config, flag, False):
      raise NotImplementedError("--%s is not implemented (no published config uses it)" % flag)
  if getattr(config, "keep_prob", 1.0) != 1.0 and getattr(config, "is_train", False):
    raise NotImplementedError("dropout (keep_prob < 1) is not implemented; every published config uses 1.0")
  return SimpleNamespace(**d)


def _soft_labels(cls, h, w, mode):
  """Soft grid labels of code/pred_models.py:1085-1136 (3x3 / 5x5 neighbourhood smoothing), for all rows at once.
  The reference convolves each one-hot map (ndimage.convolve, mode='constant'); the kernels are symmetric, so every
  cell receives exactly the kernel value at its offset from the label cell, or 0 outside the kernel."""
  tables = {1: (0.1, 1.0), 2: (0.01, 1.0), 3: (0.05, 1.0), 4: (0.0125, 0.9), 5: (0.05, 0.6), 6: (0.1, 0.2)}
  if mode == 7:
    k = np.full((5, 5), 0.0625)
    k[1:4, 1:4] = 0.0125
    k[2, 2] = 0.8
  else:
    side, centre = tables[mode]
    k = np.full((3, 3), side)
    k[1, 1] = centre
  n, t = cls.shape
  r = k.shape[0] // 2
  cell = np.arange(h * w)[np.asarray(cls).reshape(-1)]      # numpy indexing, as the reference's m[cls] = 1.0
  dy = np.arange(h)[None, :] - (cell // w)[:, None] + r     # [M, h] kernel row of every cell
  dx = np.arange(w)[None, :] - (cell % w)[:, None] + r      # [M, w]
  inside = ((dy >= 0) & (dy <= 2 * r))[:, :, None] & ((dx >= 0) & (dx <= 2 * r))[:, None, :]
  vals = k[np.clip(dy, 0, 2 * r)[:, :, None], np.clip(dx, 0, 2 * r)[:, None, :]]
  return np.where(inside, vals, 0.0).astype("float32").reshape(n, t, h, w, 1)


class Trainer(object):
  """code/pred_models.py:1636-1742."""

  def __init__(self, model, config):
    self.config = config
    self.model = model
    self.global_step = model.global_step
    self.loss = model.loss
    self.wd_loss = model.wd_loss
    if config.optimizer not in ("momentum", "adadelta", "adam", "rmsprop"):
      raise Exception("Optimizer not implemented")
    self.train_op = Handle(model, "fetch", "train_op")

  def step(self, sess, batch):
    _, batch_data = batch
    feed_dict = self.model.get_feed_dict(batch_data, is_train=True, train_traj=True)
    outputs = sess.run([self.loss, self.train_op, self.wd_loss, self.model.pred_grid_loss],
                       feed_dict=feed_dict)
    loss, train_op, wd_loss, pred_grid_loss = outputs
    return loss, train_op, wd_loss, pred_grid_loss


class Tester(object):
  """code/pred_models.py:1745-1790."""

  def __init__(self, model, config, sess=None):
    self.config = config
    self.model = model
    self.sess = sess
    self.grid_pred_decoded = self.model.grid_pred_decoded
    self.grid_pred_reg_decoded = self.model.grid_pred_reg_decoded
    self.beam_outputs = self.model.beam_outputs

  def step(self, sess, batch):
    config = self.config
    _, batch_data = batch
    feed_dict = self.model.get_feed_dict(batch_data, is_train=False)
    inputs = list(self.grid_pred_decoded) + list(self.grid_pred_reg_decoded)
    if config.use_beam_search:
      inputs.append(self.beam_outputs)
    outputs = sess.run(inputs, feed_dict=feed_dict)
    ns = len(config.scene_grids)
    grid_pred_class, grid_pred_reg = outputs[:ns], outputs[ns:2 * ns]
    beam_outputs = outputs[-1] if config.use_beam_search else None
    return grid_pred_class, grid_pred_reg, beam_outputs
