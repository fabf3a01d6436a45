# coding=utf-8
"""`tensorflow`-named shim: the ~14 TF symbols that the reference's callers (code/train.py,
code/test.py, code/multifuture_inference.py, code/pred_utils.py) touch OUTSIDE pred_models, so
those files run byte-identical on top of multiverse_b200 (SURVEY.md §8b).  Put this directory
first on sys.path.  It is not TensorFlow: there is no graph, `Session.run` hands the fetch
handles owned by multiverse_b200.pred_models.Model back to that model.

Covered call sites: tf.compat.v1.logging.{set_verbosity,ERROR} (train.py:23, test.py:20),
tf.global_variables() (train.py:156, pred_utils.py:166), tf.global_variables_initializer().run()
(pred_utils.py:162), tf.train.Saver(...).save/restore (train.py:170-171,222,244,268;
pred_utils.py:174,190,198), tf.train.get_checkpoint_state (pred_utils.py:186),
tf.ConfigProto(...).gpu_options (train.py:176-179), tf.Session (train.py:180), tf.device /
tf.name_scope (pred_models.py:28, multifuture_inference.py:454), tf.nn.{tanh,relu,leaky_relu}
as opaque activation tokens (pred_utils.py:86-94)."""
from __future__ import annotations

import contextlib
import os
import types
import weakref

import numpy as np

__version__ = "1.15.0-multiverse_b200-shim"


# --------------------------------------------------------------------------- variables
class TensorShape(tuple):
  def as_list(self):
    return list(self)


class Variable(object):
  """A named parameter.  `value` is the host fp32/int copy; models keep device copies."""

  def __init__(self, name, shape, dtype="float32", initializer=None, trainable=True, owner=None):
    self.name = name + ":0"
    self.op = types.SimpleNamespace(name=name)
    self.shape = TensorShape(shape)
    self.dtype = dtype
    self.trainable = trainable
    self.initializer_fn = initializer
    self._owner = None if owner is None else weakref.ref(owner)     # the owning model holds its variables
    self.value = np.zeros(shape, dtype=dtype)

  @property
  def owner(self):
    return None if self._owner is None else self._owner()

  def get_shape(self):
    return self.shape

  def assign(self, value):
    self.value = np.asarray(value, dtype=self.dtype).reshape(self.shape)
    if self.owner is not None:
      self.owner._variables_changed()

  def eval(self, session=None):
    if self.owner is not None:
      self.owner._sync_to_host()
    return self.value


class _Graph(object):
  def __init__(self):
    self.variables = []

  def add(self, var):
    self.variables.append(var)
    return var


_GRAPH = _Graph()


def reset_default_graph():
  _GRAPH.variables = []


def global_variables():
  return list(_GRAPH.variables)


def trainable_variables():
  return [v for v in _GRAPH.variables if v.trainable]


class _InitOp(object):
  def run(self, session=None):
    for v in _GRAPH.variables:
      if v.initializer_fn is not None:
        v.assign(v.initializer_fn(v.shape))
      else:
        v.assign(np.zeros(v.shape, dtype=v.dtype))


def global_variables_initializer():
  return _InitOp()


# --------------------------------------------------------------------------- session
class _GpuOptions(object):
  allow_growth = False
  visible_device_list = ""


class ConfigProto(object):
  def __init__(self, **kw):
    self.gpu_options = _GpuOptions()
    self.__dict__.update(kw)


class Session(object):
  def __init__(self, config=None):
    self.config = config

  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False

  def close(self):
    pass

  def run(self, fetches, feed_dict=None):
    flat = []
    tree = _flatten_fetches(fetches, flat)
    owners = [getattr(f, "owner", None) for f in flat]
    model = next((o for o in owners if o is not None), None)
    if model is None:
      raise ValueError("Session.run: nothing to fetch from a multiverse_b200 model")
    return _rebuild_fetches(tree, model._run(flat, feed_dict or {}))


# Module-level on purpose: as nested recursive closures these two formed reference cycles (function <-> its own
# closure cell) that kept every fetched array - and its pinned host block - alive until the next cyclic GC pass.
def _flatten_fetches(f, flat):
  if isinstance(f, (list, tuple)):
    return [_flatten_fetches(x, flat) for x in f]
  flat.append(f)
  return len(flat) - 1


def _rebuild_fetches(t, vals):
  return [_rebuild_fetches(x, vals) for x in t] if isinstance(t, list) else vals[t]


@contextlib.contextmanager
def device(name):
  yield


@contextlib.contextmanager
def name_scope(name, *a, **kw):
  yield name


# --------------------------------------------------------------------------- checkpoints
class _CheckpointState(object):
  def __init__(self, path):
    self.model_checkpoint_path = path


def _index_file(dirname):
  return os.path.join(dirname, "checkpoint")


class _Train(object):
  class Saver(object):
    """Writes `<path>-<step>.npz` keyed by the TF variable names plus a TF-style `checkpoint`
    index file; restore accepts those files and TensorFlow's own checkpoint bundles
    (`<path>.index` + `<path>.data-*`, read by tensorflow/_bundle.py - SURVEY.md §8 row f-2)."""

    def __init__(self, var_list=None, max_to_keep=5):
      self.var_list = var_list
      self.max_to_keep = max_to_keep
      self._kept = []

    def _vars(self):
      return self.var_list if self.var_list is not None else global_variables()

    def save(self, sess, save_path, global_step=None):
      step = None
      if global_step is not None:
        step = int(global_step.eval() if hasattr(global_step, "eval") else global_step)
      path = save_path if step is None else "%s-%d" % (save_path, step)
      os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
      np.savez(path + ".npz", **{v.name.split(":")[0]: v.eval() for v in self._vars()})
      save_dir = os.path.dirname(os.path.abspath(path))
      # TF's generate_checkpoint_state_proto: a relative save path is recorded RELATIVE TO THE CHECKPOINT
      # DIRECTORY (get_checkpoint_state joins it back), an absolute one as given
      entry = path if os.path.isabs(path) else os.path.relpath(path, save_dir)
      with open(_index_file(save_dir), "w") as f:
        f.write('model_checkpoint_path: "%s"\n' % entry)
      self._kept.append(path)
      while self.max_to_keep and len(self._kept) > self.max_to_keep:
        old = self._kept.pop(0)
        if os.path.exists(old + ".npz"):
          os.remove(old + ".npz")
      return path

    def restore(self, sess, save_path):
      from . import _bundle
      f = save_path if save_path.endswith(".npz") else save_path + ".npz"
      if os.path.exists(f):
        data = np.load(f)
      elif _bundle.is_bundle(save_path):
        f = save_path + ".index"
        data = _bundle.read_bundle(save_path, names={v.name.split(":")[0] for v in self._vars()})
      else:
        raise IOError("checkpoint %s(.npz | .index) not found" % save_path)
      for v in self._vars():
        key = v.name.split(":")[0]
        if key not in data:
          names = sorted(data.keys() if hasattr(data, "keys") else data.files)
          tail = key.split("/")[-1]
          near = [n for n in names if n.split("/")[-1] == tail][:8]
          raise KeyError("variable %s missing from %s (%d tensors; same leaf name: %s)" % (key, f, len(names), near))
        v.assign(data[key])

  @staticmethod
  def get_checkpoint_state(dirname):
    idx = _index_file(dirname)
    if not os.path.exists(idx):
      return None
    with open(idx) as f:
      for line in f:
        if line.startswith("model_checkpoint_path"):
          path = line.split(":", 1)[1].strip().strip('"')
          if not os.path.isabs(path):                     # TF resolves relative entries against the directory
            path = os.path.join(dirname, path)
          return _CheckpointState(path)
    return None


train = _Train()


# --------------------------------------------------------------------------- misc tokens
def _token(name):
  def fn(*a, **k):
    raise RuntimeError("tf.nn.%s is an activation token in this shim, not an op" % name)
  fn.__name__ = name
  return fn


nn = types.SimpleNamespace(tanh=_token("tanh"), relu=_token("relu"), leaky_relu=_token("leaky_relu"))
identity = _token("identity")


class _Logging(object):
  ERROR, WARN, INFO, DEBUG = 40, 30, 20, 10

  @staticmethod
  def set_verbosity(level):
    pass


logging = _Logging()
from . import compat  # noqa: E402,F401


def constant_initializer(value=0.0, dtype=None):
  """Only evaluated as a default argument when the reference's own pred_models.py is imported
  beside the shim (tests); returns a shape -> ndarray callable."""
  return lambda shape: np.full(tuple(shape), value, dtype="float32")
