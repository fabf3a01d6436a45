# coding=utf-8
"""CPU tests of the C-ABI boundary: the library builds, loads, and exports exactly the symbols
include/multiverse_b200.h declares (no compute calls here - there is no GPU on this box)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
  src = open(os.path.join(ROOT, "include", "multiverse_b200.h")).read()
  src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
  return sorted(set(re.findall(r"\b(mvb_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
  from multiverse_b200 import build, _lib
  build.build()
  return _lib.load()


def test_header_declares_expected_surface():
  syms = header_symbols()
  for must in ("mvb_convlstm_cell_fwd", "mvb_pack_cell_weights", "mvb_gnn_attend_fwd",
               "mvb_head_class_fwd", "mvb_head_reg_fwd", "mvb_beam_step", "mvb_beam_backtrace",
               "mvb_scene_conv_fwd", "mvb_last_error"):
    assert must in syms


def test_library_exports_every_declared_symbol(lib):
  raw = ctypes.CDLL(os.path.join(ROOT, "multiverse_b200", "libmultiverse_b200.so"))
  for s in header_symbols():
    assert hasattr(raw, s), "libmultiverse_b200.so does not export %s" % s


def test_python_binding_covers_header(lib):
  from multiverse_b200 import _lib
  assert sorted(_lib.SIGNATURES) == header_symbols()


def test_abi_version_and_error_string(lib):
  assert lib.mvb_abi_version() >= 2
  assert isinstance(lib.mvb_last_error(), bytes)
  assert lib.mvb_cell_cpad(2) == 288 and lib.mvb_cell_cpad(32) == 288 and lib.mvb_cell_cpad(64) == 320


def test_argument_validation_needs_no_gpu(lib):
  # invalid plane count is rejected before any CUDA call
  rc = lib.mvb_pack_cell_weights(None, None, None, None, 32, 7, 0, None)
  assert rc != 0 and b"planes" in lib.mvb_last_error()
  # every entry point refuses null pointers / bad sizes with an error code and a message, never a crash
  rc = lib.mvb_convlstm_cell_fwd_onehot_fanout(None, None, None, None, None, None, None, None, None, 4, 20, 36, 18, 288, 2,
                                               1.0, None)
  assert rc != 0 and lib.mvb_last_error()
  rc = lib.mvb_traj_to_grid(None, None, 30.0, 106.0, None, None, 16, 36, 18, None)
  assert rc != 0 and b"traj_to_grid" in lib.mvb_last_error()
  rc = lib.mvb_decode_trajectories(None, None, None, None, 4, 20, 12, 648, None)
  assert rc != 0 and b"decode_trajectories" in lib.mvb_last_error()
  rc = lib.mvb_beam_step(None, None, None, None, None, None, 4, 20, 648, 0, 0, 1, -4.6, None)
  assert rc != 0 and b"beam_step" in lib.mvb_last_error()


def planes_entry_points():
  """name -> parameter names of every header function that takes a `planes` argument."""
  src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "multiverse_b200.h")).read(), flags=re.S)
  out = {}
  for name, params in re.findall(r"\bint\s+(mvb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src):
    names = [p.split()[-1].lstrip("*") for p in params.split(",")]
    if "planes" in names:
      out[name] = names
  return out


@pytest.mark.parametrize("planes", [1, 3, 2 | 3 << 8])
def test_only_two_operand_formats(lib, planes):
  """planes 2 (bf16x2) and MVB_PLANES_F16F8 are the only operand formats: any other code - including an output format
  of 3 planes in the `planes | out << 8` form of the cell entry points - is refused before any CUDA call."""
  eps = planes_entry_points()
  assert len(eps) == 20 and "mvb_convlstm_cell_fwd" in eps and "mvb_cell_wgrad_direct" in eps
  from multiverse_b200 import _lib
  for name, params in sorted(eps.items()):
    if planes >> 8 and not name.startswith("mvb_convlstm_cell_fwd"):
      continue
    args = []
    for pname, ty in zip(params, _lib.SIGNATURES[name]):
      if pname == "planes":
        args.append(planes)
      elif ty is ctypes.c_void_p:      # never dereferenced: the call must return first
        args.append(None if pname == "stream" else ctypes.c_void_p(256))
      else:
        args.append(ty(1))
    rc = getattr(lib, name)(*args)
    assert rc != 0 and b"planes" in lib.mvb_last_error(), (name, lib.mvb_last_error())


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
  from multiverse_b200 import _lib
  monkeypatch.setattr(_lib, "_lib", None)
  monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
  with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
    _lib.load()


def test_product_never_imports_oracle():
  pkg = os.path.join(ROOT, "multiverse_b200")
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith(".py"):
        src = open(os.path.join(dp, f)).read()
        assert "oracle" not in re.sub(r"#.*", "", src).replace('"""', ""), \
            "%s references the oracle" % f if re.search(r"^\s*(from|import)\s+oracle", src, re.M) else True
        assert not re.search(r"^\s*(from|import)\s+\.*oracle", src, re.M), f
