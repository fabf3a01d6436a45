# coding=utf-8
"""In-tree nvcc build of libmultiverse_b200.so for the H100 (sm_90a only; no fallback arch).

``python -m multiverse_b200.build`` or ``multiverse_b200.build.build()``.
The .so and the objects are build products: git ignores them and build() recreates them.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmultiverse_b200.so")
OBJ = os.path.join(HERE, "build")
SOURCES = ["mvb_api.cu", "mvb_cell.cu", "mvb_layout.cu", "mvb_scene.cu", "mvb_gnn.cu",
           "mvb_head.cu", "mvb_beam.cu", "mvb_train.cu", "mvb_train2.cu", "mvb_metrics.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
  for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
    if cand and (os.path.sep not in cand or os.path.exists(cand)):
      return cand
  raise RuntimeError("nvcc not found")


def _stamp(paths):
  h = hashlib.sha1()
  for p in sorted(paths):
    with open(p, "rb") as f:
      h.update(f.read())
  h.update(" ".join(NVCC_FLAGS).encode())
  return h.hexdigest()


def sources():
  return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def build(force=False, verbose=False):
  """Compile every .cu into an object and link the shared library (skips if up to date).  Serialised across
  processes with a lock file: the ranks of a torchrun job all call this.  An up-to-date library is recognised
  without writing anything, so a built tree may be read-only."""
  import fcntl
  if not force and _up_to_date():
    return LIB
  os.makedirs(OBJ, exist_ok=True)
  with open(os.path.join(OBJ, ".lock"), "w") as lock:
    fcntl.flock(lock, fcntl.LOCK_EX)
    try:
      return _build_locked(force, verbose)
    finally:
      fcntl.flock(lock, fcntl.LOCK_UN)


def _current_stamp():
  deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
  deps.append(os.path.join(HERE, "..", "include", "multiverse_b200.h"))
  return _stamp(deps)


def _up_to_date(stamp=None):
  stamp_file = os.path.join(OBJ, "stamp")
  if not (os.path.exists(LIB) and os.path.exists(stamp_file)):
    return False
  with open(stamp_file) as f:
    return f.read().strip() == (stamp or _current_stamp())


def _build_locked(force, verbose):
  stamp = _current_stamp()
  if not force and _up_to_date(stamp):
    return LIB
  _compile_and_link(LIB, OBJ, NVCC_FLAGS, verbose)
  with open(os.path.join(OBJ, "stamp"), "w") as f:
    f.write(stamp)
  return LIB


def build_variant(out_dir, defines=(), verbose=False):
  """Compile the library with extra preprocessor definitions (e.g. MVB_CELL_PROBE, the cell kernel's phase profile)
  into out_dir/libmultiverse_b200.so, leaving the in-tree library alone.  Returns the library's path."""
  os.makedirs(out_dir, exist_ok=True)
  lib = os.path.join(out_dir, os.path.basename(LIB))
  _compile_and_link(lib, out_dir, NVCC_FLAGS + ["-D" + d for d in defines], verbose)
  return lib


def _compile_and_link(lib, obj_dir, flags, verbose):
  srcs = sources()
  nvcc = _nvcc()

  def compile_one(src):
    obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
    cmd = [nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if verbose:
      sys.stderr.write(r.stderr)
    return obj

  with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
    objs = list(ex.map(compile_one, srcs))
  cmd = [nvcc, "-shared", "-o", lib] + objs + GENCODE + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"]
  r = subprocess.run(cmd, capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))


if __name__ == "__main__":
  print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
