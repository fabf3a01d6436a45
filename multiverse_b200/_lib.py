# coding=utf-8
"""ctypes binding of libmultiverse_b200.so (the C ABI of include/multiverse_b200.h).

There is NO fallback: if the shared library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmultiverse_b200.so")

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float

# name -> argtypes (every function returns int unless listed in _RESTYPES)
SIGNATURES = {
    "mvb_last_error": [],
    "mvb_abi_version": [],
    "mvb_launch_count": [],
    "mvb_reset_launch_count": [],
    "mvb_cell_cpad": [_i],
    "mvb_cell_last_variant": [],
    "mvb_cell_variants_seen": [_i],
    "mvb_pack_cell_weights": [_vp, _vp, _vp, _vp, _i, _i, _i, _vp],
    "mvb_convlstm_cell_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i64, _i, _i,
                              _i, _i, _f, _vp],
    "mvb_cell_xfold_tables": [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp],
    "mvb_convlstm_cell_fwd_xdense": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i64, _i, _i,
                                     _i, _i, _f, _vp],
    "mvb_cell_xdense_weights": [_vp, _vp, _vp],
    "mvb_convlstm_cell_fwd_xsparse": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i64, _i, _i,
                                      _i, _i, _f, _vp],
    "mvb_cell_xsparse_weights": [_vp, _i, _vp, _vp],
    "mvb_cell_xsparse_table": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp],
    "mvb_convlstm_cell_fwd_onehot_fanout": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _f, _vp],
    "mvb_convlstm_cell_fwd_onehot": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i64,
                                     _i, _i, _i, _i, _f, _vp],
    "mvb_convlstm_cell_fwd_train": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i64, _i, _i,
                                    _i, _i, _f, _vp],
    "mvb_lstm_gates_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_pack_cell_weights_dgrad": [_vp, _vp, _i, _i, _vp],
    "mvb_cell_dgrad": [_vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _vp],
    "mvb_cell_wgrad_direct": [_vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_unpack_cell_wgrad": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "mvb_cell_wgrad_slabs": [_i],
    "mvb_loss_fwd_bwd": [_vp, _vp, _vp, _i64, _i, _f, _vp, _vp, _vp, _i64, _f, _vp, _vp],
    "mvb_soft_ce_fwd_bwd": [_vp, _vp, _vp, _i64, _i, _f, _vp, _vp],
    "mvb_fg_count": [_vp, _vp, _i64, _i, _vp, _vp],
    "mvb_masked_huber_fwd_bwd": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _f, _vp, _vp],
    "mvb_huber_traj_fwd_bwd": [_vp, _vp, _vp, _vp, _i64, _i, _i, _f, _vp, _vp],
    "mvb_soft_ce_label_fwd_bwd": [_vp, _vp, _i, _vp, _i64, _i, _i, _f, _vp, _vp],
    "mvb_fg_count_label": [_vp, _i, _i64, _i, _i, _vp, _vp],
    "mvb_masked_huber_traj_fwd_bwd": [_vp, _vp, _vp, _vp, _vp, _i, _i64, _i, _i, _i, _vp, _f, _vp, _vp],
    "mvb_head_bwd": [_vp, _vp, _vp, _i, _vp, _vp, _i, _i64, _i, _i, _vp],
    "mvb_emb_bwd": [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i64, _i, _i, _vp],
    "mvb_gnn_attend_bwd": [_vp, _vp, _vp, _vp, _vp, _i, _vp, _i64, _i, _i, _vp],
    "mvb_scene_conv_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_enc_class_input_bwd": [_vp, _i, _vp, _vp, _vp, _i64, _i, _i, _vp],
    "mvb_scene_time_mean_bwd": [_vp, _vp, _vp, _i64, _i, _i64, _vp],
    "mvb_clip_adadelta": [_vp, _vp, _vp, _vp, _i64, _f, _f, _f, _f, _f, _f, _vp],
    "mvb_nhwc_to_planes": [_vp, _vp, _i64, _i, _i, _i64, _i, _i, _i, _i, _i, _vp],
    "mvb_nhwc_to_halo": [_vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_halo_to_nhwc": [_vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_enc_class_input": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_scene_conv_fwd": [_vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_scene_time_mean": [_vp, _vp, _vp, _i64, _i, _i64, _vp],
    "mvb_gnn_attend_fwd": [_vp, _vp, _vp, _i, _vp, _i64, _i, _i, _i64, _i, _i, _i, _vp],
    "mvb_head_class_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_head_class_fwd_dense": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_head_reg_fwd": [_vp, _vp, _vp, _vp, _vp, _i, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_emb_onehot_fwd": [_vp, _vp, _vp, _i, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_emb_dense_fwd": [_vp, _vp, _vp, _i, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_beam_step": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _f, _vp],
    "mvb_traj_to_grid": [_vp, _vp, C.c_double, C.c_double, _vp, _vp, _i64, _i, _i, _vp],
    "mvb_traj_to_planes": [_vp, _i64, _vp, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_decode_trajectories": [_vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_clip_update": [_vp, _vp, _vp, _vp, _i64, _i, _f, _f, _f, _f, _f, _f, _f, _vp],
    "mvb_adv_step": [_vp, _vp, _vp, _vp, _f, _f, _i64, _vp],
    "mvb_ce_rows": [_vp, _vp, _vp, _i64, _i, _vp],
    "mvb_enc_class_input_mix": [_vp, _vp, _vp, _vp, _f, _vp, _i64, _i, _i64, _i, _i, _i, _vp],
    "mvb_enc_class_input_mix_bwd": [_vp, _i, _vp, _vp, _vp, _f, _vp, _i64, _i, _i, _vp],
    "mvb_mix": [_vp, _vp, _vp, _f, _i64, _vp],
    "mvb_min_ade_fde": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_beam_nll": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _vp],
    "mvb_beam_nll_ragged": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _vp],
    "mvb_min_ade_fde_cells": [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i,
                              _vp],
    "mvb_points_to_cells": [_vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_beam_backtrace": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_beam_backtrace_ragged": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_gather_offsets": [_vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
    "mvb_beam_gather_h_f16f8": [_vp, _vp, _vp, _i64, _i, _i64, _i, _i, _vp],
    "mvb_beam_band": [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _vp],
    "mvb_beam_band_copy": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
}
_RESTYPES = {"mvb_last_error": C.c_char_p, "mvb_launch_count": C.c_longlong, "mvb_cell_variants_seen": C.c_longlong,
             "mvb_reset_launch_count": None}

_lib = None


def load():
  """Load the library once; raises RuntimeError if it has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        "libmultiverse_b200.so is not built (%s). Run `python -m multiverse_b200.build`; "
        "there is no CPU or PyTorch fallback for the hot path." % LIB_PATH)
  lib = C.CDLL(LIB_PATH)
  for name, args in SIGNATURES.items():
    fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
    fn.argtypes = args
    fn.restype = _RESTYPES.get(name, C.c_int)
  _lib = lib
  return lib


def check(rc, what):
  if rc != 0:
    msg = load().mvb_last_error()
    raise RuntimeError("%s failed (code %d): %s" % (what, rc, msg.decode() if msg else "?"))


def call(name, *args):
  """Call an int-returning entry point and raise on a non-zero code."""
  check(getattr(load(), name)(*args), name)
