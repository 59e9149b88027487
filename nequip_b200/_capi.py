"""ctypes binding of libnqb.so (the C ABI declared in include/nqb.h).

Only raw pointers, sizes and the CUDA stream cross this boundary.  Importing this
module never falls back to anything: if the library cannot be built/loaded the
error propagates.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

from . import build

_lib: Optional[C.CDLL] = None


class NqbIrrep(C.Structure):
    _fields_ = [("mul", C.c_int32), ("l", C.c_int32), ("p", C.c_int32)]


class NqbInstruction(C.Structure):
    _fields_ = [("i_in1", C.c_int32), ("i_in2", C.c_int32), ("i_out", C.c_int32)]


_vp, _i64, _i32, _dbl = C.c_void_p, C.c_int64, C.c_int, C.c_double

#: name -> (restype, argtypes); kept in one table so tests can check it against nqb.h
SIGNATURES = {
    "nqb_abi_version": (_i32, []),
    "nqb_last_error": (C.c_char_p, []),
    "nqb_launch_count": (_i64, []),
    "nqb_plan_create": (
        _i32,
        [C.POINTER(NqbIrrep), _i32, C.POINTER(NqbIrrep), _i32, C.POINTER(NqbIrrep), _i32,
         C.POINTER(NqbInstruction), _i32, C.c_char_p, C.POINTER(_vp)],
    ),
    "nqb_plan_destroy": (None, [_vp]),
    "nqb_plan_dims": (_i32, [_vp, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)]),
    "nqb_plan_signature": (_i32, [_vp, C.c_char_p, _i32]),
    "nqb_csr_check_sorted": (_i32, [_vp, _i64, _vp, _vp]),
    "nqb_csr_from_sorted": (_i32, [_vp, _i64, _i64, _vp, _vp]),
    "nqb_tp_scatter_fwd": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "nqb_tp_scatter_bwd": (
        _i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _vp]),
    "nqb_tp_fused_slices": (_i32, [_vp]),
    "nqb_tp_fused_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _vp]),
    "nqb_tp_scatter_gy_slices": (_i32, [_vp, _i32]),
    "nqb_segment_sum": (_i32, [_i32, _vp, _i32, _vp, _vp, _i64, _vp, _vp]),
    "nqb_nl_bin": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_count": (_i32, [_i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_fill": (_i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_pad": (_i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_fill_capacity": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_params_bytes": (_i64, []),
    "nqb_nl_params_pack": (_i32, [_vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp]),
    "nqb_nl_bin_dp": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_count_dp": (_i32, [_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_fill_capacity_dp": (_i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_params_pack_open": (_i32, [_vp, _vp, _vp, _vp, _vp, _dbl, _vp, _i32, _vp, _vp]),
    "nqb_nl_bbox": (_i32, [_vp, _i64, _vp, _vp, _vp]),
    "nqb_sh_fwd": (_i32, [_i32, _vp, _i64, _i32, _vp, _vp]),
    "nqb_sh_bwd": (_i32, [_i32, _vp, _i64, _i32, _vp, _vp, _vp]),
    "nqb_edge_embed_fwd": (
        _i32, [_i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _vp, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp]),
    "nqb_edge_embed_bwd": (
        _i32, [_i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nqb_zbl_fwd": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp]),
    "nqb_zbl_bwd": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp, _vp, _vp]),
    "nqb_edge_embed_fwd_typed": (
        _i32, [_i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp,
               _vp]),
    "nqb_edge_embed_bwd_typed": (
        _i32, [_i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nqb_zbl_fwd_typed": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp, _vp]),
    "nqb_zbl_bwd_typed": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_count_typed": (_i32, [_i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "nqb_nl_fill_typed": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "nqb_nl_fill_capacity_typed": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp,
               _vp, _vp]),
    "nqb_nl_count_dp_typed": (_i32, [_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "nqb_nl_fill_capacity_dp_typed": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "nqb_nl_frames_pack": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp]),
    "nqb_nl_bin_frames": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nl_count_frames": (_i32, [_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "nqb_nl_fill_frames": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "nqb_nl_frames_pack_capacity": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp]),
    "nqb_nl_bbox_frames": (_i32, [_vp, _i32, _vp, _vp, _vp]),
    "nqb_nl_fill_capacity_frames": (
        _i32, [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "nqb_edge_embed_fwd_frames": (
        _i32, [_i32, _i32, _dbl, _dbl, _dbl, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp,
               _vp, _vp]),
    "nqb_zbl_fwd_frames": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp, _vp]),
    "nqb_zbl_bwd_frames": (
        _i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64, _dbl, _dbl, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nqb_md_kick_drift": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp]),
    "nqb_md_bath": (_i32, [_i32, _i32, _vp, _vp, _vp, _dbl, _vp, _vp, _vp]),
    "nqb_md_kick": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _dbl, _vp, _vp, _vp, _vp]),
    "nqb_md_log": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "nqb_nl_frames_set_cells": (_i32, [_i32, _vp, _vp, _vp, _vp]),
    "nqb_relax_fire": (_i32, [_i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_relax_move": (_i32, [_i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_relax_gforce": (_i32, [_i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_relax_finish": (
        _i32, [_i32, _i32, _vp, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _dbl, _vp, _vp, _vp, _vp, _vp, _i64,
               _vp, _vp, _vp, _vp]),
    "nqb_npt_pre": (_i32, [_i32, _i32, _i32, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_npt_move": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_npt_kick": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_npt_post": (
        _i32, [_i32, _i32, _i32, _i32, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_npt_scale": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp]),
    "nqb_npt_log": (_i32, [_i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "nqb_nptf_pre": (_i32, [_i32, _i32, _i32, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nptf_move": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nptf_kick": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nptf_post": (
        _i32, [_i32, _i32, _i32, _i32, _i32, _i32, _dbl, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_nptf_scale": (_i32, [_i32, _i32, _vp, _vp, _vp, _vp]),
    "nqb_nptf_log": (_i32, [_i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "nqb_mlp_hidden_fwd":(_i32, [_vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "nqb_mlp_hidden_bwd": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "nqb_mlp_hidden_fwd_rows": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "nqb_mlp_hidden_bwd_rows": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "nqb_edge_pairs_work_size": (_i64, [_i64]),
    "nqb_edge_pairs": (_i32, [_vp, _i64, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nqb_gemm_prepared_floats": (_i64, [_i32, _i32]),
    "nqb_gemm_prepare": (_i32, [_vp, _i64, _i32, _i32, _i32, C.c_float, _vp, _vp]),
    "nqb_gate_fwd": (_i32, [_i32, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nqb_gate_bwd": (_i32, [_i32, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    "nqb_gemm_grouped": (_i32, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "nqb_gemm_grouped_act": (_i32, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "nqb_gemm_grouped_pairs": (_i32, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "nqb_gemm_grouped_pair_sum": (_i32, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
}


def lib() -> C.CDLL:
    """Load (building first if needed) libnqb.so."""
    global _lib
    if _lib is None:
        # NQB_RUNTIME_LIB: load an alternative build of the same sources (kernel-variant experiments)
        path = os.environ.get("NQB_RUNTIME_LIB") or build.ensure_runtime()
        L = C.CDLL(path, mode=C.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        if L.nqb_abi_version() != 2:
            raise RuntimeError("libnqb.so ABI version mismatch")
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().nqb_last_error()
        raise RuntimeError(f"libnqb {what}: {msg.decode() if msg else 'error'} (rc={rc})")


def launch_count() -> int:
    return int(lib().nqb_launch_count())
