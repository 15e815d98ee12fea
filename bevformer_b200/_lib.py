"""ctypes binding of ``libbevformer_b200.so`` (the C ABI declared in ``include/bevformer_b200.h``).

There is no fallback: if the library is missing and cannot be built, importing an op raises.
"""
from __future__ import annotations

import ctypes
import os
import threading

from . import build as _build

_lock = threading.Lock()
_lib = None

c_void_p, c_int, c_int64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64

# name -> (restype, argtypes); mirrors include/bevformer_b200.h one to one
SIGNATURES = {
    "bevf_version": (c_int, []),
    "bevf_last_error": (ctypes.c_char_p, []),
    "bevf_launch_count": (c_int64, []),
    "bevf_msda_forward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_int] + [c_int] * 7 + [c_void_p]),
    "bevf_msda_backward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 7
                           + [c_void_p]),
    "bevf_msda_rows_forward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_int, c_void_p] + [c_int] * 7 + [c_void_p]),
    "bevf_msda_rows_backward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
                                + [c_int] * 7 + [c_void_p]),
    "bevf_msda_rows_backward_ordered": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p] + [c_int] * 7 + [c_void_p]),
    "bevf_msda_set_backward_mode": (c_int, [c_int]),
    "bevf_abs_max": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "bevf_msda_rows_backward_f16acc": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 7
                                       + [c_void_p]),
    "bevf_gv16_unscale": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "bevf_msda_rows_backward_mixed": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                              c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                              c_void_p] + [c_int] * 7 + [c_void_p]),
    "bevf_msda_rows_backward_mixed_dense": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                    c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                    c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "bevf_gv_merge": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "bevf_msda_fx_frac_bits": (c_int, [c_int64, c_int, c_int]),
    "bevf_msda_backward_fx": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                      c_void_p, c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "bevf_msda_rows_backward_fx": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                           c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 7
                                   + [c_void_p]),
    "bevf_msda_fx_convert": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int64, c_void_p]),
    "bevf_msda_rows_backward_dense": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
                                      + [c_int] * 7 + [c_void_p]),
    "bevf_msda_set_dense_backward": (c_int, [c_int]),
    "bevf_msda_get_dense_backward": (c_int, []),
    "bevf_msda_dense_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "bevf_sca_plan_workspace_ints": (c_int64, [c_int, c_int]),
    "bevf_sca_plan_build": (c_int, [c_void_p] * 10 + [c_int] * 5 + [c_void_p]),
    "bevf_sca_prep_forward": (c_int, [c_void_p] * 7 + [c_int] * 8 + [c_void_p]),
    "bevf_sca_prep_backward": (c_int, [c_void_p] * 6 + [c_int] * 8 + [c_void_p]),
    "bevf_sca_rows_forward_fused": (c_int, [c_void_p, c_int] + [c_void_p] * 9 + [c_int, c_void_p, c_int, c_void_p]
                                    + [c_int] * 12 + [c_void_p]),
    "bevf_sca_rows_backward_fused": (c_int, [c_void_p, c_int] + [c_void_p] * 7 + [c_int] + [c_void_p] * 5
                                     + [c_int, c_void_p, c_void_p, c_void_p, c_int, c_int] + [c_void_p] * 5
                                     + [c_int] * 12 + [c_void_p]),
    "bevf_sca_prep_backward_multi": (c_int, [c_void_p] * 6 + [c_int] * 8 + [c_void_p]),
    "bevf_tsa_prep_forward": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_void_p]),
    "bevf_tsa_prep_backward": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p]),
    "bevf_query_prep_forward": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p]),
    "bevf_query_prep_backward": (c_int, [c_void_p] * 5 + [c_int] * 8 + [c_void_p]),
    "bevf_refine_points": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "bevf_layernorm_forward": (c_int, [c_void_p] * 4 + [c_int] + [c_void_p] * 5
                               + [c_int64, c_int, ctypes.c_float, ctypes.c_float, ctypes.c_uint64, c_void_p,
                                  c_int, c_void_p]),
    "bevf_layernorm_backward": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 4 + [c_int64]
                                + [c_void_p] * 4
                                + [c_int64, c_int, ctypes.c_float, ctypes.c_uint64, c_void_p, c_int,
                                   c_void_p]),
    "bevf_layernorm_backward_workspace_bytes": (c_int64, [c_int64, c_int]),
    "bevf_layernorm_backward_det": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 4 + [c_int64]
                                    + [c_void_p] * 5 + [c_int64]
                                    + [c_int64, c_int, ctypes.c_float, ctypes.c_uint64, c_void_p, c_int,
                                       c_void_p]),
    "bevf_sca_combine_forward": (c_int, [c_void_p] * 4 + [c_int] * 6 + [c_void_p]),
    "bevf_sca_combine_backward": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_void_p]),
    "bevf_linear_forward": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 2
                            + [c_int, c_int64, c_int, c_int, c_int, c_void_p]),
    "bevf_flatten_feats": (c_int, [c_void_p] * 4 + [c_int] * 7 + [c_void_p]),
    "bevf_linear_dgrad": (c_int, [c_void_p] * 3 + [c_int64, c_int, c_int, c_void_p]),
    "bevf_linear_dgrad_acc": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_void_p]),
    "bevf_linear_wgrad": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_void_p]),
    "bevf_linear_wgrad_workspace_bytes": (c_int64, [c_int64, c_int, c_int]),
    "bevf_linear_wgrad_out": (c_int, [c_void_p] * 4 + [c_int, c_void_p, c_int64, c_int64, c_int, c_int,
                                                      c_void_p]),
    "bevf_sum_tensors": (c_int, [c_void_p, c_int, c_void_p, c_int64, c_int, c_void_p]),
    "bevf_linear_wgrad_into": (c_int, [c_void_p] * 5 + [c_int64, c_int64, c_int, c_int, c_void_p]),
    "bevf_linear_forward_dt": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 2
                               + [c_int, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "bevf_linear_dgrad_dt": (c_int, [c_void_p] * 3 + [c_int64, c_int, c_int, c_int, c_void_p]),
    "bevf_linear_dgrad_acc_dt": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_int, c_void_p]),
    "bevf_linear_wgrad_dt": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_int, c_void_p]),
    "bevf_linear_wgrad_out_dt": (c_int, [c_void_p] * 4 + [c_int, c_void_p, c_int64, c_int64, c_int, c_int, c_int,
                                                         c_void_p]),
    "bevf_linear_wgrad_into_dt": (c_int, [c_void_p] * 5 + [c_int64, c_int64, c_int, c_int, c_int, c_void_p]),
    "bevf_colsum": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "bevf_colsum_workspace_bytes": (c_int64, [c_int64, c_int]),
    "bevf_colsum_det": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p]),
    "bevf_dropout_inplace": (c_int, [c_void_p, c_int64, ctypes.c_float, ctypes.c_uint64, c_void_p, c_int,
                                     c_void_p]),
    "bevf_relu_dropout_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, ctypes.c_float, c_int,
                                           c_void_p]),
    "bevf_point_sampling": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_float, ctypes.c_float,
                                    c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "bevf_attn_forward": (c_int, [c_void_p, c_int64] * 4 + [c_void_p] + [c_int] * 6
                          + [ctypes.c_float, ctypes.c_float, ctypes.c_uint64, c_void_p, c_int, c_void_p]),
    "bevf_attn_backward": (c_int, [c_void_p, c_int64] * 5 + [c_void_p, c_void_p] + [c_void_p, c_int64] * 3
                           + [c_int] * 6 + [ctypes.c_float, ctypes.c_float, ctypes.c_uint64, c_void_p, c_int,
                                            c_void_p]),
    "bevf_attn_dropout_mask": (c_int, [c_void_p] + [c_int] * 5 + [ctypes.c_float, ctypes.c_uint64, c_void_p,
                                                                  c_void_p]),
    "bevf_ego_motion": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int]
                        + [ctypes.c_double] * 4 + [c_int, c_void_p]),
    "bevf_rotate_bev": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "bevf_det_branches_forward": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p, c_void_p, c_int,
                                          c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 6
                                  + [ctypes.c_float, c_void_p, c_void_p]),
    "bevf_nms_free_decode": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_int] * 5
                             + [c_void_p, c_int, ctypes.c_double, c_int] + [c_void_p] * 5),
    "bevf_nms_free_decode_smem_bytes": (c_int64, [c_int, c_int, c_int]),
    "bevf_det_match_cost": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 4 + [c_int] * 6
                            + [ctypes.c_float] * 5 + [c_void_p]),
    "bevf_det_match_cost_smem_bytes": (c_int64, [c_int, c_int]),
    "bevf_det_loss_forward": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 8 + [c_int] * 7
                              + [ctypes.c_float] * 5 + [c_void_p]),
    "bevf_det_loss_backward": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 10 + [c_int] * 7
                               + [ctypes.c_float] * 5 + [c_void_p]),
    "bevf_dcn_sampling_forward": (c_int, [c_void_p] * 3 + [c_int, c_void_p] + [c_int] * 15 + [c_void_p]),
    "bevf_dcn_sampling_backward": (c_int, [c_void_p] * 4 + [c_int] + [c_void_p] * 3 + [c_int] * 15 + [c_void_p]),
    "bevf_dcn_sampling_backward_fx": (c_int, [c_void_p] * 4 + [c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]
                                      + [c_int] * 15 + [c_void_p]),
}


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True):
    """Load (building first if the in-tree .so is absent or stale and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = _build.LIB_PATH
        if build_if_missing:
            try:
                path = _build.build()
            except Exception as e:  # no nvcc on this box: use the prebuilt .so if there is one
                if not os.path.exists(path):
                    raise RuntimeError(
                        "bevformer_b200: the CUDA library is missing and could not be built "
                        f"({e}); there is no CPU fallback") from e
        if not os.path.exists(path):
            raise RuntimeError(f"bevformer_b200: {path} not found; there is no CPU fallback")
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        have = lib.bevf_version()
        if have != ABI_VERSION:
            raise RuntimeError(f"bevformer_b200: ABI mismatch (library {have}, binding {ABI_VERSION})")
        _lib = lib
    return _lib


ABI_VERSION = 4


def check(status: int, lib=None) -> None:
    """Non-zero status -> RuntimeError carrying the library's message (what mmcv's TORCH_CHECK
    failures look like from Python)."""
    if status != 0:
        lib = lib or load()
        raise RuntimeError(lib.bevf_last_error().decode() or f"bevformer_b200 error {status}")


def launch_count() -> int:
    return int(load().bevf_launch_count())
