"""ctypes binding of libb200mp.so -- the thin layer between torch tensors and the C ABI.

There is NO CPU fallback and no PyTorch-eager fallback: if the library cannot be loaded (or
built), importing this module raises.  Every wrapper in ops.py refuses non-CUDA tensors.
"""
from __future__ import annotations

import ctypes
import os
import re

from . import _build

_I64 = ctypes.c_int64
_INT = ctypes.c_int
_P = ctypes.c_void_p
_F = ctypes.c_float
_U64 = ctypes.c_uint64
_D = ctypes.c_double

# name -> (restype, argtypes); mirrors include/b200mp.h one to one
_SIGS = {
    "b200mp_version": (ctypes.c_char_p, []),
    "b200mp_last_error": (ctypes.c_char_p, []),
    "b200mp_device_info": (_INT, [_P, _P, _P, _P]),
    "b200mp_set_option": (_INT, [ctypes.c_char_p, _INT]),
    "b200mp_degree": (_INT, [_P, _I64, _I64, _P, _INT, _P]),
    "b200mp_index2ptr": (_INT, [_P, _I64, _I64, _P, _INT, _P]),
    "b200mp_ptr2index": (_INT, [_P, _I64, _I64, _P, _INT, _P]),
    "b200mp_index_stats": (_INT, [_P, _I64, _P, _INT, _P]),
    "b200mp_sort_workspace_bytes": (_I64, [_I64, _I64, _INT]),
    "b200mp_sort_by_key": (_INT, [_P, _I64, _I64, _P, _P, _P, _P, _I64, _INT, _P]),
    "b200mp_permute": (_INT, [_P, _P, _P, _I64, _INT, _INT, _P]),
    "b200mp_convert_index": (_INT, [_P, _INT, _P, _INT, _I64, _P]),
    "b200mp_self_loops_workspace_bytes": (_I64, [_I64, _I64, _INT]),
    "b200mp_self_loops": (_INT, [_P, _P, _P, _I64, _I64, _F, _INT, _P, _P, _P, _P, _P, _I64, _INT, _P]),
    "b200mp_gcn_norm_csr": (_INT, [_P, _P, _P, _I64, _I64, _P, _P, _INT, _P]),
    "b200mp_csr_plan_count": (_INT, [_P, _I64, _I64, _P, _INT, _P]),
    "b200mp_csr_plan_workspace_bytes": (_I64, [_I64, _I64, _INT]),
    "b200mp_csr_plan_fill": (_INT, [_P, _I64, _I64, _I64, _P, _P, _P, _I64, _INT, _P]),
    "b200mp_spmm_csr": (_INT, [_P, _P, _P, _P, _P, _I64, _I64, _I64, _INT, _P, _P, _I64, _I64, _I64, _P,
                               _P, _P, _I64, _INT, _P, _I64, _P, _INT, _INT, _P]),
    "b200mp_spmm_csr_self_colsum": (_INT, [_P, _P, _P, _P, _P, _P, _I64, _I64, _P, _P, _I64, _I64, _I64, _P, _P, _I64,
                                           _INT, _INT, _P]),
    "b200mp_segment_csr": (_INT, [_P, _P, _P, _I64, _I64, _I64, _INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_minmax_ties": (_INT, [_P, _P, _P, _P, _P, _P, _I64, _I64, _INT, _INT, _INT, _P]),
    "b200mp_minmax_backward": (_INT, [_P, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _INT, _INT, _P]),
    "b200mp_sddmm_csr": (_INT, [_P, _P, _P, _P, _P, _I64, _I64, _INT, _INT, _P]),
    "b200mp_edge_relu_csr": (_INT, [_P] * 7 + [_I64] * 4 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_edge_relu_backward_x": (_INT, [_P] * 7 + [_I64, _I64, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_edge_relu_backward_edge": (_INT, [_P] * 5 + [_I64, _I64, _INT, _P, _P, _I64, _I64, _I64, _INT, _INT, _P]),
    "b200mp_gated_csr": (_INT, [_P] * 6 + [_I64] * 5 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_gated_backward_dst": (_INT, [_P] * 7 + [_I64] * 5 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_gated_backward_src": (_INT, [_P] * 9 + [_I64] * 5 + [_P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_cg_csr": (_INT, [_P] * 7 + [_I64] * 6 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_cg_backward_dst": (_INT, [_P] * 9 + [_I64] * 6 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_cg_backward_src": (_INT, [_P] * 9 + [_I64] * 6 + [_P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_softmax_aggr_csr": (_INT, [_P] * 8 + [_I64] * 4 + [_INT, _F, _INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT,
                                                                _P]),
    "b200mp_softmax_aggr_workspace": (_I64, [_I64, _I64, _I64]),
    "b200mp_softmax_aggr_backward_dst": (_INT, [_P] * 12 + [_I64] * 4 + [_INT, _F, _INT, _INT, _P, _P, _I64, _I64, _I64,
                                                                           _INT, _INT, _P]),
    "b200mp_softmax_aggr_backward_src": (_INT, [_P] * 10 + [_I64] * 4 + [_INT, _F, _INT, _INT, _P, _P, _I64, _I64, _I64,
                                                                           _P, _INT, _INT, _P]),
    "b200mp_power_mean_csr": (_INT, [_P] * 8 + [_I64] * 4 + [_INT, _F, _INT, _F, _F, _P, _P, _I64, _I64, _I64, _P,
                                                              _INT, _INT, _P]),
    "b200mp_power_mean_workspace": (_I64, [_I64, _I64, _I64, _I64]),
    "b200mp_power_mean_backward_dst": (_INT, [_P] * 12 + [_I64] * 4 + [_INT, _F, _INT, _F, _F, _P, _P, _I64, _I64, _I64,
                                                                         _INT, _INT, _P]),
    "b200mp_power_mean_backward_src": (_INT, [_P] * 13 + [_I64] * 4 + [_INT, _F, _INT, _F, _F, _P, _P, _I64, _I64, _I64,
                                                                         _P, _INT, _INT, _P]),
    "b200mp_quantile_bits_words": (_I64, [_I64, _I64, _INT, _I64]),
    "b200mp_quantile_csr": (_INT, [_P] * 6 + [_I64, _INT, _F, _P, _P] + [_I64] * 4 + [_P, _P, _I64, _I64, _I64, _INT,
                                                                                  _INT, _P]),
    "b200mp_quantile_backward_dst": (_INT, [_P] * 3 + [_I64, _INT, _P, _P, _P] + [_I64] * 3 + [_P, _P, _I64, _I64, _I64,
                                                                                              _INT, _INT, _P]),
    "b200mp_quantile_backward_src": (_INT, [_P] * 5 + [_I64, _INT, _P, _P, _P] + [_I64] * 4 + [_P, _P, _I64, _I64, _I64,
                                                                                              _P, _INT, _INT, _P]),
    "b200mp_nn_conv_supported": (_INT, [_I64, _I64, _INT]),
    "b200mp_nn_conv_csr": (_INT, [_P] * 6 + [_I64] * 7 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_nn_conv_backward_dst": (_INT, [_P] * 8 + [_I64] * 7 + [_INT, _P, _P, _I64, _I64, _I64, _INT, _INT, _P]),
    "b200mp_spline_supported": (_INT, [_I64, _I64, _I64, _INT]),
    "b200mp_spline_basis": (_INT, [_P] * 5 + [_I64, _I64, _INT, _INT, _INT, _P]),
    "b200mp_spline_basis_backward": (_INT, [_P] * 5 + [_I64, _I64, _INT, _INT, _P]),
    "b200mp_spline_weighting": (_INT, [_P] * 5 + [_I64] * 5 + [_INT, _INT, _P]),
    "b200mp_spline_weighting_backward": (_INT, [_P] * 10 + [_I64] * 5 + [_INT, _INT, _P]),
    "b200mp_spline_csr": (_INT, [_P] * 7 + [_I64] * 8 + [_INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_spline_backward_dst": (_INT, [_P] * 9 + [_I64] * 8 + [_INT, _P, _P, _I64, _I64, _I64, _INT, _INT, _P]),
    "b200mp_knn": (_INT, [_P] * 4 + [_I64] * 6 + [_INT, _P, _P, _INT, _INT, _P]),
    "b200mp_knn_compact": (_INT, [_P, _P, _I64, _I64, _P, _I64, _P]),
    "b200mp_radius_count": (_INT, [_P] * 4 + [_I64] * 5 + [_F, _I64, _INT, _P, _INT, _INT, _P]),
    "b200mp_radius_fill": (_INT, [_P] * 4 + [_I64] * 5 + [_F, _I64, _INT, _P, _P, _I64, _INT, _INT, _P]),
    "b200mp_nearest": (_INT, [_P] * 4 + [_I64] * 5 + [_P, _P, _INT, _INT, _P]),
    "b200mp_fps_count": (_INT, [_P, _I64, _I64, _D, _P, _INT, _P]),
    "b200mp_fps": (_INT, [_P, _P, _I64, _I64, _I64, _P, _P, _P, _P, _INT, _INT, _P]),
    "b200mp_graclus": (_INT, [_P, _P, _P, _I64, _U64, _P, _P, _INT, _INT, _P]),
    "b200mp_grid_cluster": (_INT, [_P] * 4 + [_I64, _I64, _P, _P, _INT, _P]),
    "b200mp_random_walk": (_INT, [_P] * 3 + [_I64] * 4 + [_D, _D, _I64, _U64, _P, _INT, _P, _INT, _P]),
    "b200mp_scatter_coo": (_INT, [_P, _P, _P, _P, _I64, _I64, _I64, _INT, _INT, _P]),
    "b200mp_split_tf32": (_INT, [_P, _P, _P, _I64, _P]),
    "b200mp_split_tf32_transposed": (_INT, [_P, _P, _P, _I64, _I64, _P]),
    "b200mp_linear_tf32x3": (_INT, [_P, _P, _P, _P, _I64, _I64, _I64, _P]),
    "b200mp_linear_grad_input_tf32x3": (_INT, [_P, _P, _P, _P, _I64, _I64, _I64, _P]),
    "b200mp_linear_grad_weight_workspace_bytes": (_I64, [_I64, _I64, _I64]),
    "b200mp_linear_grad_weight_tf32x3": (_INT, [_P, _P, _P, _I64, _I64, _I64, _P, _I64, _P]),
    "b200mp_gemm_pair_tf32x3": (_INT, [_P, _I64, _P, _I64, _P, _P, _INT, _P, _INT, _P, _I64, _P, _I64, _I64, _P]),
    "b200mp_segment_matmul_tf32x3": (_INT, [_P, _P, _I64, _P, _P, _INT, _P, _I64, _I64, _I64, _P]),
    "b200mp_index_add_rows": (_INT, [_P, _P, _P, _I64, _I64, _INT, _P]),
    "b200mp_gather_rows": (_INT, [_P, _P, _P, _P, _I64, _I64, _INT, _INT, _P]),
    "b200mp_softmax_csr": (_INT, [_P, _P, _P, _I64, _I64, _I64, _INT, _P]),
    "b200mp_softmax_csr_backward": (_INT, [_P, _P, _P, _P, _I64, _I64, _I64, _INT, _P]),
    "b200mp_gat_fused_csr": (_INT, [_P] * 10 + [_I64, _I64, _I64, _I64, _F, _P, _P, _I64, _I64, _I64, _P, _P, _INT, _INT, _P]),
    "b200mp_gat_fused_csr_backward": (_INT, [_P] * 18 + [_I64, _I64, _I64, _I64, _I64, _F, _P, _P, _I64, _I64, _I64, _P,
                                              _INT, _INT, _P]),
    "b200mp_scatter_arg": (_INT, [_P, _P, _P, _P, _I64, _I64, _I64, _INT, _P]),
    "b200mp_spmm_csr_arg": (_INT, [_P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _INT, _P]),
    "b200mp_attn_supported": (_INT, [_I64, _I64, _INT]),
    "b200mp_attn_csr_forward": (_INT, [_INT] + [_P] * 9 + [_I64] * 3 + [_P] * 4 + [_I64] * 4 + [_F, _F, _P, _P, _I64, _I64, _I64,
                                       _P, _P, _F, _U64, _P, _INT, _INT, _P]),
    "b200mp_attn_backward_partial_width": (_I64, [_INT, _I64, _I64, _INT]),
    "b200mp_attn_gatt_rows": (_I64, []),
    "b200mp_attn_csr_backward": (_INT, [_INT] + [_P] * 12 + [_I64] * 3 + [_P] * 12 + [_I64] * 5 + [_F, _F, _P, _P, _I64, _I64,
                                        _I64, _P, _P, _P, _I64, _I64, _P, _F, _U64, _P, _P, _INT, _INT, _P]),
    "b200mp_column_sum_parts": (_I64, [_I64]),
    "b200mp_column_sum": (_INT, [_P, _P, _P, _I64, _I64, _I64, _INT, _P]),
    "b200mp_softmax_edge_op": (_INT, [_INT, _P, _P, _P, _P, _P, _I64, _I64, _INT, _P]),
    "b200mp_multi_aggr_csr": (_INT, [_P] * 12 + [_I64, _I64, _I64, _INT, _P, _P, _I64, _I64, _I64, _P, _INT, _INT, _P]),
    "b200mp_multi_aggr_mask_supported": (_INT, [_I64, _INT, _INT]),
    "b200mp_head_dot_supported": (_INT, [_I64, _I64, _INT]),
    "b200mp_head_dot_parts": (_I64, [_I64, _I64, _I64, _INT]),
    "b200mp_head_dot": (_INT, [_P] * 5 + [_I64, _I64, _I64, _INT, _P]),
    "b200mp_head_dot_backward": (_INT, [_P] * 9 + [_I64, _I64, _I64, _I64, _INT, _P]),
    "b200mp_multi_aggr_prepare_backward": (_INT, [_P] * 15 + [_I64, _I64, _INT, _INT, _INT, _P]),
    "b200mp_multi_aggr_backward": (_INT, [_P] * 12 + [_I64, _I64, _INT, _INT, _INT, _P]),
    "b200mp_pna_epilogue": (_INT, [_P, _P, _P, _I64] + [_P] * 4 + [_P, _INT, _P, _INT, _P, _P, _P, _I64, _I64, _I64,
                                                                   _INT, _INT, _INT, _P]),
    "b200mp_pna_prologue": (_INT, [_P, _P, _P, _I64] + [_P] * 6 + [_P, _INT, _P, _INT] + [_P] * 7 + [_I64, _P, _P,
                                                                                               _I64, _I64, _I64,
                                                                                               _INT, _INT, _INT, _P]),
    "b200mp_pna_edge_stats": (_INT, [_P, _P, _P, _P, _I64] + [_P] * 7 + [_I64] * 4 + [_P, _P, _I64, _I64, _I64, _P, _INT,
                                                                                    _INT, _P]),
    "b200mp_pna_edge_backward": (_INT, [_P, _P, _P, _P, _I64] + [_P] * 8 + [_I64, _P] + [_I64] * 4 + [_INT, _INT, _P]),
}

_lib = None


def header_symbols() -> list[str]:
    """Every function declared in include/b200mp.h (used by the symbol-export test)."""
    with open(os.path.join(_build.INCLUDE, "b200mp.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200mp_[a-z0-9_]+)\s*\(", text)))


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        path = _build.LIB
        if _build.needs_build():
            try:
                path = _build.build()
            except Exception as exc:  # no silent fallback, and no stale library either (its ABI may not match _SIGS)
                state = "is missing" if not os.path.exists(_build.LIB) else "is stale (sources changed since it was built)"
                raise RuntimeError(
                    f"pytorch_geometric_b200: libb200mp.so {state} and could not be rebuilt ({exc}); "
                    "there is no CPU / eager fallback.") from exc
        l = ctypes.CDLL(path)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


class B200MPError(RuntimeError):
    pass


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().b200mp_last_error().decode()
        raise B200MPError(f"{what or 'b200mp'} failed (code {rc}): {msg}")
