"""ctypes binding of the C-ABI library (include/occ_b200.h).  There is NO fallback: if the library is
missing or a call fails, a RuntimeError is raised -- the product path never routes through PyTorch
reference code or the oracle."""
import ctypes
import os
from ctypes import c_double, c_float, c_int, c_longlong, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libocc_b200.so")
_lib = None

P = c_void_p
STREAM = c_void_p

# name -> (restype, argtypes)   -- mirrors include/occ_b200.h exactly
SIGNATURES = {
    "occ_version": (c_int, []),
    "occ_voxel_pool_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "occ_voxel_pool_workspace_layout": (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P, P]),
    "occ_lss_geometry": (c_int, [P, c_int, P, P, P, c_int, c_int, P, P, P, c_int, c_int, c_int, P, STREAM]),
    "occ_lift_prologue": (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, STREAM]),
    "occ_lift_splat": (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, c_int] + [c_float] * 9 +
                       [c_int, c_int, c_int, P, c_size_t, STREAM]),
    "occ_lift_splat_fused": (c_int, [P, c_longlong, P, c_longlong, P, P, P, P, c_int, c_int, P, P, P, c_int, P, P, P, P] +
                             [c_int] * 5 + [c_float] * 9 +
                             [c_int, c_int, c_int, P, c_size_t, STREAM]),
    "occ_voxel_pool_geom": (c_int, [P, P, P, c_int, c_int, c_int] + [c_float] * 9 + [c_int, c_int, c_int, P, c_size_t, STREAM]),
    "occ_bev_pool": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, c_size_t, STREAM]),
    "occ_gemm_bf16x3": (c_int, [P, P, P, c_int, c_int, c_int, P, P, c_int, c_int, P, c_int, c_int, STREAM]),
    "occ_conv_workspace_bytes": (c_size_t, []),
    "occ_conv_bf16x3": (c_int, [P, P, P] + [c_int] * 11 + [P, P, c_int, c_int, P, c_int, P, c_size_t, STREAM]),
    "occ_conv_plan": (c_int, [c_int] * 12 + [P]),
    "occ_conv_taps_bf16x3": (c_int, [P, P, P] + [c_int] * 7 + [P, P, c_int, STREAM]),
    "occ_set_mma_passes": (c_int, [c_int]),
    "occ_get_mma_passes": (c_int, []),
    "occ_split_rows": (c_int, [P, P, c_longlong, c_int, STREAM]),
    "occ_unsplit_rows": (c_int, [P, P, c_longlong, c_int, STREAM]),
    "occ_gn_relu_zmean_ln": (c_int, [P] * 8 + [c_int] * 7 + [STREAM]),
    "occ_window_layout_rows": (c_longlong, [c_int] * 4),
    "occ_stats_regroup": (c_int, [P, P, c_int, c_int, c_int, STREAM]),
    "occ_layernorm": (c_int, [P, P, P, P, c_longlong, c_int, c_int, STREAM]),
    "occ_gn_apply": (c_int, [P] * 7 + [c_longlong, c_int, c_int, c_int, c_int, c_int, c_int, STREAM]),
    "occ_aspp_gap_branch": (c_int, [P] * 6 + [c_int] * 6 + [STREAM]),
    "occ_dualpath_fuse": (c_int, [P, P, P, c_float, P, c_int, P, P, P, c_int, P, P, c_int, c_int, c_int, c_int, STREAM]),
    "occ_swin_proj_ffn": (c_int, [P] * 11 + [c_longlong, c_int, STREAM]),
    "occ_window_attention": (c_int, [P, P, P, P] + [c_int] * 8 + [STREAM]),
    "occ_swin_qkv_attention": (c_int, [P] * 5 + [c_int] * 7 + [STREAM]),
    "occ_neck_token_prep": (c_int, [P] * 7 + [c_int, c_int, P, c_int, STREAM]),
    "occ_ms_deform_attn": (c_int, [P, c_int, c_int, P, P, c_int, c_int, P, P, c_int, c_int, c_int, STREAM]),
    "occ_gn_upsample_add": (c_int, [P] * 4 + [c_int, P, P] + [c_int] * 8 + [STREAM]),
    "occ_gn_stats": (c_int, [P, P, c_int, c_int, c_int, c_int, STREAM]),
    "occ_sine_pos3d": (c_int, [P, c_int, c_int, c_int, c_int, c_float, c_float, c_float, c_float, STREAM]),
    "occ_head_prep": (c_int, [P, c_int, P, P, P, P, c_int, c_longlong, c_int, STREAM]),
    "occ_query_head": (c_int, [P, P, P, P, P, P, P, P, c_int, P, P, P, P, P, P, P, P, P, c_int, P, P, c_float, P, P, c_int,
                                c_int, c_int, STREAM]),
    "occ_mask_pool": (c_int, [P, P, P] + [c_int] * 8 + [STREAM]),
    "occ_mask_gemm_pool": (c_int, [P, P, P, P, P] + [c_int] * 9 + [STREAM]),
    "occ_cross_attn_tc_partials": (c_int, [c_int]),
    "occ_mask_bits": (c_int, [P, P, c_int, c_int, c_int, STREAM]),
    "occ_cross_attn_tc": (c_int, [P, P, P, c_int, c_int, c_int, P, P, P] + [c_int] * 5 + [STREAM]),
    "occ_cross_merge": (c_int, [P, c_int, c_int, P, P, c_int, P, P, P, P, P, P, c_float, P, P, c_int, c_int, STREAM]),
    "occ_self_attn_ffn": (c_int, [P, P, c_int, P, P, P, P, P, P, P, P, c_int, P, P, P, c_int, c_int, c_int, STREAM]),
    "occ_classmix": (c_int, [P, P, P, P] + [c_int] * 9 + [STREAM]),
    "occ_transpose_sq": (c_int, [P, P, c_int, c_longlong, c_int, STREAM]),
    "occ_ssc_counts": (c_int, [P, P, c_longlong, c_int, c_int, P, P, STREAM]),
    "occ_lidarseg_hist": (c_int, [P, P, c_int, c_int, P, STREAM]),
    "occ_lidarseg_points": (c_int, [P, P, c_int, c_int] + [c_float] * 6 + [c_int] * 5 + [P, STREAM]),
}


def lib():
    """Load (once) and return the shared library; raise loudly if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"occformer_b200: {LIB_PATH} is missing. Build it with `python -m occformer_b200.build` "
            "(or __graft_entry__.build()). There is no CPU / PyTorch fallback for the hot path.")
    l = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(l, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = l
    return l


def check(rc, what):
    if rc != 0:
        kind = "argument error" if rc < 0 else "cudaError"
        raise RuntimeError(f"occformer_b200: {what} failed with {kind} {rc}")
