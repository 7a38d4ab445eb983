"""ctypes binding of libgigapose_b200.so (the C ABI declared in include/gigapose_b200.h).

There is no CPU fallback: if the shared library is missing the import fails loudly.  The library itself refuses
non-sm_90 devices at gp_create.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libgigapose_b200.so")

GP_ABI_VERSION = 2
LAYOUT_CHANNEL_MAJOR = 0
LAYOUT_PATCH_MAJOR = 1
LAYOUT_VIT_TOKENS = 2
PRECISION_FP32_SPLIT = 0
PRECISION_BF16 = 1
MAX_NUM_TEMPLATES = 12032      # GP_MAX_NUM_TEMPLATES: largest num_templates per handle


class GpConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("device", C.c_int32), ("num_objects", C.c_int32), ("num_templates", C.c_int32),
        ("num_templates_global", C.c_int32), ("template_id_stride", C.c_int32), ("template_id_offset", C.c_int32),
        ("max_batch", C.c_int32), ("top_k", C.c_int32), ("sim_threshold", C.c_float), ("patch_threshold", C.c_float),
        ("pixel_threshold", C.c_float), ("patch_size", C.c_int32), ("precision", C.c_int32),
        ("ist_bank_global", C.c_int32),
    ]


class GpCandidates(C.Structure):
    _fields_ = [("score", C.c_void_p), ("id", C.c_void_p), ("pts_score", C.c_void_p), ("idx", C.c_void_p),
                ("valid", C.c_void_p), ("rel_scale", C.c_void_p), ("rel_inplane", C.c_void_p)]


class GpMatches(C.Structure):
    _fields_ = [("id_src", C.c_void_p), ("score_src", C.c_void_p), ("score_pts", C.c_void_p), ("tar_pts", C.c_void_p),
                ("src_pts", C.c_void_p)]


class GpDebugGemm(C.Structure):
    _fields_ = [("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("bn", C.c_int32), ("passes", C.c_int32),
                ("mode", C.c_int32), ("swap", C.c_int32), ("f16", C.c_int32), ("acc_scale", C.c_float),
                ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("w_hi", C.c_void_p), ("w_lo", C.c_void_p),
                ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("bias", C.c_void_p), ("gamma", C.c_void_p),
                ("x", C.c_void_p), ("pos", C.c_void_p), ("res_hi", C.c_void_p), ("res_lo", C.c_void_p),
                ("m_dev", C.c_void_p), ("tokens_per_img", C.c_int32), ("patches_per_img", C.c_int32),
                ("qkv_crop_stride", C.c_int32)]


# gp_debug_gemm_t.mode
GEMM_PLANES, GEMM_PLANES_GELU, GEMM_SCALE_RESIDUAL, GEMM_PATCH_EMBED, GEMM_QKV_HEADS = 0, 1, 2, 3, 4
GEMM_PLANES_RELU, GEMM_PLANES_ADD_RELU, GEMM_ROWS_F32, GEMM_ROWS_F32_RELU = 5, 6, 7, 8


class GpRansacOut(C.Structure):
    _fields_ = [("M", C.c_void_p), ("failed", C.c_void_p), ("inlier_src_pts", C.c_void_p),
                ("inlier_tar_pts", C.c_void_p), ("inlier_scores", C.c_void_p), ("inlier_count", C.c_void_p)]


class GpPredictions(C.Structure):
    _fields_ = [("matches", GpMatches), ("rel_scale", C.c_void_p), ("rel_inplane", C.c_void_p),
                ("ransac", GpRansacOut), ("scores", C.c_void_p), ("poses", C.c_void_p)]


# every symbol include/gigapose_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "gp_last_error": (C.c_char_p, []),
    "gp_abi_version": (C.c_int, []),
    "gp_query_sizes": (C.c_int, [C.POINTER(GpConfig), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "gp_create": (C.c_int, [C.POINTER(GpConfig), C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "gp_destroy": (C.c_int, [C.c_void_p]),
    "gp_bank_write": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "gp_bank_write_ist": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "gp_bank_set_poses": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_set_ist_weights": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_void_p]),
    "gp_set_queries": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                 C.c_void_p, C.c_void_p]),
    "gp_sim_candidates": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(GpCandidates), C.c_void_p]),
    "gp_topk_merge": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(GpCandidates), C.c_size_t, C.POINTER(GpMatches),
                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_sim_topk": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(GpMatches), C.c_void_p]),
    "gp_ist_mlp": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(GpMatches), C.c_void_p, C.c_void_p,
                             C.c_void_p]),
    "gp_ransac": (C.c_int, [C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.POINTER(GpRansacOut), C.c_void_p]),
    "gp_pose_recover": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_sort_and_pose": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(GpMatches),
                                   C.c_void_p, C.c_void_p, C.POINTER(GpRansacOut), C.POINTER(GpPredictions), C.c_void_p]),
    "gp_comm_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "gp_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "gp_topk_allgather_merge": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(GpCandidates),
                                          C.POINTER(GpMatches), C.c_void_p]),
    "gp_vit_query_sizes": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "gp_vit_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p,
                                C.c_void_p, C.POINTER(C.c_void_p)]),
    "gp_vit_destroy": (C.c_int, [C.c_void_p]),
    "gp_vit_forward": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_launch_count": (C.c_uint64, []),
    "gp_debug_attention_timeline": (C.c_int, [C.c_void_p]),
    "gp_debug_gemm_timeline": (C.c_int, [C.c_void_p]),
    "gp_crop_resize_pad": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_render_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "gp_render_templates": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_ist_trunk_query_sizes":(C.c_int, [C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "gp_ist_trunk_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(C.c_void_p)]),
    "gp_ist_trunk_destroy": (C.c_int, [C.c_void_p]),
    "gp_ist_trunk_forward": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_debug_ist_trunk": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gp_debug_sim_tiles": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gp_debug_gemm": (C.c_int, [C.POINTER(GpDebugGemm), C.c_void_p]),
    "gp_debug_attention": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "gp_normalize_patch_tokens": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_vit_time_linears": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_void_p]),
    "gp_time_sim_kernel": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_void_p]),
}

_lib = None


class GigaPoseNativeError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Loads the shared library (once).  Raises if it has not been built: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GigaPoseNativeError(
            f"{LIB_PATH} not found: build it with `python -m gigapose_b200.build` (nvcc, sm_90a). "
            "gigapose_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError here == the .so does not export the declared ABI
        fn.restype = res
        fn.argtypes = args
    if lib.gp_abi_version() != GP_ABI_VERSION:
        raise GigaPoseNativeError(f"ABI mismatch: library {lib.gp_abi_version()} vs binding {GP_ABI_VERSION}")
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().gp_last_error()
        raise GigaPoseNativeError(f"gigapose_b200 error {status}: {msg.decode() if msg else '?'}")
