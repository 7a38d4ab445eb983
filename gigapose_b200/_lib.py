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
BOP_MAX_TAU = 16               # GP_BOP_MAX_TAU
BOP_MAX_OBJECTS = 256          # GP_BOP_MAX_OBJECTS
BOP_MAX_GT_PER_GROUP = 1024    # GP_BOP_MAX_GT_PER_GROUP
BOP_MAX_RECALL = 128           # GP_BOP_MAX_RECALL
BOP_MATCH_GROUP_BYTES = 32     # GP_BOP_MATCH_GROUP_BYTES
BOP_LABEL_FP, BOP_LABEL_TP, BOP_LABEL_IGNORED = 0, 1, 2          # GP_BOP_LABEL_*
BOP_ADD_CHUNK = 1024           # GP_BOP_ADD_CHUNK
VIS_CROP = 224                 # GP_VIS_CROP
VIS_MAX_SIDE = 16384           # GP_VIS_MAX_SIDE
TSDF_MAX_VOXELS = 1 << 27      # GP_TSDF_MAX_VOXELS


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
                ("qkv_crop_stride", C.c_int32), ("stamp", C.c_int32)]


# gp_debug_gemm_t.mode
GEMM_PLANES, GEMM_PLANES_GELU, GEMM_SCALE_RESIDUAL, GEMM_PATCH_EMBED, GEMM_QKV_HEADS = 0, 1, 2, 3, 4
GEMM_PLANES_RELU, GEMM_PLANES_ADD_RELU, GEMM_ROWS_F32, GEMM_ROWS_F32_RELU = 5, 6, 7, 8


class GpRansacOut(C.Structure):
    _fields_ = [("M", C.c_void_p), ("failed", C.c_void_p), ("inlier_src_pts", C.c_void_p),
                ("inlier_tar_pts", C.c_void_p), ("inlier_scores", C.c_void_p), ("inlier_count", C.c_void_p)]


class GpPredictions(C.Structure):
    _fields_ = [("matches", GpMatches), ("rel_scale", C.c_void_p), ("rel_inplane", C.c_void_p),
                ("ransac", GpRansacOut), ("scores", C.c_void_p), ("poses", C.c_void_p)]


class GpIcpTrace(C.Structure):
    """gp_icp_trace_t: one ICP iteration of one hypothesis (456 bytes; np.dtype(GpIcpTrace) reads an array of them)."""
    _fields_ = [("level", C.c_int32), ("iteration", C.c_int32), ("n", C.c_int32), ("found", C.c_int32),
                ("kept", C.c_int32), ("done", C.c_int32), ("median_bits", C.c_uint32), ("reserved", C.c_int32),
                ("Tf", C.c_float * 12), ("sums", C.c_double * 29), ("xi", C.c_double * 6), ("dT", C.c_double * 12)]


class GpIcpDebug(C.Structure):
    _fields_ = [("counts", C.c_void_p), ("sources", C.c_void_p), ("assoc", C.c_void_p), ("pose0", C.c_void_p),
                ("iterations", C.c_void_p), ("trace", C.c_void_p), ("trace_capacity", C.c_int32),
                ("trace_count", C.c_void_p)]


class GpIcpParams(C.Structure):
    _fields_ = [("unit_per_m", C.c_float), ("min_points", C.c_int32), ("num_levels", C.c_int32),
                ("max_iters", C.c_int32), ("rejection_scale", C.c_float), ("max_residual", C.c_float),
                ("min_step_rad", C.c_float), ("min_step_m", C.c_float), ("debug", GpIcpDebug)]


class GpIcpMaskSet(C.Structure):
    """gp_icp_mask_set_t: the HOST description of the detections of the masked mode."""
    _fields_ = [("n_det", C.c_int32), ("frame", C.POINTER(C.c_int32)), ("boxes", C.POINTER(C.c_int32)),
                ("run_offsets", C.POINTER(C.c_int64))]


# gp_icp_refine statuses (GP_ICP_*)
ICP_OK, ICP_TOO_FEW_POINTS, ICP_DEGENERATE, ICP_RESIDUAL, ICP_INVALID, ICP_LOST = 0, 1, 2, 3, 4, 5


class GpTeaserGnc(C.Structure):
    """gp_teaser_gnc_t: one GNC-TLS iteration of one hypothesis (112 bytes; np.dtype(GpTeaserGnc) reads an array)."""
    _fields_ = [("iteration", C.c_int32), ("members", C.c_int32), ("stopped", C.c_int32), ("reserved", C.c_int32),
                ("mu", C.c_double), ("cost", C.c_double), ("max_residual", C.c_double), ("R", C.c_double * 9)]


class GpTeaserDebug(C.Structure):
    _fields_ = [("counts", C.c_void_p), ("points", C.c_void_p), ("samples", C.c_void_p), ("adjacency", C.c_void_p),
                ("clique", C.c_void_p), ("gnc", C.c_void_p), ("gnc_weights", C.c_void_p),
                ("gnc_capacity", C.c_int32), ("stop_after", C.c_int32), ("transform", C.c_void_p)]


class GpTeaserParams(C.Structure):
    _fields_ = [("unit_per_m", C.c_float), ("min_points", C.c_int32), ("n_points", C.c_int32),
                ("noise_bound", C.c_float), ("cbar2", C.c_float), ("min_inliers", C.c_int32),
                ("gnc_factor", C.c_float), ("gnc_max_iters", C.c_int32), ("gnc_cost_threshold", C.c_double),
                ("clique_budget", C.c_int64), ("debug", GpTeaserDebug)]


# gp_teaser_refine statuses (GP_TEASER_*)
TEASER_OK, TEASER_TOO_FEW_POINTS, TEASER_CLIQUE_TOO_SMALL, TEASER_CLIQUE_BUDGET = 0, 1, 2, 3
TEASER_TOO_FEW_INLIERS, TEASER_INVALID = 4, 5
TEASER_MAX_POINTS = 1024       # GP_TEASER_MAX_POINTS


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
    "gp_crop_resize_pad_rle": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "gp_render_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "gp_render_templates": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_render_depth": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_recentre_boxes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_double),
                                    C.POINTER(C.c_int64), C.c_void_p, C.c_void_p]),
    "gp_recentre_crop": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_double),
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_tsdf_fuse": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_float, C.c_float, C.c_int,
                               C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float),
                               C.c_void_p, C.c_void_p]),
    "gp_tsdf_extract_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "gp_tsdf_extract_count": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_tsdf_extract_emit": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_float, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_bop_vsd":(C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                             C.c_int, C.POINTER(C.c_float), C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_bop_mssd_mspd": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.POINTER(C.c_int32),
                                   C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]),
    "gp_bop_match": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                               C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_bop_average_precision": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p,
                                           C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_double), C.c_void_p,
                                           C.c_void_p]),
    "gp_bop_add": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_int, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_vis_vertex_errors": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_vis_heat_colors": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]),
    "gp_vis_overlay": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "gp_vis_kabsch": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    "gp_icp_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "gp_icp_prepare_scene": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                                       C.c_void_p]),
    "gp_icp_refine": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.POINTER(GpIcpParams), C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_icp_masked_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(GpIcpMaskSet), C.POINTER(C.c_size_t),
                                            C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "gp_icp_masked_decode": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(GpIcpMaskSet), C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "gp_icp_prepare_masked_scene": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(GpIcpMaskSet), C.c_void_p,
                                              C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]),
    "gp_icp_refine_masked": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(GpIcpMaskSet), C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(GpIcpParams),
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "gp_debug_icp_select": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "gp_depth_score": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gp_teaser_query_sizes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "gp_teaser_refine": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.POINTER(GpTeaserParams), C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
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
    "gp_debug_layernorm": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
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


def ptr(t):
    """Device address of a tensor, or None (a NULL pointer) for None."""
    return None if t is None else t.data_ptr()


def cuda_device(device, what: str):
    """torch.device of a CUDA `device` with its index resolved ("cuda" = the current device); refuses anything else."""
    import torch
    device = torch.device(device)
    if device.type != "cuda":
        raise GigaPoseNativeError(f"{what} on CUDA devices only (no CPU fallback)")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def aligned_buffer(nbytes: int, device, zero: bool = False):
    """Caller-owned device memory for the library, which wants its bank / workspace / weight memory 1024-byte aligned
    (the TMA swizzle atoms).  Returns (owner, view): `view` is the `nbytes`-byte slice of `owner` that starts on a
    1024-byte boundary; keep `owner` alive as long as the library holds the address."""
    import torch
    owner = (torch.zeros if zero else torch.empty)(nbytes + 1024, dtype=torch.uint8, device=device)
    off = (-owner.data_ptr()) % 1024
    return owner, owner[off:off + nbytes]
