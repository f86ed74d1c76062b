"""ctypes binding of libvlfm_b200.so (the C-ABI declared in include/vlfm_b200.h).

The product path has NO fallback: if the library is missing or a call fails, we raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvlfm_b200.so")

VLFM_OK = 0
ST_CAMERA_OFF_GRID = 1
ST_SCATTER_OOB = 2
ST_FRONTIER_OVERFLOW = 4
FUSE_WEIGHTED, FUSE_MAX_CONFIDENCE, FUSE_REPLACE, FUSE_EQUAL = 0, 1, 2, 4
EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RESID_F32, EPI_BIAS_F32, EPI_BIAS_RELU_F16 = 0, 1, 2, 3, 4
EPI_BIAS_GELU_F16X2 = 6
EPI_BIAS_SILU_F16 = 7
EPI_CLUSTER_SPLIT = 256      # flag bit of vlfm_gemm_f16's epilogue: the batch-1 ViT cluster-split plan is allowed
DRAW_LINE, DRAW_CIRCLE, DRAW_RECORD_INTS = 0, 1, 8


class ValueParams(C.Structure):
    _fields_ = [
        ("H", C.c_int32), ("W", C.c_int32), ("G", C.c_int32), ("C", C.c_int32), ("R", C.c_int32),
        ("ppm", C.c_int32), ("depth_scale", C.c_float), ("depth_offset", C.c_float),
        ("decision_threshold", C.c_float), ("fusion", C.c_int32), ("rows_per_tile", C.c_int32),
    ]


class ObstacleParams(C.Structure):
    _fields_ = [
        ("H", C.c_int32), ("W", C.c_int32), ("G", C.c_int32), ("ppm", C.c_int32),
        ("depth_scale", C.c_float), ("depth_offset", C.c_float), ("max_depth_f32", C.c_float),
        ("fx", C.c_double), ("fy", C.c_double), ("min_height", C.c_double), ("max_height", C.c_double),
        ("kernel", C.c_int32), ("full_grid", C.c_int32), ("roi_half", C.c_int32),
    ]


class ExploreEnv(C.Structure):
    """VlfmExploreEnv (include/vlfm_b200.h)"""
    _fields_ = [
        ("slot", C.c_int32), ("agent_col", C.c_int32), ("agent_row", C.c_int32), ("frame", C.c_int32 * 4), ("pad", C.c_int32),
        ("heading_deg", C.c_double), ("fov_deg", C.c_double), ("max_line_len", C.c_double), ("area_thresh_px", C.c_double),
    ]


class YoloParams(C.Structure):
    """VlfmYoloParams (include/vlfm_b200.h)"""
    _fields_ = [("conf_thres", C.c_float), ("iou_thres", C.c_float), ("agnostic", C.c_int32), ("pad", C.c_int32),
                ("class_mask", C.c_uint32 * 4)]


_P = C.c_void_p
_SIGNATURES = {
    "vlfm_last_error": (C.c_char_p, []),
    "vlfm_version": (C.c_int, []),
    "vlfm_launch_count": (C.c_ulonglong, []),
    "vlfm_value_workspace_bytes": (C.c_int, [C.POINTER(ValueParams), C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_value_update": (C.c_int, [C.POINTER(ValueParams), C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlfm_value_mask_unexplored": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "vlfm_value_disc_median": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "vlfm_value_disc_median_batch": (C.c_int, [C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "vlfm_obstacle_update": (C.c_int, [C.POINTER(ObstacleParams), C.c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlfm_value_cone_template": (C.c_int, [C.c_double, C.c_double, C.c_int, C.c_double, _P, _P, C.c_size_t, _P]),
    "vlfm_biattn_f16": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P]),
    "vlfm_cast_f32_f16": (C.c_int, [_P, _P, C.c_long, _P]),
    "vlfm_cast_addpos_f16": (C.c_int, [_P, _P, _P, _P, C.c_long, _P]),
    "vlfm_msda_fused": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_holes_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_fill_small_holes": (C.c_int, [_P, C.c_int, C.c_int, C.c_double, _P, _P, _P, _P]),
    "vlfm_gemm_f16": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "vlfm_gemm_csplit_plan": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "vlfm_gemm_f16_resid_ln": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 6 + [_P, _P, _P, C.c_int, _P, C.c_int, C.c_float, _P, C.c_size_t, _P]),
    "vlfm_layernorm_reduce": (C.c_int, [_P, _P, C.c_int, C.c_longlong, _P, _P, _P, _P] + [C.c_int] * 5 + [C.c_float, _P]),
    "vlfm_preprocess_im2col": (C.c_int, [_P, _P, _P] + [C.c_int] * 7 + [_P, _P, C.c_int, _P, _P, C.c_int,
                                         C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "vlfm_assemble_tokens": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "vlfm_layernorm": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P]),
    "vlfm_attention_f16": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 9 + [C.c_float, _P]),
    "vlfm_gemm_f16x2": (C.c_int, [_P] * 7 + [C.c_int] * 7 + [_P]),
    "vlfm_gemm_f16x2_resid_ln": (C.c_int, [_P] * 6 + [C.c_int] * 6 + [_P, _P, _P, _P, C.c_int, _P, C.c_int, C.c_float, _P, C.c_size_t, _P]),
    "vlfm_layernorm_x2": (C.c_int, [_P] * 6 + [C.c_int] * 5 + [C.c_float, _P]),
    "vlfm_layernorm_reduce_x2": (C.c_int, [_P, _P, C.c_int, C.c_longlong, _P, _P, _P, _P, _P] + [C.c_int] * 5 + [C.c_float, _P]),
    "vlfm_split_x2": (C.c_int, [_P, _P, _P, C.c_longlong, _P]),
    "vlfm_attention_f32": (C.c_int, [_P] * 5 + [C.c_int] * 9 + [C.c_float, _P]),
    "vlfm_swin_patch_im2col": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "vlfm_swin_window_attention": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 6 + [_P]),
    "vlfm_swin_patch_merge": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "vlfm_explore_workspace_bytes": (C.c_int, [C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_explore_update": (C.c_int, [C.c_int, _P, _P, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, _P, _P, _P, _P, _P]),
    "vlfm_explore_env_record_bytes": (C.c_size_t, []),
    "vlfm_explore_batch_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_explore_update_batch": (C.c_int, [C.c_int, C.c_int, C.POINTER(ExploreEnv), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, C.c_size_t, _P]),
    "vlfm_explore_prepare_batch": (C.c_int, [C.c_int, C.c_int, C.POINTER(ExploreEnv), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, C.c_size_t]),
    "vlfm_explore_launch_batch": (C.c_int, [C.c_int, C.c_int, _P, _P, _P]),
    "vlfm_holes_batch_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_fill_small_holes_batch": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_double, _P, _P, C.c_size_t, _P, _P, C.c_size_t, _P]),
    "vlfm_itc_head": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "vlfm_itc_head_multi": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "vlfm_im2col_f16": (C.c_int, [_P, C.c_int, _P] + [C.c_int] * 7 + [_P]),
    "vlfm_groupnorm_rows": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, C.c_float, _P, C.c_int, C.c_int, _P]),
    "vlfm_mask_rows_f16": (C.c_int, [_P, _P, _P, C.c_long, C.c_int, _P]),
    "vlfm_proposal_scores": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_topk_rows": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_decoder_query_pos": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "vlfm_gather_rows": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_box_finish": (C.c_int, [_P, _P, _P, C.c_long, _P]),
    "vlfm_contrastive_sigmoid": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_object_cloud_extract": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_double, C.c_double, _P, C.c_int, _P, _P,
                                            C.c_size_t, _P]),
    "vlfm_dbscan_workspace_bytes": (C.c_int, [C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_dbscan_largest_cluster": (C.c_int, [_P, _P, C.c_int, C.c_double, C.c_int, _P, _P, _P, _P, C.c_size_t, _P]),
    "vlfm_render_workspace_bytes": (C.c_int, [C.c_int, C.POINTER(C.c_size_t)]),
    "vlfm_render_value": (C.c_int, [C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, C.c_size_t, _P]),
    "vlfm_render_obstacle": (C.c_int, [C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "vlfm_render_draw": (C.c_int, [C.c_int, C.c_int, _P, _P, C.c_size_t, _P, C.c_size_t, _P]),
    "vlfm_sam_preprocess": (C.c_int, [_P, _P, _P] + [C.c_int] * 6 + [_P, _P, C.c_int, _P, _P, C.c_int, C.c_int,
                                      C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "vlfm_sam_dwconv3x3": (C.c_int, [_P, C.c_int, _P, _P, _P] + [C.c_int] * 7 + [_P]),
    "vlfm_sam_add_act": (C.c_int, [_P, _P, _P, _P, C.c_longlong, C.c_int, _P]),
    "vlfm_sam_window_attention": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 6 + [C.c_float, _P]),
    "vlfm_sam_box_tokens": (C.c_int, [_P] + [C.c_int] * 6 + [_P, _P, _P, C.c_int, _P]),
    "vlfm_sam_add_pe_f16": (C.c_int, [_P, _P, _P, _P, C.c_longlong, C.c_longlong, C.c_int, _P]),
    "vlfm_sam_decoder_init": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 4 + [_P]),
    "vlfm_sam_t2i_attention": (C.c_int, [_P, _P, _P, _P] + [C.c_int] * 8 + [C.c_float, _P, C.c_size_t, _P]),
    "vlfm_sam_pixel_shuffle2": (C.c_int, [_P, _P] + [C.c_int] * 4 + [_P]),
    "vlfm_sam_mask_logits": (C.c_int, [_P, _P, _P] + [C.c_int] * 4 + [_P]),
    "vlfm_sam_mask_finish": (C.c_int, [_P, _P] + [C.c_int] * 7 + [_P]),
    "vlfm_pointnav_depth_in": (C.c_int, [_P] + [C.c_int] * 5 + [_P, C.c_int, _P, _P]),
    "vlfm_pointnav_groupnorm": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, _P, _P] + [C.c_int] * 4 + [C.c_float, C.c_int, _P]),
    "vlfm_pointnav_maxpool3s2": (C.c_int, [_P, _P, _P] + [C.c_int] * 4 + [_P]),
    "vlfm_pointnav_gemv_f32": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P] + [C.c_int] * 5 + [_P]),
    "vlfm_pointnav_lstm_prep": (C.c_int, [_P, _P, _P, C.c_int] + [_P] * 9 + [C.c_int, _P]),
    "vlfm_pointnav_lstm_cell": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "vlfm_pointnav_lstm_head": (C.c_int, [_P] * 5 + [C.c_int] + [_P] * 6 + [C.c_int, _P]),
    "vlfm_yolo_preprocess": (C.c_int, [_P, _P] + [C.c_int] * 5 + [_P] * 7),
    "vlfm_yolo_maxpool2": (C.c_int, [_P, C.c_int, _P] + [C.c_int] * 5 + [_P]),
    "vlfm_yolo_spp_pools": (C.c_int, [_P, C.c_int, _P] + [C.c_int] * 5 + [_P]),
    "vlfm_yolo_upsample2": (C.c_int, [_P, C.c_int, _P] + [C.c_int] * 5 + [_P]),
    "vlfm_yolo_add": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_longlong, C.c_int, _P]),
    "vlfm_yolo_decode": (C.c_int, [_P] + [C.c_int] * 6 + [_P, C.c_float, C.c_int, C.c_int, _P, _P, _P, _P]),
    "vlfm_yolo_sort": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "vlfm_yolo_nms": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P]),
    "vlfm_yolo_boxes": (C.c_int, [_P, _P, _P] + [C.c_int] * 3 + [C.c_float] * 3 + [C.c_int] * 2 + [_P] * 5),
}

_lib = None


class VlfmError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the C-ABI library; raise loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VlfmError(
                f"{LIB_PATH} is missing: build it with `python -m vlfm_b200.build` "
                "(or __graft_entry__.build()). There is no CPU fallback."
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def declared_symbols():
    return list(_SIGNATURES)


def check(rc: int, what: str) -> None:
    if rc != VLFM_OK:
        raise VlfmError(f"{what} failed (code {rc}): {load().vlfm_last_error().decode()}")


def ptr(t) -> int:
    """Device (or host) address of a torch tensor, or None."""
    return None if t is None else t.data_ptr()


def stream_ptr():
    import torch

    return torch.cuda.current_stream().cuda_stream


def launch_count() -> int:
    return int(load().vlfm_launch_count())
