"""ctypes binding of libyolort_b200.so (the C ABI declared in include/yolort_b200.h).

PyTorch is used here only as the owner of device memory and streams: every wrapper hands raw
`data_ptr()`s and the current CUDA stream to the native library.  There is no fallback: if the
library is missing, or a wrapper is asked to run without a CUDA device, it raises.
"""
import ctypes
import itertools
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# YB_LIB_PATH: A/B timing of alternative builds of the same ABI (scripts/ab_step.py); never set in product use
LIB_PATH = os.environ.get("YB_LIB_PATH") or os.path.join(_HERE, "libyolort_b200.so")

YB_U8, YB_F16, YB_BF16, YB_F32, YB_F8E4M3 = 0, 1, 2, 3, 4
YB_LAYOUT_NCHW, YB_LAYOUT_S2D16 = 0, 1
YB_OP_CONV, YB_OP_SPP_POOL, YB_OP_UPSAMPLE2X, YB_OP_ATTENTION, YB_OP_DWCONV, YB_OP_SE, YB_OP_AVGPOOL = 0, 1, 2, 3, 4, 5, 6
YB_OP_QUANTIZE = 7
YB_ACT_NONE, YB_ACT_SILU, YB_ACT_HARDSWISH, YB_ACT_LEAKY01, YB_ACT_RELU = 0, 1, 2, 3, 4
# yb_op_desc.reserved option bits of a convolution (fp16 / bf16; e4m3 convolutions take the last two only)
YB_CONV_FORCE_IM2COL, YB_CONV_BAND_STEM, YB_CONV_FORCE_PLANES, YB_CONV_NO_NSPLIT, YB_CONV_ONE_CTA = 1, 2, 4, 8, 16
YB_CONV_NO_TAIL_SPLIT = 64
YB_CONV_PAIR_N64 = 128
YB_CONV_NO_TEAMS = 256
YB_CONV_E4M3_F16_OUT, YB_CONV_E4M3_BF16_OUT = 16, 32
YB_CONV_KERNEL_IM2COL, YB_CONV_KERNEL_PATCH, YB_CONV_KERNEL_E4M3 = 0, 1, 2
PATCH_TILINGS = {1: "classic", 2: "wrap", 3: "stride2"}      # yb_conv_info.tiling of the halo-patch kernel
YB_MAX_LEVELS, YB_MAX_ANCHORS = 4, 4
NMS_TV_AUTO, NMS_EXACT_PER_CLASS, NMS_OFFSET_TRICK = 0, 1, 2

# every symbol include/yolort_b200.h declares (tests check that the built library exports all of them)
EXPORTED_SYMBOLS = (
    "yb_last_error",
    "yb_abi_version",
    "yb_letterbox_geometry",
    "yb_letterbox",
    "yb_letterbox_strided",
    "yb_canvas_rescale",
    "yb_scale_coords_params",
    "yb_conv_chain_supported",
    "yb_conv_config",
    "yb_plan_create",
    "yb_plan_run",
    "yb_plan_run_range",
    "yb_plan_num_launches",
    "yb_plan_destroy",
    "yb_decode_nms_workspace_bytes",
    "yb_decode_nms_debug_offset",
    "yb_decode_nms",
    "yb_decode_dense",
    "yb_decode_nms_tta_workspace_bytes",
    "yb_decode_nms_tta",
    "yb_nms_layout",
    "yb_nms_begin",
    "yb_nms_finish",
    "yb_decode_candidates",
    "yb_batched_nms_workspace_bytes",
    "yb_batched_nms",
    "yb_jpeg_parse",
    "yb_jpeg_workspace_bytes",
    "yb_jpeg_decode",
    "yb_coco_append",
    "yb_coco_evaluate_workspace_bytes",
    "yb_coco_evaluate",
    "yb_yolo_loss_workspace_bytes",
    "yb_yolo_loss_layout",
    "yb_yolo_loss_forward",
    "yb_yolo_loss_backward",
    "yb_augment_prepare",
    "yb_augment",
    "yb_augment_sample",
    "yb_v5_augment_prepare",
    "yb_v5_augment",
    "yb_v5_mixup",
    "yb_v5_resize_prepare",
    "yb_v5_resize",
    "yb_v5_resize_area_prepare",
    "yb_v5_resize_area",
    "yb_v5_compose_prepare",
    "yb_v5_compose",
    "yb_v5_rescale_coords",
    "yb_conv_wgrad_workspace_bytes",
    "yb_conv_wgrad_config",
    "yb_conv_wgrad",
    "yb_anchor_metric",
    "yb_kmeans_workspace_bytes",
    "yb_kmeans",
    "yb_anchor_evolve",
    "yb_v5m_match_workspace_bytes",
    "yb_v5m_match",
    "yb_v5m_ap_workspace_bytes",
    "yb_v5m_ap",
)


class LetterboxGeom(ctypes.Structure):
    _fields_ = [
        ("src_h", ctypes.c_int32), ("src_w", ctypes.c_int32),
        ("new_h", ctypes.c_int32), ("new_w", ctypes.c_int32),
        ("top", ctypes.c_int32), ("left", ctypes.c_int32),
        ("ratio_h", ctypes.c_float), ("ratio_w", ctypes.c_float),
    ]


class OpDesc(ctypes.Structure):
    _fields_ = [
        ("kind", ctypes.c_int32), ("dtype", ctypes.c_int32),
        ("N", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("Cin", ctypes.c_int32), ("in_cstride", ctypes.c_int32),
        ("in_", ctypes.c_void_p),
        ("Ho", ctypes.c_int32), ("Wo", ctypes.c_int32),
        ("Cout", ctypes.c_int32), ("out_cstride", ctypes.c_int32),
        ("out", ctypes.c_void_p),
        ("ksize", ctypes.c_int32), ("stride", ctypes.c_int32), ("pad", ctypes.c_int32),
        ("act", ctypes.c_int32),
        ("weight", ctypes.c_void_p),
        ("Cin_pad", ctypes.c_int32), ("Cout_pad", ctypes.c_int32),
        ("bias", ctypes.c_void_p),
        ("residual", ctypes.c_void_p),
        ("res_cstride", ctypes.c_int32), ("reserved", ctypes.c_int32),
        ("decode", ctypes.c_void_p),
        ("chain", ctypes.c_void_p),
    ]


class ConvChain(ctypes.Structure):
    """yb_conv_chain: the pointwise tail fused onto a convolution (include/yolort_b200.h)."""
    _fields_ = [
        ("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p),
        ("Cout", ctypes.c_int32), ("Cout_pad", ctypes.c_int32), ("K_pad", ctypes.c_int32),
        ("act", ctypes.c_int32),
        ("out", ctypes.c_void_p), ("out_cstride", ctypes.c_int32),
        ("own_C", ctypes.c_int32),
        ("extra", ctypes.c_void_p), ("extra_C", ctypes.c_int32), ("extra_cstride", ctypes.c_int32),
        ("store_first", ctypes.c_int32),
    ]


class ConvInfo(ctypes.Structure):
    """yb_conv_info: how a convolution is launched (include/yolort_b200.h)."""
    _fields_ = [(name, ctypes.c_int32) for name in (
        "kernel", "block_n", "n_tiles", "weights_resident", "tiles_per_pass", "slots", "ring", "store_cols", "store_bufs",
        "groups", "resident_ctas", "chained", "smem_bytes", "grid", "tiling", "m_tiles", "work_items", "tail_n",
        "tail_tiles", "tail_split")]


class HeadDecode(ctypes.Structure):
    _fields_ = [
        ("n_anchors", ctypes.c_int32), ("n_classes", ctypes.c_int32),
        ("level_start", ctypes.c_int32), ("anchors_per_image", ctypes.c_int32),
        ("stride_px", ctypes.c_float), ("anchors_px", ctypes.c_float * 8),
        ("score_thresh", ctypes.c_float),
        ("cap_per_image", ctypes.c_int64),
        ("keys", ctypes.c_void_p), ("boxes", ctypes.c_void_p),
        ("img_count", ctypes.c_void_p), ("img_maxc", ctypes.c_void_p),
    ]


class NmsLayout(ctypes.Structure):
    _fields_ = [
        ("keys", ctypes.c_void_p), ("boxes", ctypes.c_void_p),
        ("img_count", ctypes.c_void_p), ("img_maxc", ctypes.c_void_p),
        ("cap_per_image", ctypes.c_int64), ("anchors_per_image", ctypes.c_int32),
        ("level_start", ctypes.c_int32 * YB_MAX_LEVELS),
    ]


class HeadLevel(ctypes.Structure):
    _fields_ = [
        ("logits", ctypes.c_void_p), ("dtype", ctypes.c_int32),
        ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("stride_n", ctypes.c_int64), ("stride_a", ctypes.c_int64),
        ("stride_y", ctypes.c_int64), ("stride_x", ctypes.c_int64),
        ("stride_px", ctypes.c_float),
        ("anchors_px", ctypes.c_float * (2 * YB_MAX_ANCHORS)),
    ]


YB_TTA_MAX_PASSES = 3


class TtaPass(ctypes.Structure):
    _fields_ = [
        ("n_levels", ctypes.c_int32), ("flip_lr", ctypes.c_int32),
        ("scale", ctypes.c_float), ("canvas_w", ctypes.c_float),
        ("levels", HeadLevel * YB_MAX_LEVELS),
    ]


class NmsParams(ctypes.Structure):
    _fields_ = [
        ("n_images", ctypes.c_int32), ("n_levels", ctypes.c_int32),
        ("n_anchors", ctypes.c_int32), ("n_classes", ctypes.c_int32),
        ("score_thresh", ctypes.c_float), ("iou_thresh", ctypes.c_float),
        ("max_det", ctypes.c_int32), ("semantics", ctypes.c_int32),
        ("max_candidates", ctypes.c_int64),
    ]


class JpegInfo(ctypes.Structure):
    """yb_jpeg_info: what yb_jpeg_parse reads from a file's markers (include/yolort_b200.h)."""
    _fields_ = [
        ("supported", ctypes.c_int32), ("reason", ctypes.c_char * 92),
        ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("ncomp", ctypes.c_int32),
        ("h_samp", ctypes.c_int32 * 3), ("v_samp", ctypes.c_int32 * 3),
        ("restart_interval", ctypes.c_int32),
        ("mcus_x", ctypes.c_int32), ("mcus_y", ctypes.c_int32), ("blocks_per_mcu", ctypes.c_int32),
        ("scan_begin", ctypes.c_int64), ("scan_end", ctypes.c_int64), ("data_offset", ctypes.c_int64),
        ("quant", (ctypes.c_uint16 * 64) * 3),
        ("dc_bits", (ctypes.c_uint8 * 16) * 3), ("ac_bits", (ctypes.c_uint8 * 16) * 3),
        ("dc_vals", (ctypes.c_uint8 * 16) * 3),
        ("ac_vals", (ctypes.c_uint8 * 256) * 3),
    ]


YB_JPEG_ST_HUFFMAN, YB_JPEG_ST_COEF, YB_JPEG_ST_TRUNCATED, YB_JPEG_ST_RESTART, YB_JPEG_ST_RANGE = 1, 2, 4, 8, 16


class CocoGt(ctypes.Structure):
    """yb_coco_gt: an annotation file's GT in the layout the evaluation kernels read (include/yolort_b200.h)."""
    _fields_ = [
        ("n_images", ctypes.c_int32), ("n_categories", ctypes.c_int32), ("n_gt", ctypes.c_int32),
        ("max_gt_per_pair", ctypes.c_int32),
        ("img_start", ctypes.c_void_p), ("gt_img", ctypes.c_void_p), ("gt_cat", ctypes.c_void_p),
        ("gt_box", ctypes.c_void_p), ("gt_area", ctypes.c_void_p), ("gt_flags", ctypes.c_void_p),
    ]


YB_COCO_GT_CROWD, YB_COCO_GT_ID_NONZERO = 1, 2
YB_COCO_ST_UNKNOWN_IMAGE, YB_COCO_ST_BAD_LABEL = 1, 2
YB_COCO_ROW_DROPPED, YB_COCO_RECORD_INT32, YB_COCO_NUM_PARAMS = -2, 8, 119


class LossLevel(ctypes.Structure):
    """yb_loss_level: one head output of the training loss (include/yolort_b200.h)."""
    _fields_ = [
        ("logits", ctypes.c_void_p), ("dtype", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("stride_px", ctypes.c_float), ("anchors_px", ctypes.c_float * (2 * YB_MAX_ANCHORS)),
    ]


class YoloLossParams(ctypes.Structure):
    """yb_yolo_loss_params: SetCriterion's hyperparameters (include/yolort_b200.h)."""
    _fields_ = [
        ("n_images", ctypes.c_int32), ("n_levels", ctypes.c_int32), ("n_anchors", ctypes.c_int32),
        ("n_classes", ctypes.c_int32),
        ("box_gain", ctypes.c_float), ("cls_gain", ctypes.c_float), ("obj_gain", ctypes.c_float),
        ("cls_pos", ctypes.c_float), ("obj_pos", ctypes.c_float), ("anchor_thresh", ctypes.c_float),
        ("smooth_pos", ctypes.c_float), ("smooth_neg", ctypes.c_float), ("gr", ctypes.c_float),
        ("balance", ctypes.c_float * YB_MAX_LEVELS),
    ]


YB_LOSS_ST_IMAGE, YB_LOSS_ST_CLASS, YB_LOSS_ST_NONFINITE = 1, 2, 4
YB_AUG_MAX_OPS, YB_AUG_MAX_CONTRAST = 16, 4
(YB_AUG_BRIGHTNESS, YB_AUG_CONTRAST, YB_AUG_SATURATION, YB_AUG_HUE, YB_AUG_PERMUTE, YB_AUG_ZOOM_OUT, YB_AUG_CROP,
 YB_AUG_HFLIP) = range(1, 9)


class AugOp(ctypes.Structure):
    """yb_aug_op: one op of an image's augmentation recipe (include/yolort_b200.h)."""
    _fields_ = [("kind", ctypes.c_int32), ("arg", ctypes.c_int32 * 7), ("factor", ctypes.c_float),
                ("one_minus", ctypes.c_float)]


class AugImage(ctypes.Structure):
    """yb_aug_image: one image, its recipe and where its output goes (include/yolort_b200.h)."""
    _fields_ = [
        ("src", ctypes.c_void_p), ("stride_c", ctypes.c_int64), ("stride_y", ctypes.c_int64),
        ("stride_x", ctypes.c_int64),
        ("src_h", ctypes.c_int32), ("src_w", ctypes.c_int32), ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32),
        ("out_offset", ctypes.c_int64), ("n_ops", ctypes.c_int32), ("n_contrast", ctypes.c_int32),
        ("out_block_start", ctypes.c_int32), ("mean_block_start", ctypes.c_int32 * YB_AUG_MAX_CONTRAST),
        ("reserved", ctypes.c_int32), ("ops", AugOp * YB_AUG_MAX_OPS),
    ]


YB_AUG_MAX_TRANSFORMS, YB_AUG_MAX_OPTIONS, YB_AUG_CROP_ROUNDS = 16, 16, 1024
YB_AUG_S_NONE, YB_AUG_S_PHOTOMETRIC, YB_AUG_S_ZOOM_OUT, YB_AUG_S_IOU_CROP, YB_AUG_S_HFLIP = range(5)
YB_AUG_ST_CROP_ROUNDS = 1


class AugSampler(ctypes.Structure):
    """yb_aug_sampler: one transform of the device parameter sampler (include/yolort_b200.h)."""
    _fields_ = [
        ("kind", ctypes.c_int32), ("jitter", ctypes.c_int32), ("trials", ctypes.c_int32), ("n_options", ctypes.c_int32),
        ("fill", ctypes.c_uint32), ("p", ctypes.c_float), ("lo", ctypes.c_float * 4), ("span", ctypes.c_float * 4),
        ("min_aspect", ctypes.c_double), ("max_aspect", ctypes.c_double),
        ("options", ctypes.c_double * YB_AUG_MAX_OPTIONS),
    ]
YB_LOSS_MATCH_INT32 = 24
YB_WGRAD_MAX_PROBLEMS = 8


YB_V5_MAX_RECTS = 31
(YB_V5_AFFINE, YB_V5_PERSPECTIVE, YB_V5_TO_HSV, YB_V5_LUT, YB_V5_FROM_HSV, YB_V5_RGB, YB_V5_FLIP_LR,
 YB_V5_FLIP_UD) = (1 << k for k in range(8))


class V5Image(ctypes.Structure):
    """yb_v5_image: one image of the YOLOv5 augmentation kernel (include/yolort_b200.h)."""
    _fields_ = [
        ("src", ctypes.c_void_p), ("dst", ctypes.c_void_p),
        ("src_stride_y", ctypes.c_int64), ("src_stride_x", ctypes.c_int64), ("src_stride_c", ctypes.c_int64),
        ("dst_stride_y", ctypes.c_int64), ("dst_stride_x", ctypes.c_int64), ("dst_stride_c", ctypes.c_int64),
        ("src_h", ctypes.c_int32), ("src_w", ctypes.c_int32), ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32),
        ("ops", ctypes.c_int32), ("n_rects", ctypes.c_int32), ("block_start", ctypes.c_int32),
        ("reserved", ctypes.c_int32), ("inv", ctypes.c_double * 9),
        ("rects", (ctypes.c_int32 * 4) * YB_V5_MAX_RECTS), ("rect_color", ctypes.c_uint32 * YB_V5_MAX_RECTS),
        ("lut", (ctypes.c_uint8 * 256) * 3),
    ]


YB_V5_MAX_PLACES = 4


class V5ResizeJob(ctypes.Structure):
    """yb_v5_resize_job: one cv2.resize(INTER_LINEAR or INTER_AREA) of load_image (include/yolort_b200.h)."""
    _fields_ = [
        ("src", ctypes.c_void_p), ("dst", ctypes.c_void_p),
        ("src_stride_y", ctypes.c_int64), ("src_stride_x", ctypes.c_int64), ("src_stride_c", ctypes.c_int64),
        ("src_h", ctypes.c_int32), ("src_w", ctypes.c_int32), ("dst_h", ctypes.c_int32), ("dst_w", ctypes.c_int32),
        ("block_start", ctypes.c_int32), ("reserved", ctypes.c_int32),
    ]


class V5Place(ctypes.Structure):
    """yb_v5_place: one image placed on a virtual canvas (include/yolort_b200.h)."""
    _fields_ = [
        ("src", ctypes.c_void_p),
        ("stride_y", ctypes.c_int64), ("stride_x", ctypes.c_int64), ("stride_c", ctypes.c_int64),
        ("y0", ctypes.c_int32), ("x0", ctypes.c_int32), ("y1", ctypes.c_int32), ("x1", ctypes.c_int32),
        ("oy", ctypes.c_int32), ("ox", ctypes.c_int32),
    ]


class V5Canvas(ctypes.Structure):
    """yb_v5_canvas: a virtual canvas and its inverse warp (include/yolort_b200.h)."""
    _fields_ = [
        ("inv", ctypes.c_double * 9), ("warp", ctypes.c_int32), ("n_places", ctypes.c_int32),
        ("places", V5Place * YB_V5_MAX_PLACES),
    ]


class V5Sample(ctypes.Structure):
    """yb_v5_sample: one training sample of the compose kernel (include/yolort_b200.h)."""
    _fields_ = [
        ("dst", ctypes.c_void_p),
        ("dst_stride_y", ctypes.c_int64), ("dst_stride_x", ctypes.c_int64), ("dst_stride_c", ctypes.c_int64),
        ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32), ("ops", ctypes.c_int32), ("n_canvases", ctypes.c_int32),
        ("mix_r", ctypes.c_double), ("mix_omr", ctypes.c_double), ("canvas", V5Canvas * 2),
        ("lut", (ctypes.c_uint8 * 256) * 3),
    ]


class V5Rescale(ctypes.Structure):
    """yb_v5_rescale: val.py's scale_coords / clip_coords of one batch (include/yolort_b200.h)."""
    _fields_ = [
        ("boxes", ctypes.c_void_p), ("counts", ctypes.c_void_p), ("targets", ctypes.c_void_p),
        ("targets_out", ctypes.c_void_p), ("params", ctypes.c_void_p), ("n", ctypes.c_int32), ("D", ctypes.c_int32),
        ("T", ctypes.c_int64), ("canvas_w", ctypes.c_float), ("canvas_h", ctypes.c_float),
    ]


class WgradProblem(ctypes.Structure):
    """yb_wgrad_problem: one 1x1-convolution weight gradient (include/yolort_b200.h)."""
    _fields_ = [
        ("dtype", ctypes.c_int32), ("out_dtype", ctypes.c_int32), ("P", ctypes.c_int64), ("Cout", ctypes.c_int32),
        ("Cin", ctypes.c_int32), ("dy", ctypes.c_void_p), ("dy_stride", ctypes.c_int64), ("x", ctypes.c_void_p),
        ("x_stride", ctypes.c_int64), ("dw", ctypes.c_void_p), ("db", ctypes.c_void_p),
    ]


_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load (once) the native library; raise loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} is missing. Build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "yolort_b200 has no PyTorch/CPU fallback path."
        )
    L = ctypes.CDLL(LIB_PATH)
    L.yb_last_error.restype = ctypes.c_char_p
    L.yb_abi_version.restype = ctypes.c_int
    L.yb_letterbox_geometry.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_int32), ctypes.c_float, ctypes.c_float, ctypes.c_int,
        ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(LetterboxGeom), ctypes.POINTER(ctypes.c_int32)]
    L.yb_letterbox.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(LetterboxGeom),
        ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]
    L.yb_letterbox_strided.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.POINTER(LetterboxGeom),
        ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]
    L.yb_scale_coords_params.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.POINTER(ctypes.c_float)]
    L.yb_plan_create.argtypes = [ctypes.POINTER(OpDesc), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    L.yb_conv_chain_supported.argtypes = [ctypes.POINTER(OpDesc)]
    L.yb_conv_config.argtypes = [ctypes.POINTER(OpDesc), ctypes.POINTER(ConvInfo)]
    L.yb_plan_run.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.yb_plan_run_range.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.yb_plan_num_launches.argtypes = [ctypes.c_void_p]
    L.yb_plan_destroy.argtypes = [ctypes.c_void_p]
    L.yb_decode_nms_workspace_bytes.restype = ctypes.c_size_t
    L.yb_decode_nms_workspace_bytes.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel)]
    L.yb_decode_nms_debug_offset.restype = ctypes.c_size_t
    L.yb_decode_nms_debug_offset.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel)]
    L.yb_decode_nms.argtypes = [
        ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_size_t, ctypes.c_void_p]
    L.yb_canvas_rescale.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_int] * 5 + [
        ctypes.c_float, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.yb_decode_nms_tta_workspace_bytes.restype = ctypes.c_size_t
    L.yb_decode_nms_tta_workspace_bytes.argtypes = [ctypes.POINTER(NmsParams), ctypes.c_int, ctypes.POINTER(TtaPass)]
    L.yb_decode_nms_tta.argtypes = [ctypes.POINTER(NmsParams), ctypes.c_int, ctypes.POINTER(TtaPass)] + \
        [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_void_p]
    L.yb_decode_dense.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p,
                                  ctypes.c_void_p, ctypes.c_void_p]
    L.yb_nms_layout.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_size_t,
                                ctypes.POINTER(NmsLayout)]
    L.yb_nms_begin.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
                               ctypes.c_size_t, ctypes.c_void_p]
    L.yb_nms_finish.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                ctypes.c_size_t, ctypes.c_void_p]
    L.yb_decode_candidates.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_size_t,
                                       ctypes.c_void_p]
    L.yb_batched_nms_workspace_bytes.restype = ctypes.c_size_t
    L.yb_batched_nms_workspace_bytes.argtypes = [ctypes.c_int64]
    L.yb_batched_nms.argtypes = [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int,
        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.yb_jpeg_parse.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(JpegInfo)]
    L.yb_jpeg_workspace_bytes.restype = ctypes.c_size_t
    L.yb_jpeg_workspace_bytes.argtypes = [ctypes.c_int, ctypes.POINTER(JpegInfo)]
    L.yb_jpeg_decode.argtypes = [ctypes.c_int, ctypes.POINTER(JpegInfo), ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p),
                                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.yb_coco_append.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_int32] + \
        [ctypes.c_void_p] * 3
    L.yb_coco_evaluate_workspace_bytes.restype = ctypes.c_size_t
    L.yb_coco_evaluate_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.POINTER(CocoGt)]
    L.yb_coco_evaluate.argtypes = [ctypes.POINTER(CocoGt), ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 6 + \
        [ctypes.c_size_t, ctypes.c_void_p]
    L.yb_yolo_loss_workspace_bytes.restype = ctypes.c_size_t
    L.yb_yolo_loss_workspace_bytes.argtypes = [ctypes.POINTER(YoloLossParams), ctypes.POINTER(LossLevel), ctypes.c_int64]
    L.yb_yolo_loss_layout.argtypes = [ctypes.POINTER(YoloLossParams), ctypes.POINTER(LossLevel), ctypes.c_int64,
                                      ctypes.POINTER(ctypes.c_int64)]
    L.yb_yolo_loss_forward.argtypes = [ctypes.POINTER(YoloLossParams), ctypes.POINTER(LossLevel), ctypes.c_void_p,
                                       ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                       ctypes.c_void_p]
    L.yb_yolo_loss_backward.argtypes = [ctypes.POINTER(YoloLossParams), ctypes.POINTER(LossLevel), ctypes.c_int64,
                                        ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p,
                                        ctypes.c_size_t, ctypes.c_void_p]
    L.yb_augment_prepare.argtypes = [ctypes.c_int, ctypes.POINTER(AugImage), ctypes.POINTER(ctypes.c_int64)]
    L.yb_augment.argtypes = [ctypes.c_int, ctypes.POINTER(AugImage), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                             ctypes.c_void_p, ctypes.c_void_p]
    L.yb_augment_sample.argtypes = [ctypes.c_int, ctypes.POINTER(AugSampler), ctypes.c_int] + [ctypes.c_void_p] * 10
    L.yb_v5_augment_prepare.argtypes = [ctypes.c_int, ctypes.POINTER(V5Image), ctypes.POINTER(ctypes.c_int64)]
    L.yb_v5_augment.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    L.yb_v5_mixup.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_double,
                              ctypes.c_void_p]
    L.yb_v5_resize_prepare.argtypes = [ctypes.c_int, ctypes.POINTER(V5ResizeJob), ctypes.POINTER(ctypes.c_int64)]
    L.yb_v5_resize.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    L.yb_v5_resize_area_prepare.argtypes = [ctypes.c_int, ctypes.POINTER(V5ResizeJob), ctypes.POINTER(ctypes.c_int64)]
    L.yb_v5_resize_area.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    L.yb_v5_rescale_coords.argtypes = [ctypes.POINTER(V5Rescale), ctypes.c_void_p]
    L.yb_v5_compose_prepare.argtypes = [ctypes.c_int, ctypes.POINTER(V5Sample), ctypes.POINTER(ctypes.c_int64)]
    L.yb_v5_compose.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    L.yb_conv_wgrad_workspace_bytes.restype = ctypes.c_size_t
    L.yb_conv_wgrad_workspace_bytes.argtypes = [ctypes.POINTER(WgradProblem), ctypes.c_int]
    L.yb_conv_wgrad_config.argtypes = [ctypes.POINTER(WgradProblem), ctypes.c_int, ctypes.POINTER(ctypes.c_int32)]
    L.yb_conv_wgrad.argtypes = [ctypes.POINTER(WgradProblem), ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                ctypes.c_void_p]
    L.yb_anchor_metric.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                   ctypes.c_void_p]
    L.yb_kmeans_workspace_bytes.restype = ctypes.c_size_t
    L.yb_kmeans_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int]
    L.yb_kmeans.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_double,
                            ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                            ctypes.POINTER(ctypes.c_int32), ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.yb_anchor_evolve.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.yb_v5m_match_workspace_bytes.restype = ctypes.c_size_t
    L.yb_v5m_match_workspace_bytes.argtypes = [ctypes.c_int]
    L.yb_v5m_match.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 5 + [ctypes.c_int] + \
        [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int] + \
        [ctypes.c_void_p] * 5 + [ctypes.c_size_t, ctypes.c_void_p]
    L.yb_v5m_ap_workspace_bytes.restype = ctypes.c_size_t
    L.yb_v5m_ap_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int]
    L.yb_v5m_ap.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 7 + \
        [ctypes.c_size_t, ctypes.c_void_p]
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().yb_last_error().decode("utf-8", "replace")
        raise NativeLibraryError(f"{what} failed (status {rc}): {msg}")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return {torch.uint8: YB_U8, torch.float16: YB_F16, torch.bfloat16: YB_BF16, torch.float32: YB_F32,
                torch.float8_e4m3fn: YB_F8E4M3}[dt]
    except KeyError:
        raise NativeLibraryError(f"unsupported tensor dtype {dt}") from None


def current_stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class _NoGuard:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


_NO_GUARD = _NoGuard()


def device_guard(device: torch.device):
    """Context manager that makes `device` the current CUDA device for the native launches inside it (the kernels are
    launched on `device`'s current stream, which must belong to the current device: the reference works on any
    device, and so does this path).  Free when `device` already is current."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if torch.cuda.current_device() == idx:
        return _NO_GUARD
    return torch.cuda.device(idx)


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise NativeLibraryError(
            f"{what}: tensor lives on {t.device}; the yolort_b200 path runs on sm_90a only (no CPU fallback)")


# ---------------------------------------------------------------------------------------------------
# letterbox
# ---------------------------------------------------------------------------------------------------
def letterbox_geometry(sizes: Sequence[Tuple[int, int]], min_size: float, max_size: float,
                       size_divisible: int = 32, fixed_shape: Optional[Tuple[int, int]] = None):
    """Host-only geometry of the letterbox (transform.py:53-97, :297-330). Returns (geoms, (Hb, Wb))."""
    n = len(sizes)
    hw = (ctypes.c_int32 * (2 * n))(*[int(v) for s in sizes for v in s])
    geoms = (LetterboxGeom * n)()
    bhw = (ctypes.c_int32 * 2)()
    fs = None
    if fixed_shape is not None:
        fs = (ctypes.c_int32 * 2)(int(fixed_shape[0]), int(fixed_shape[1]))
    check(lib().yb_letterbox_geometry(n, hw, float(min_size), float(max_size), int(size_divisible), fs, geoms, bhw),
          "yb_letterbox_geometry")
    return geoms, (int(bhw[0]), int(bhw[1]))


def scale_coords_params(Hb: int, Wb: int, h: int, w: int) -> Tuple[float, float, float]:
    out = (ctypes.c_float * 3)()
    check(lib().yb_scale_coords_params(int(Hb), int(Wb), int(h), int(w), out), "yb_scale_coords_params")
    return float(out[0]), float(out[1]), float(out[2])


_u8_lut: Dict[torch.device, torch.Tensor] = {}


def u8_lut(device: torch.device) -> torch.Tensor:
    """[256] fp32 table of torch's own `uint8 / 255.0` (the default loader's normalisation,
    yolort/models/yolov5.py:228), so uint8 inputs reproduce it bit for bit."""
    t = _u8_lut.get(device)
    if t is None:
        t = (torch.arange(256, dtype=torch.uint8) / 255.0).to(torch.float32).to(device)
        _u8_lut[device] = t
    return t


YB_SRC_CHW, YB_SRC_HWC = 0, 1


def _is_hwc_view(im: torch.Tensor) -> bool:
    _, h, w = im.shape
    return tuple(im.stride()) == (1, 3 * w, 3) and (h > 1 or w > 1)


def letterbox(images: List[torch.Tensor], geoms, Hb: int, Wb: int, fill: float, out: torch.Tensor,
              layout: int) -> torch.Tensor:
    n = len(images)
    dev = out.device
    require_cuda(out, "letterbox")
    src_dtype = images[0].dtype
    ptrs = (ctypes.c_void_p * n)()
    keep = []
    for im in images:
        require_cuda(im, "letterbox")
        if im.dtype != src_dtype:
            raise NativeLibraryError("letterbox: all images of a batch must share a dtype")
        if im.dim() != 3 or im.shape[0] != 3:
            raise ValueError(f"images is expected to be a list of 3d tensors of shape [C, H, W], but got '{im.shape}'.")
    # [3,H,W] views of interleaved HWC memory (decoded image files) are read in place; anything else goes planar
    hwc = all(_is_hwc_view(im) for im in images)
    for i, im in enumerate(images):
        if not hwc:
            im = im.contiguous()
        keep.append(im)
        ptrs[i] = im.data_ptr()
    lut = u8_lut(dev) if src_dtype == torch.uint8 else None
    with device_guard(dev):
        check(lib().yb_letterbox_strided(n, ptrs, dtype_code(src_dtype), YB_SRC_HWC if hwc else YB_SRC_CHW, geoms,
                                         int(Hb), int(Wb), float(fill), lut.data_ptr() if lut is not None else None,
                                         out.data_ptr(), dtype_code(out.dtype), int(layout), current_stream_ptr(dev)),
              "yb_letterbox")
    # the kernel reads the sources asynchronously on this stream: one record per distinct storage (the images of a
    # packed batch are views of one buffer)
    stream = torch.cuda.current_stream(dev)
    seen = set()
    for im in keep:
        key = im.untyped_storage().data_ptr()
        if key not in seen:
            seen.add(key)
            im.record_stream(stream)
    return out


# ---------------------------------------------------------------------------------------------------
# execution plan
# ---------------------------------------------------------------------------------------------------
def conv_chain_supported(op: "OpDesc") -> bool:
    """Whether the native library can run `op` (with op.chain set) as one fused launch (pure host logic)."""
    return bool(lib().yb_conv_chain_supported(ctypes.byref(op)))


def conv_config(op: "OpDesc") -> dict:
    """How the library would launch this convolution (host-only): kernel, tiling, residency, shared memory."""
    info = ConvInfo()
    check(lib().yb_conv_config(ctypes.byref(op), ctypes.byref(info)), "yb_conv_config")
    patch = info.kernel == YB_CONV_KERNEL_PATCH
    cfg = {k: int(getattr(info, k)) for k in ("block_n", "n_tiles", "weights_resident", "tiles_per_pass", "slots", "ring",
                                               "store_cols", "smem_bytes", "grid", "chained", "resident_ctas", "m_tiles",
                                               "work_items", "tail_n", "tail_tiles", "tail_split")}
    cfg["patch_kernel"] = int(patch)
    cfg["e4m3_kernel"] = int(info.kernel == YB_CONV_KERNEL_E4M3)
    # the halo-patch kernel reports its staging buffers, the others their consumer warpgroups (which share two buffers)
    cfg["store_bufs" if patch else "epilogue_groups"] = int(info.store_bufs if patch else info.groups)
    # CTAs per SM x consumer warpgroups: "1x2", "2x2" (the 104-register instances) or "2x1"; "ctas_per_sm" names the
    # 104-register layout only.  The 1x1 / im2col kernel's two-tile tasks on four warpgroups are "1x4x2" (x M tiles per
    # task), apart from its two consumer teams of single-tile tasks ("1x4").
    pairs = not patch and info.groups == 4 and info.tiles_per_pass == 2
    cfg["layout"] = f"{info.resident_ctas}x{info.groups}" + ("x2" if pairs else "")
    # consumer warpgroups per CTA: 2, 1 (the 2x1 layout) or 4 (halo patch: 128-column pair tasks; 1x1 / im2col kernel:
    # two-tile tasks, tiles_per_pass 2; either kernel: two consumer teams of single-tile tasks, tiles_per_pass 1)
    cfg["consumer_groups"] = int(info.groups)
    cfg["ctas_per_sm"] = 2 if cfg["layout"] == "2x2" else 1
    if patch:
        cfg["patch_tiling"] = PATCH_TILINGS[info.tiling]
    return cfg


class Plan:
    """Owns a native yb_plan handle (list of prepared launches)."""

    def __init__(self, ops: Sequence[OpDesc], device: torch.device):
        arr = (OpDesc * len(ops))(*ops)
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            check(lib().yb_plan_create(arr, len(ops), ctypes.byref(handle)), "yb_plan_create")
        self._h = handle
        self.device = device
        self.n_ops = len(ops)

    def run(self, first: int = 0, count: Optional[int] = None) -> None:
        if count is None:
            count = self.n_ops - first
        with device_guard(self.device):
            check(lib().yb_plan_run_range(self._h, first, count, current_stream_ptr(self.device)), "yb_plan_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and _lib is not None:
            _lib.yb_plan_destroy(h)
            self._h = None


# ---------------------------------------------------------------------------------------------------
# post-process
# ---------------------------------------------------------------------------------------------------
class _NmsArena:
    """Per-device reusable workspace; grows when the candidate count exceeds its capacity."""

    def __init__(self):
        self.ws: Optional[torch.Tensor] = None
        self.cap_per_image = 16384


_arenas: Dict[torch.device, _NmsArena] = {}


def _level_struct(t: torch.Tensor, layout: str, n_anchors: int, n_outputs: int, stride_px: float,
                  anchors: Sequence[float]) -> HeadLevel:
    lv = HeadLevel()
    lv.logits = t.data_ptr()
    lv.dtype = dtype_code(t.dtype)
    if layout == "nahwk":  # reference layout [N, A, H, W, K]
        if t.dim() != 5 or t.shape[1] != n_anchors or t.shape[4] != n_outputs or not t.is_contiguous():
            raise NativeLibraryError(f"decode_nms: expected contiguous [N,{n_anchors},H,W,{n_outputs}], got {tuple(t.shape)}")
        N, A, H, W, K = t.shape
        lv.H, lv.W = H, W
        lv.stride_n, lv.stride_a, lv.stride_y, lv.stride_x = A * H * W * K, H * W * K, W * K, K
    elif layout == "nhwc":  # plan layout [N, H, W, Cpad] with channel a*K + k
        if t.dim() != 4 or t.shape[3] < n_anchors * n_outputs or not t.is_contiguous():
            raise NativeLibraryError(f"decode_nms: expected contiguous [N,H,W,>={n_anchors * n_outputs}], got {tuple(t.shape)}")
        N, H, W, C = t.shape
        lv.H, lv.W = H, W
        lv.stride_n, lv.stride_a, lv.stride_y, lv.stride_x = H * W * C, n_outputs, W * C, C
    else:
        raise NativeLibraryError(f"unknown head layout {layout!r}")
    lv.stride_px = float(stride_px)
    for i, v in enumerate(anchors):
        lv.anchors_px[i] = float(v)
    return lv


def decode_nms_padded(head_outputs: List[torch.Tensor], layout: str, strides: Sequence[float],
                      anchors_px: Sequence[Sequence[float]], num_classes: int, score_thresh: float,
                      nms_thresh: float, detections_per_img: int, semantics: int = NMS_TV_AUTO,
                      rescale: Optional[torch.Tensor] = None, stage_hook=None):
    """Launches decode+NMS; returns padded device tensors (boxes [N,D,4], scores [N,D], labels [N,D],
    counts [N], status [4]) without synchronising -- the caller reads `counts`/`status`."""
    t0 = head_outputs[0]
    require_cuda(t0, "decode_nms")
    dev = t0.device
    n_images = int(t0.shape[0])
    n_levels = len(head_outputs)
    n_anchors = len(anchors_px[0]) // 2
    if n_levels > YB_MAX_LEVELS or n_anchors > YB_MAX_ANCHORS:
        raise NativeLibraryError("decode_nms: too many levels/anchors")
    arena = _arenas.setdefault(dev, _NmsArena())
    levels = (HeadLevel * n_levels)(*[
        _level_struct(t, layout, n_anchors, num_classes + 5, strides[i], anchors_px[i])
        for i, t in enumerate(head_outputs)])
    D = int(detections_per_img)
    boxes = torch.empty((n_images, D, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n_images, D), dtype=torch.float32, device=dev)
    labels = torch.empty((n_images, D), dtype=torch.int64, device=dev)
    counts = torch.empty((n_images,), dtype=torch.int32, device=dev)
    status = torch.empty((4,), dtype=torch.int64, device=dev)
    p = NmsParams(n_images, n_levels, n_anchors, int(num_classes), float(score_thresh), float(nms_thresh), D,
                  int(semantics), int(arena.cap_per_image) * n_images)
    need = lib().yb_decode_nms_workspace_bytes(ctypes.byref(p), levels)
    if arena.ws is None or arena.ws.numel() < need or arena.ws.device != dev:
        arena.ws = torch.empty((need,), dtype=torch.uint8, device=dev)
    with device_guard(dev):
        if stage_hook is None:
            check(lib().yb_decode_nms(ctypes.byref(p), levels, rescale.data_ptr() if rescale is not None else None,
                                      boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                      status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), current_stream_ptr(dev)),
                  "yb_decode_nms")
        else:   # same three steps, with a callback between them (bench.py records CUDA events per stage)
            st = current_stream_ptr(dev)
            check(lib().yb_nms_begin(ctypes.byref(p), levels, status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), st),
                  "yb_nms_begin")
            stage_hook("begin")
            check(lib().yb_decode_candidates(ctypes.byref(p), levels, arena.ws.data_ptr(), arena.ws.numel(), st),
                  "yb_decode_candidates")
            stage_hook("decode")
            check(lib().yb_nms_finish(ctypes.byref(p), levels, rescale.data_ptr() if rescale is not None else None,
                                      boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                      status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), st), "yb_nms_finish")
            stage_hook("nms")
    arena.debug_offset = lib().yb_decode_nms_debug_offset(ctypes.byref(p), levels)
    return boxes, scores, labels, counts, status


def decode_dense(head_outputs: List[torch.Tensor], layout: str, strides: Sequence[float],
                 anchors_px: Sequence[Sequence[float]], num_classes: int):
    """LogitsDecoder (yolort/relay/logits_decoder.py:26-61): (boxes [N,A,4] xyxy fp32, scores [N,A,nc] fp32) for
    every anchor, no threshold and no NMS; one launch, no host synchronisation."""
    t0 = head_outputs[0]
    require_cuda(t0, "decode_dense")
    dev = t0.device
    n_images, n_levels = int(t0.shape[0]), len(head_outputs)
    n_anchors = len(anchors_px[0]) // 2
    if n_levels > YB_MAX_LEVELS or n_anchors > YB_MAX_ANCHORS:
        raise NativeLibraryError("decode_dense: too many levels/anchors")
    levels = (HeadLevel * n_levels)(*[
        _level_struct(t, layout, n_anchors, num_classes + 5, strides[i], anchors_px[i])
        for i, t in enumerate(head_outputs)])
    total = sum(n_anchors * int(lv.H) * int(lv.W) for lv in levels)
    boxes = torch.empty((n_images, total, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n_images, total, int(num_classes)), dtype=torch.float32, device=dev)
    p = NmsParams(n_images, n_levels, n_anchors, int(num_classes), 0.0, 0.0, 1, 0, 0)
    with device_guard(dev):
        check(lib().yb_decode_dense(ctypes.byref(p), levels, boxes.data_ptr(), scores.data_ptr(), current_stream_ptr(dev)),
              "yb_decode_dense")
    return boxes, scores


def nms_phase_clocks(device) -> list:
    """Debug: clock counts of the NMS kernel phases for image 0 of the last decode_nms call on `device`."""
    arena = _arenas[torch.device(device)]
    off = arena.debug_offset
    return arena.ws[off: off + 128].view(torch.int64)[4:10].cpu().tolist()


def decode_nms(head_outputs: List[torch.Tensor], layout: str, strides, anchors_px, score_thresh: float,
               nms_thresh: float, detections_per_img: int, semantics: int = NMS_TV_AUTO,
               rescale: Optional[torch.Tensor] = None, num_classes: Optional[int] = None) -> List[Dict[str, torch.Tensor]]:
    """Full post-process returning the reference's List[Dict] (keys in order scores, labels, boxes:
    yolort/models/box_head.py:427).  One device->host read of counts+status; re-runs with a larger
    arena when an image overflowed its candidate share (never truncates silently)."""
    if num_classes is None:
        t0 = head_outputs[0]
        num_classes = int(t0.shape[4]) - 5 if layout == "nahwk" else None
        if num_classes is None:
            raise NativeLibraryError("decode_nms: num_classes is required for the nhwc layout")
    boxes, scores, labels, counts, host = decode_nms_complete(head_outputs, layout, strides, anchors_px, num_classes,
                                                              score_thresh, nms_thresh, detections_per_img, semantics,
                                                              rescale)
    n = counts.numel()
    return [{"scores": scores[i, :host[i]], "labels": labels[i, :host[i]], "boxes": boxes[i, :host[i]]} for i in range(n)]


def decode_nms_complete(head_outputs: List[torch.Tensor], layout: str, strides, anchors_px, num_classes: int,
                        score_thresh: float, nms_thresh: float, detections_per_img: int, semantics: int = NMS_TV_AUTO,
                        rescale: Optional[torch.Tensor] = None):
    """decode_nms_padded that drops nothing: one device->host read of counts + status, and a rerun with a larger
    arena while an image overflowed its candidate share.  Returns (boxes, scores, labels, counts, host), host the
    counts followed by the status as a python list."""
    dev = head_outputs[0].device
    while True:
        boxes, scores, labels, counts, status = decode_nms_padded(
            head_outputs, layout, strides, anchors_px, num_classes, score_thresh, nms_thresh,
            detections_per_img, semantics, rescale)
        host = torch.cat([counts.to(torch.int64), status]).tolist()     # one D2H + one conversion for the whole batch
        n = counts.numel()
        if host[n + 1] == 0:
            return boxes, scores, labels, counts, host
        arena = _arenas[dev]
        arena.cap_per_image = max(2 * arena.cap_per_image, int(host[n + 2]))
        arena.ws = None


class FusedPost:
    """Post-processing state of a plan whose head convolutions decode in their epilogue: a fixed candidate arena
    (the heads hold raw pointers into it), the NMS parameters, and begin()/finish() around the plan run."""

    def __init__(self, n_images: int, level_hw: Sequence[Tuple[int, int]], strides: Sequence[float],
                 anchors_px: Sequence[Sequence[float]], num_classes: int, score_thresh: float, nms_thresh: float,
                 detections_per_img: int, semantics: int, device: torch.device, cap_per_image: int = 32768):
        self.device = device
        self.n_images, self.D = n_images, int(detections_per_img)
        n_levels, n_anchors = len(level_hw), len(anchors_px[0]) // 2
        self.levels = (HeadLevel * n_levels)()
        for i, (h, w) in enumerate(level_hw):
            self.levels[i].H, self.levels[i].W = int(h), int(w)
            self.levels[i].dtype = YB_F16
            self.levels[i].stride_px = float(strides[i])
            for j, v in enumerate(anchors_px[i]):
                self.levels[i].anchors_px[j] = float(v)
        self.params = NmsParams(n_images, n_levels, n_anchors, int(num_classes), float(score_thresh), float(nms_thresh),
                                self.D, int(semantics), int(cap_per_image) * n_images)
        need = lib().yb_decode_nms_workspace_bytes(ctypes.byref(self.params), self.levels)
        self.ws = torch.empty((need,), dtype=torch.uint8, device=device)
        self.layout = NmsLayout()
        check(lib().yb_nms_layout(ctypes.byref(self.params), self.levels, self.ws.data_ptr(), self.ws.numel(),
                                  ctypes.byref(self.layout)), "yb_nms_layout")
        self.head_decode = []
        for i in range(n_levels):
            hd = HeadDecode()
            hd.n_anchors, hd.n_classes = n_anchors, int(num_classes)
            hd.level_start, hd.anchors_per_image = int(self.layout.level_start[i]), int(self.layout.anchors_per_image)
            hd.stride_px = float(strides[i])
            for j, v in enumerate(anchors_px[i]):
                hd.anchors_px[j] = float(v)
            hd.score_thresh = float(score_thresh)
            hd.cap_per_image = int(self.layout.cap_per_image)
            hd.keys, hd.boxes = self.layout.keys, self.layout.boxes
            hd.img_count, hd.img_maxc = self.layout.img_count, self.layout.img_maxc
            self.head_decode.append(hd)
        self.status = torch.empty((4,), dtype=torch.int64, device=device)

    def begin(self) -> None:
        with device_guard(self.device):
            check(lib().yb_nms_begin(ctypes.byref(self.params), self.levels, self.status.data_ptr(), self.ws.data_ptr(),
                                     self.ws.numel(), current_stream_ptr(self.device)), "yb_nms_begin")

    def finish(self, rescale: Optional[torch.Tensor]):
        n, D, dev = self.n_images, self.D, self.device
        boxes = torch.empty((n, D, 4), dtype=torch.float32, device=dev)
        scores = torch.empty((n, D), dtype=torch.float32, device=dev)
        labels = torch.empty((n, D), dtype=torch.int64, device=dev)
        counts = torch.empty((n,), dtype=torch.int32, device=dev)
        with device_guard(dev):
            check(lib().yb_nms_finish(ctypes.byref(self.params), self.levels,
                                      rescale.data_ptr() if rescale is not None else None, boxes.data_ptr(),
                                      scores.data_ptr(), labels.data_ptr(), counts.data_ptr(), self.status.data_ptr(),
                                      self.ws.data_ptr(), self.ws.numel(), current_stream_ptr(dev)), "yb_nms_finish")
        return boxes, scores, labels, counts, self.status


# ---------------------------------------------------------------------------------------------------
# test-time augmentation (yolort/v5/models/yolo.py:152-208)
# ---------------------------------------------------------------------------------------------------
TTA_SCALES = (1.0, 0.83, 0.67)      # _forward_augment's fixed lists (yolo.py:154-155): scale, left-right mirror
TTA_FLIPS = (False, True, False)
TTA_FILL = 0.447                    # scale_img's pad value (torch_utils.py:300)


def tta_pass_geometry(Hb: int, Wb: int, gs: int) -> List[Tuple[int, int, int, int]]:
    """(nh, nw, Hp, Wp) per pass: scale_img (torch_utils.py:288-300) of an Hb x Wb canvas, resized to
    int(H * s) x int(W * s) and padded to ceil(H * s / gs) * gs x ceil(W * s / gs) * gs (Python doubles, as the
    reference); scale 1 is the canvas itself."""
    out = []
    for s in TTA_SCALES:
        if s == 1.0:
            out.append((Hb, Wb, Hb, Wb))
            continue
        out.append((int(Hb * s), int(Wb * s), math.ceil(Hb * s / gs) * gs, math.ceil(Wb * s / gs) * gs))
    return out


def canvas_rescale(src: torch.Tensor, dst: torch.Tensor, nh: int, nw: int, flip_lr: bool, fill: float = TTA_FILL) -> torch.Tensor:
    """One pass canvas: src [N, Hb/2, Wb/2, 16] space-to-depth (fp16 / bf16) -> dst [N, Hp/2, Wp/2, 16], the bilinear
    resize of the (mirrored) canvas to nh x nw at the top left, `fill` elsewhere (yb_canvas_rescale)."""
    require_cuda(src, "canvas_rescale")
    if src.dtype != dst.dtype or src.dim() != 4 or dst.dim() != 4 or src.shape[3] != 16 or dst.shape[3] != 16 \
            or src.shape[0] != dst.shape[0] or not src.is_contiguous() or not dst.is_contiguous():
        raise NativeLibraryError(f"canvas_rescale: expected two contiguous [N,H/2,W/2,16] canvases of one dtype, got "
                                 f"{tuple(src.shape)} {src.dtype} -> {tuple(dst.shape)} {dst.dtype}")
    n, h2, w2, _ = src.shape
    _, hp2, wp2, _ = dst.shape
    dev = src.device
    with device_guard(dev):
        check(lib().yb_canvas_rescale(int(n), src.data_ptr(), dtype_code(src.dtype), 2 * int(h2), 2 * int(w2), int(nh),
                                      int(nw), int(bool(flip_lr)), float(fill), dst.data_ptr(), 2 * int(hp2),
                                      2 * int(wp2), current_stream_ptr(dev)), "yb_canvas_rescale")
    return dst


_tta_arenas: Dict[torch.device, _NmsArena] = {}


def decode_nms_tta_padded(passes, canvas_w: int, strides: Sequence[float], anchors_px: Sequence[Sequence[float]],
                          num_classes: int, score_thresh: float, nms_thresh: float, detections_per_img: int,
                          semantics: int = NMS_TV_AUTO, rescale: Optional[torch.Tensor] = None):
    """Multi-pass decode + one NMS per image.  `passes`: per pass (heads, level_ids, scale, flip_lr) with `heads` the
    pass's NHWC head buffers and `level_ids` the levels that take part, in order.  Padded device outputs as
    decode_nms_padded, without synchronising."""
    t0 = passes[0][0][0]
    require_cuda(t0, "decode_nms_tta")
    dev = t0.device
    n_images = int(t0.shape[0])
    n_anchors = len(anchors_px[0]) // 2
    if len(passes) > YB_TTA_MAX_PASSES or n_anchors > YB_MAX_ANCHORS:
        raise NativeLibraryError("decode_nms_tta: too many passes/anchors")
    arr = (TtaPass * len(passes))()
    for q, (heads, level_ids, scale, flip) in enumerate(passes):
        if len(level_ids) > YB_MAX_LEVELS:
            raise NativeLibraryError("decode_nms_tta: too many levels")
        arr[q].n_levels, arr[q].flip_lr = len(level_ids), int(bool(flip))
        arr[q].scale, arr[q].canvas_w = float(scale), float(canvas_w)
        for j, l in enumerate(level_ids):
            require_cuda(heads[l], "decode_nms_tta")
            arr[q].levels[j] = _level_struct(heads[l], "nhwc", n_anchors, num_classes + 5, strides[l], anchors_px[l])
    arena = _tta_arenas.setdefault(dev, _NmsArena())
    D = int(detections_per_img)
    boxes = torch.empty((n_images, D, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n_images, D), dtype=torch.float32, device=dev)
    labels = torch.empty((n_images, D), dtype=torch.int64, device=dev)
    counts = torch.empty((n_images,), dtype=torch.int32, device=dev)
    status = torch.empty((4,), dtype=torch.int64, device=dev)
    p = NmsParams(n_images, 0, n_anchors, int(num_classes), float(score_thresh), float(nms_thresh), D, int(semantics),
                  int(arena.cap_per_image) * n_images)
    need = lib().yb_decode_nms_tta_workspace_bytes(ctypes.byref(p), len(passes), arr)
    if need == 0:
        raise NativeLibraryError(f"yb_decode_nms_tta_workspace_bytes: {lib().yb_last_error().decode()}")
    if arena.ws is None or arena.ws.numel() < need or arena.ws.device != dev:
        arena.ws = None
        arena.ws = torch.empty((need,), dtype=torch.uint8, device=dev)
    with device_guard(dev):
        check(lib().yb_decode_nms_tta(ctypes.byref(p), len(passes), arr, rescale.data_ptr() if rescale is not None else None,
                                      boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                      status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), current_stream_ptr(dev)),
              "yb_decode_nms_tta")
    return boxes, scores, labels, counts, status


def decode_nms_tta(passes, canvas_w: int, strides, anchors_px, num_classes: int, score_thresh: float, nms_thresh: float,
                   detections_per_img: int, semantics: int = NMS_TV_AUTO,
                   rescale: Optional[torch.Tensor] = None) -> List[Dict[str, torch.Tensor]]:
    """decode_nms_tta_padded + the reference's List[Dict]: one device->host read of counts + status; an image that
    overflowed its share of the candidate arena grows it and re-runs (never truncates)."""
    dev = passes[0][0][0].device
    while True:
        boxes, scores, labels, counts, status = decode_nms_tta_padded(
            passes, canvas_w, strides, anchors_px, num_classes, score_thresh, nms_thresh, detections_per_img, semantics,
            rescale)
        host = torch.cat([counts.to(torch.int64), status]).tolist()
        n = counts.numel()
        if host[n + 1] == 0:
            break
        arena = _tta_arenas[dev]
        arena.cap_per_image = max(2 * arena.cap_per_image, int(host[n + 2]))
        arena.ws = None
    return [{"scores": scores[i, :host[i]], "labels": labels[i, :host[i]], "boxes": boxes[i, :host[i]]} for i in range(n)]


def batched_nms(boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, iou_threshold: float,
                semantics: int = NMS_TV_AUTO, max_keep: int = 4096) -> torch.Tensor:
    """torchvision.ops.batched_nms on the device (first `max_keep` survivors, score-descending)."""
    require_cuda(boxes, "batched_nms")
    dev = boxes.device
    boxes = boxes.contiguous().float()
    scores = scores.contiguous().float()
    labels = labels.contiguous().to(torch.int64)
    n = int(boxes.shape[0])
    keep = torch.empty((max_keep,), dtype=torch.int64, device=dev)
    n_keep = torch.zeros((1,), dtype=torch.int32, device=dev)
    need = lib().yb_batched_nms_workspace_bytes(n)
    ws = torch.empty((need,), dtype=torch.uint8, device=dev)
    with device_guard(dev):
        check(lib().yb_batched_nms(boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), n, float(iou_threshold),
                                   int(semantics), int(max_keep), keep.data_ptr(), n_keep.data_ptr(), ws.data_ptr(),
                                   ws.numel(), current_stream_ptr(dev)), "yb_batched_nms")
    return keep[: int(n_keep.item())]


# ---------------------------------------------------------------------------------------------------
# JPEG decode
# ---------------------------------------------------------------------------------------------------
def jpeg_parse(data: bytes) -> JpegInfo:
    """Host-only marker parse (yb_jpeg_parse); `.supported` says whether jpeg_decode takes the file."""
    info = JpegInfo()
    buf = (ctypes.c_uint8 * len(data)).from_buffer_copy(data) if len(data) else None
    check(lib().yb_jpeg_parse(buf, len(data), ctypes.byref(info)), "yb_jpeg_parse")
    return info


_jpeg_staging: Dict[torch.device, dict] = {}


def _jpeg_stage(device: torch.device, nbytes: int) -> list:
    """A pinned host buffer of >= nbytes for the next decode on `device`: two alternate, and the copy out of a buffer
    must have finished before it is refilled (fresh pinned allocations cost about as much as the decode itself)."""
    st = _jpeg_staging.setdefault(device, {"slots": [None, None], "next": 0})
    k = st["next"]
    st["next"] = k ^ 1
    slot = st["slots"][k]
    if slot is not None and slot[1] is not None:
        slot[1].synchronize()
    if slot is None or slot[0].numel() < nbytes:
        slot = [torch.empty((max(nbytes + nbytes // 4, 1 << 20),), dtype=torch.uint8, pin_memory=True), None]
        st["slots"][k] = slot
    return slot


def jpeg_decode(datas: Sequence, infos: Sequence[JpegInfo], device: torch.device,
                dst: Optional[Sequence[torch.Tensor]] = None):
    """Decodes supported JPEG files (bytes, or 1-D uint8 host tensors, with their parse results) on `device`'s
    current stream.  The infos and the compressed bytes cross PCIe as one copy from pinned memory.  Returns ([3,H,W]
    uint8 CHW views of HWC memory, status int32 [n] on the device); nothing is synchronised.  `dst` optionally gives
    the contiguous [H,W,3] uint8 device tensors to write into."""
    device = torch.device(device)
    if device.type != "cuda":
        raise NativeLibraryError("jpeg_decode runs on a CUDA device only (no CPU fallback)")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    n = len(datas)
    isz = ctypes.sizeof(JpegInfo)
    arr = (JpegInfo * n)()
    off = (n * isz + 15) // 16 * 16
    lens = []
    for i, (d, info) in enumerate(zip(datas, infos)):
        if not info.supported:
            raise NativeLibraryError(f"jpeg_decode: image {i} is not supported: {info.reason.decode()}")
        ctypes.memmove(ctypes.byref(arr[i]), ctypes.byref(info), isz)
        arr[i].data_offset = off
        lens.append(int(d.numel()) if isinstance(d, torch.Tensor) else len(d))
        off += (lens[-1] + 15) // 16 * 16
    slot = _jpeg_stage(device, off)
    base = slot[0].data_ptr()
    ctypes.memmove(base, ctypes.addressof(arr), n * isz)
    for i, d in enumerate(datas):
        if isinstance(d, torch.Tensor):
            if d.is_cuda or d.dtype != torch.uint8 or d.dim() != 1:
                raise NativeLibraryError("jpeg_decode: file contents must be 1-D uint8 host tensors or bytes")
            d = d.contiguous()
            ctypes.memmove(base + int(arr[i].data_offset), d.data_ptr(), lens[i])
        else:
            ctypes.memmove(base + int(arr[i].data_offset), bytes(d), lens[i])
    host = slot[0][:off]
    ws_bytes = int(lib().yb_jpeg_workspace_bytes(n, arr))
    with device_guard(device):
        src = host.to(device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        slot[1] = ev
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
        sizes = [int(a.height) * int(a.width) * 3 for a in arr]
        if dst is None:
            out = torch.empty((sum(sizes),), dtype=torch.uint8, device=device)
            offs = [0] + list(itertools.accumulate(sizes))[:-1]
            dst = [out[o:o + sz].view(int(a.height), int(a.width), 3) for o, sz, a in zip(offs, sizes, arr)]
        status = torch.empty((n,), dtype=torch.int32, device=device)
        ptrs = (ctypes.c_void_p * n)()
        images = []
        for i, (a, t) in enumerate(zip(arr, dst)):
            if (t.device != device or t.dtype != torch.uint8 or not t.is_contiguous()
                    or tuple(t.shape) != (int(a.height), int(a.width), 3)):
                raise NativeLibraryError(f"jpeg_decode: dst[{i}] must be a contiguous uint8 [{a.height},{a.width},3] "
                                         f"tensor on {device}")
            ptrs[i] = t.data_ptr()
            images.append(t.permute(2, 0, 1))
        check(lib().yb_jpeg_decode(n, arr, src.data_ptr(), ptrs, status.data_ptr(), ws.data_ptr(), ws_bytes,
                                   current_stream_ptr(device)), "yb_jpeg_decode")
    return images, status


# ---------------------------------------------------------------------------------------------------
# COCO box evaluation
# ---------------------------------------------------------------------------------------------------
def coco_append(boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, counts: torch.Tensor,
                row_image: torch.Tensor, label_map: torch.Tensor, records: torch.Tensor, status: torch.Tensor) -> None:
    """yb_coco_append on the current stream of `records`' device: boxes fp32 [n,d,4], scores fp32 [n,d], labels int64
    [n,d], counts int32 [n], row_image int32 [n], label_map int32 [L]; records int32 [n*d, 8]; status int32 [1]."""
    dev = records.device
    if dev.type != "cuda":
        raise NativeLibraryError("coco_append runs on a CUDA device only (no CPU fallback)")
    n, d = int(scores.shape[0]), int(scores.shape[1])
    ts = (boxes, scores, labels, counts, row_image, label_map, records, status)
    want = (torch.float32, torch.float32, torch.int64, torch.int32, torch.int32, torch.int32, torch.int32, torch.int32)
    for t, dt in zip(ts, want):
        if t.device != dev or t.dtype != dt or not t.is_contiguous():
            raise NativeLibraryError(f"coco_append: every tensor must be a contiguous {dt} tensor on {dev}")
    if tuple(boxes.shape) != (n, d, 4) or tuple(labels.shape) != (n, d) or counts.numel() != n \
            or row_image.numel() != n or tuple(records.shape) != (n * d, YB_COCO_RECORD_INT32):
        raise NativeLibraryError("coco_append: shapes do not agree")
    with device_guard(dev):
        check(lib().yb_coco_append(n, d, boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                   row_image.data_ptr(), label_map.data_ptr(), label_map.numel(), records.data_ptr(),
                                   status.data_ptr(), current_stream_ptr(dev)), "yb_coco_append")


def coco_evaluate(gt: CocoGt, records: torch.Tensor, evaluated: torch.Tensor, params: torch.Tensor):
    """yb_coco_evaluate: records int32 [n, 8], evaluated uint8 [n_images], params float64 [119], all on one CUDA device.
    Returns float64 device tensors precision [10,101,K,4,3], recall [10,K,4,3], scores [10,101,K,4,3]."""
    dev = records.device
    if dev.type != "cuda":
        raise NativeLibraryError("coco_evaluate runs on a CUDA device only (no CPU fallback)")
    for t, dt in ((records, torch.int32), (evaluated, torch.uint8), (params, torch.float64)):
        if t.device != dev or t.dtype != dt or not t.is_contiguous():
            raise NativeLibraryError(f"coco_evaluate: expected a contiguous {dt} tensor on {dev}")
    if evaluated.numel() != gt.n_images or params.numel() != YB_COCO_NUM_PARAMS:
        raise NativeLibraryError("coco_evaluate: evaluated / params have the wrong size")
    n = int(records.shape[0])
    K = int(gt.n_categories)
    with device_guard(dev):
        ws_bytes = int(lib().yb_coco_evaluate_workspace_bytes(n, ctypes.byref(gt)))
        if ws_bytes == 0:
            raise NativeLibraryError(f"coco_evaluate: no workspace size for {n} records: {lib().yb_last_error()}")
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        precision = torch.empty((10, 101, K, 4, 3), dtype=torch.float64, device=dev)
        recall = torch.empty((10, K, 4, 3), dtype=torch.float64, device=dev)
        scores = torch.empty_like(precision)
        check(lib().yb_coco_evaluate(ctypes.byref(gt), records.data_ptr() if n else None, n, evaluated.data_ptr(),
                                     params.data_ptr(), precision.data_ptr(), recall.data_ptr(), scores.data_ptr(),
                                     ws.data_ptr(), ws_bytes, current_stream_ptr(dev)), "yb_coco_evaluate")
    return precision, recall, scores


# ---------------------------------------------------------------------------------------------------
# YOLOv5 training loss
# ---------------------------------------------------------------------------------------------------
def yolo_loss_levels(head_outputs: Sequence[torch.Tensor], strides: Sequence[int],
                     anchors_px: Sequence[Sequence[float]]):
    """yb_loss_level array over contiguous [N, A, H, W, K] head outputs (one dtype, one device)."""
    levels = (LossLevel * len(head_outputs))()
    for i, t in enumerate(head_outputs):
        lv = levels[i]
        lv.logits = t.data_ptr()
        lv.dtype = dtype_code(t.dtype)
        lv.H, lv.W = int(t.shape[2]), int(t.shape[3])
        lv.stride_px = float(strides[i])
        for j, v in enumerate(anchors_px[i]):
            lv.anchors_px[j] = float(v)
    return levels


def yolo_loss_forward(params: YoloLossParams, levels, targets: torch.Tensor, device: torch.device):
    """yb_yolo_loss_forward on `device`'s current stream.  targets: contiguous fp32 [T, 6] on the device.  Returns
    (losses fp32 [3 + L], status int32 [1], workspace uint8); nothing is synchronised."""
    n = int(targets.shape[0])
    ws_bytes = int(lib().yb_yolo_loss_workspace_bytes(ctypes.byref(params), levels, n))
    if ws_bytes == 0:
        raise NativeLibraryError(f"yolo_loss: {lib().yb_last_error().decode('utf-8', 'replace')}")
    with device_guard(device):
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
        out = torch.empty((3 + params.n_levels,), dtype=torch.float32, device=device)
        status = torch.zeros((1,), dtype=torch.int32, device=device)
        check(lib().yb_yolo_loss_forward(ctypes.byref(params), levels, targets.data_ptr() if n else None, n,
                                         out.data_ptr(), status.data_ptr(), ws.data_ptr(), ws_bytes,
                                         current_stream_ptr(device)), "yb_yolo_loss_forward")
    return out, status, ws


def yolo_loss_backward(params: YoloLossParams, levels, n_targets: int, grad_losses: torch.Tensor, ws: torch.Tensor,
                       grads: Sequence[torch.Tensor]) -> None:
    """yb_yolo_loss_backward: writes d loss / d logits into `grads` (contiguous, shaped and typed as the head
    outputs) from grad_losses fp32 [3] on the device."""
    dev = ws.device
    ptrs = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
    with device_guard(dev):
        check(lib().yb_yolo_loss_backward(ctypes.byref(params), levels, int(n_targets), grad_losses.data_ptr(), ptrs,
                                          ws.data_ptr(), ws.numel(), current_stream_ptr(dev)), "yb_yolo_loss_backward")


def yolo_loss_matches(params: YoloLossParams, levels, n_targets: int, ws: torch.Tensor):
    """The matches a forward call left in `ws` (test and debugging aid; synchronises): (records int32 [M, 24],
    start index of each level's matches + the total, as a list)."""
    out = (ctypes.c_int64 * 3)()
    check(lib().yb_yolo_loss_layout(ctypes.byref(params), levels, int(n_targets), out), "yb_yolo_loss_layout")
    cap = int(out[2])
    per_level = cap // params.n_levels if params.n_levels else 0
    pos = ws[int(out[1]): int(out[1]) + 4 * (cap + 1)].view(torch.int32).cpu()
    bounds = [int(pos[l * per_level]) for l in range(params.n_levels)] + [int(pos[cap])]
    rec = ws[int(out[0]): int(out[0]) + 4 * YB_LOSS_MATCH_INT32 * bounds[-1]].view(torch.int32)
    return rec.view(-1, YB_LOSS_MATCH_INT32).cpu(), bounds


# ---------------------------------------------------------------------------------------------------
# training augmentations
# ---------------------------------------------------------------------------------------------------
def augment(descs, out: torch.Tensor, sources: Sequence[torch.Tensor]) -> torch.Tensor:
    """Runs the prepared-here recipes `descs` (AugImage array, src pointers set) into `out` (uint8 or float32, on the
    sources' device).  The descriptors cross to the device in one asynchronous copy from pinned memory."""
    n = len(descs)
    dev = out.device
    require_cuda(out, "augment")
    totals = (ctypes.c_int64 * (1 + YB_AUG_MAX_CONTRAST))()
    check(lib().yb_augment_prepare(n, descs, totals), "yb_augment_prepare")
    raw = torch.frombuffer(bytearray(ctypes.string_at(ctypes.addressof(descs), ctypes.sizeof(descs))), dtype=torch.uint8)
    with device_guard(dev):
        d_descs = raw.pin_memory().to(dev, non_blocking=True)
        sums = torch.empty((n * YB_AUG_MAX_CONTRAST,), dtype=torch.int64, device=dev)
        check(lib().yb_augment(n, descs, d_descs.data_ptr(), out.data_ptr(), dtype_code(out.dtype), sums.data_ptr(),
                               current_stream_ptr(dev)), "yb_augment")
        stream = torch.cuda.current_stream(dev)
        seen = set()
        for im in sources:
            key = im.untyped_storage().data_ptr()
            if key not in seen:
                seen.add(key)
                im.record_stream(stream)
    return out


def augment_sample(samplers, sources: Sequence[torch.Tensor], key: torch.Tensor, boxes: Sequence[torch.Tensor],
                   labels: Sequence[torch.Tensor], boxes_to_host: bool):
    """Draws the recipes of the images `sources` on the device (yb_augment_sample) with the transforms `samplers`
    (AugSampler array) and `key` (int64 [2] on the sources' device).  boxes / labels: fp32 [n, 4] / int64 [n] per image;
    when all are on the host they cross in the one host-to-device copy that also carries the descriptors.

    Returns (descs, counts, status, boxes, labels): the AugImage array (src pointers, sizes and recipes set), lists of
    the kept-box counts and YB_AUG_ST_* bits per image, and the batch's boxes [N, 4] / labels [N], image i's kept ones
    first in its input rows; on the host when `boxes_to_host`, else views into a device buffer.  The read-back of the
    descriptors, counts and status (and boxes) is the one host synchronisation."""
    n, dev = len(sources), key.device
    nb = sum(int(b.shape[0]) for b in boxes)
    descs = (AugImage * n)()
    for d, im in zip(descs, sources):
        d.src = im.data_ptr()
        d.stride_c, d.stride_y, d.stride_x = (int(v) for v in im.stride())
        d.src_h, d.src_w = int(im.shape[1]), int(im.shape[2])
    # one device buffer: the inputs (uploaded in one copy), then the outputs (read back in one copy)
    layout = {"start": (torch.int32, (n + 1,)), "boxes": (torch.float32, (nb, 4)), "labels": (torch.int64, (nb,)),
              "descs": (torch.uint8, (ctypes.sizeof(descs),)), "counts": (torch.int32, (n,)),
              "status": (torch.int32, (n,)), "boxes_out": (torch.float32, (nb, 4)), "labels_out": (torch.int64, (nb,))}
    off, end = {}, 0
    for name, (dtype, shape) in layout.items():
        off[name] = end
        end += -(-math.prod(shape) * dtype.itemsize // 16) * 16

    def part(t, name, base=0):
        dtype, shape = layout[name]
        o = off[name] - base
        return t[o: o + math.prod(shape) * dtype.itemsize].view(dtype).view(shape)

    stage = torch.empty((off["counts"],), dtype=torch.uint8, pin_memory=True)
    part(stage, "start").copy_(torch.tensor([0] + list(itertools.accumulate(int(b.shape[0]) for b in boxes)),
                                            dtype=torch.int32))
    on_host = all(t.device.type == "cpu" for t in list(boxes) + list(labels))
    if nb and on_host:
        torch.cat(list(boxes), out=part(stage, "boxes"))
        torch.cat(list(labels), out=part(stage, "labels"))
    ctypes.memmove(stage.data_ptr() + off["descs"], ctypes.addressof(descs), ctypes.sizeof(descs))
    with device_guard(dev):
        buf = torch.empty((end,), dtype=torch.uint8, device=dev)
        buf[: off["counts"]].copy_(stage, non_blocking=True)
        if nb and not on_host:
            torch.cat([b.to(dev) for b in boxes], out=part(buf, "boxes"))
            torch.cat([l.to(dev) for l in labels], out=part(buf, "labels"))
        p = buf.data_ptr()
        ptr = {k: p + off[k] if nb or k not in ("boxes", "labels", "boxes_out", "labels_out") else None for k in off}
        check(lib().yb_augment_sample(n, samplers, len(samplers), key.data_ptr(), ptr["descs"], ptr["boxes"],
                                      ptr["labels"], ptr["start"], ptr["boxes_out"], ptr["labels_out"], ptr["counts"],
                                      ptr["status"], current_stream_ptr(dev)), "yb_augment_sample")
        host = buf[off["descs"]: end if boxes_to_host else off["boxes_out"]].cpu()
    base = off["descs"]
    descs = (AugImage * n).from_buffer_copy(host[: ctypes.sizeof(descs)].numpy())
    src, src_base = (host, base) if boxes_to_host else (buf, 0)
    return (descs, part(host, "counts", base).tolist(), part(host, "status", base).tolist(),
            part(src, "boxes_out", src_base), part(src, "labels_out", src_base))


# ---------------------------------------------------------------------------------------------------
# weight gradient of 1x1 convolutions
# ---------------------------------------------------------------------------------------------------
def v5_augment(descs, sources: Sequence[torch.Tensor], device: torch.device) -> None:
    """Runs the YOLOv5 augmentation descriptors `descs` (V5Image array, pointers set) in one launch.  The descriptors
    (LUTs included) cross to the device in one asynchronous copy from pinned memory; nothing synchronises."""
    n = len(descs)
    total = ctypes.c_int64(0)
    check(lib().yb_v5_augment_prepare(n, descs, ctypes.byref(total)), "yb_v5_augment_prepare")
    raw = torch.frombuffer(bytearray(ctypes.string_at(ctypes.addressof(descs), ctypes.sizeof(descs))), dtype=torch.uint8)
    with device_guard(device):
        d_descs = raw.pin_memory().to(device, non_blocking=True)
        check(lib().yb_v5_augment(n, d_descs.data_ptr(), total.value, current_stream_ptr(device)), "yb_v5_augment")
        stream = torch.cuda.current_stream(device)
        seen = set()
        for im in sources:
            key = im.untyped_storage().data_ptr()
            if key not in seen:
                seen.add(key)
                im.record_stream(stream)


def v5_mixup(a: torch.Tensor, b: torch.Tensor, r: float) -> torch.Tensor:
    """uint8(trunc(a * r + b * (1 - r))) in IEEE double, elementwise over two contiguous uint8 tensors of one shape."""
    out = torch.empty_like(a, memory_format=torch.contiguous_format)
    with device_guard(a.device):
        check(lib().yb_v5_mixup(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), float(r),
                                current_stream_ptr(a.device)), "yb_v5_mixup")
    return out


def _descs_to_device(descs, device: torch.device) -> torch.Tensor:
    raw = torch.frombuffer(bytearray(ctypes.string_at(ctypes.addressof(descs), ctypes.sizeof(descs))), dtype=torch.uint8)
    return raw.pin_memory().to(device, non_blocking=True)


def _keep_alive(tensors: Sequence[torch.Tensor], device: torch.device) -> None:
    stream = torch.cuda.current_stream(device)
    seen = set()
    for t in tensors:
        key = t.untyped_storage().data_ptr()
        if key not in seen:
            seen.add(key)
            t.record_stream(stream)


def v5_resize(jobs, tensors: Sequence[torch.Tensor], device: torch.device, area: bool = False) -> None:
    """Runs the load_image resize jobs `jobs` (V5ResizeJob array, pointers set) in one launch, INTER_LINEAR or, with
    `area`, INTER_AREA (every job shrinking); `tensors` are the sources and destinations they point into.  Nothing
    synchronises."""
    n = len(jobs)
    total = ctypes.c_int64(0)
    L = lib()
    prepare, run, what = ((L.yb_v5_resize_area_prepare, L.yb_v5_resize_area, "yb_v5_resize_area") if area else
                          (L.yb_v5_resize_prepare, L.yb_v5_resize, "yb_v5_resize"))
    check(prepare(n, jobs, ctypes.byref(total)), what + "_prepare")
    with device_guard(device):
        d_jobs = _descs_to_device(jobs, device)
        check(run(n, d_jobs.data_ptr(), total.value, current_stream_ptr(device)), what)
        _keep_alive(tensors, device)


def v5_rescale_coords(boxes: Optional[torch.Tensor], counts: Optional[torch.Tensor], targets: Optional[torch.Tensor],
                      targets_out: Optional[torch.Tensor], params: torch.Tensor, canvas_hw=(0, 0)) -> None:
    """yb_v5_rescale_coords: `boxes` [n, D, 4] float32 (slots below `counts` [n] int32) rescaled in place by the
    per-image `params` [n, 5] (gain, pad_w, pad_h, h0, w0); `targets` [T, 6] normalised to the canvas_hw canvas into
    `targets_out` as native xyxy.  Contiguous CUDA tensors of one device; one launch, nothing synchronises."""
    r = V5Rescale()
    dev = params.device
    r.params = params.data_ptr()
    r.n = int(params.shape[0])
    if boxes is not None:
        r.boxes, r.counts, r.D = boxes.data_ptr(), counts.data_ptr(), int(boxes.shape[1])
    if targets is not None:
        r.targets, r.targets_out, r.T = targets.data_ptr(), targets_out.data_ptr(), int(targets.shape[0])
    r.canvas_h, r.canvas_w = float(canvas_hw[0]), float(canvas_hw[1])
    with device_guard(dev):
        check(lib().yb_v5_rescale_coords(ctypes.byref(r), current_stream_ptr(dev)), "yb_v5_rescale_coords")


def v5_compose(samples, tensors: Sequence[torch.Tensor], device: torch.device) -> None:
    """Runs the training-sample descriptors `samples` (V5Sample array, pointers set) in one launch; `tensors` are the
    placed images and the outputs they point into.  Nothing synchronises."""
    n = len(samples)
    blocks = ctypes.c_int64(0)
    check(lib().yb_v5_compose_prepare(n, samples, ctypes.byref(blocks)), "yb_v5_compose_prepare")
    with device_guard(device):
        d_samples = _descs_to_device(samples, device)
        check(lib().yb_v5_compose(n, d_samples.data_ptr(), blocks.value, current_stream_ptr(device)), "yb_v5_compose")
        _keep_alive(tensors, device)


def wgrad_problems(specs) -> "ctypes.Array":
    """yb_wgrad_problem array from (dy [P, >= Cout], x [P, >= Cin], dw [Cout, Cin], db [Cout] or None) tuples of
    row-major device tensors (unit column stride); dtypes are read from the tensors."""
    probs = (WgradProblem * len(specs))()
    for pr, (dy, x, dw, db) in zip(probs, specs):
        for t, what in ((dy, "dy"), (x, "x")):
            if t.dim() != 2 or t.stride(1) != 1:
                raise ValueError(f"conv_wgrad: {what} must be a [P, C] view with unit column stride")
        if not dw.is_contiguous() or (db is not None and not db.is_contiguous()):
            raise ValueError("conv_wgrad: dw and db must be contiguous")
        pr.dtype, pr.out_dtype = dtype_code(dy.dtype), dtype_code(dw.dtype)
        pr.P, pr.Cout, pr.Cin = int(dy.shape[0]), int(dw.shape[0]), int(dw.shape[1])
        pr.dy, pr.dy_stride = dy.data_ptr(), int(dy.stride(0))
        pr.x, pr.x_stride = x.data_ptr(), int(x.stride(0))
        pr.dw, pr.db = dw.data_ptr(), (db.data_ptr() if db is not None else None)
        if int(x.shape[0]) != pr.P or dy.dtype != x.dtype:
            raise ValueError("conv_wgrad: dy and x must have the same rows and dtype")
        if db is not None and db.dtype != dw.dtype:
            raise ValueError("conv_wgrad: db must have the dtype of dw")
    return probs


def conv_wgrad_config(probs) -> dict:
    """How yb_conv_wgrad splits these problems (host-only): launch shape and, per problem, tiles and pixel slices."""
    n = len(probs)
    info = (ctypes.c_int32 * (8 + 4 * n))()
    check(lib().yb_conv_wgrad_config(probs, n, info), "yb_conv_wgrad_config")
    v = [int(x) for x in info]
    keys = ("items", "grid", "smem_bytes", "stages", "stage_pixels", "tile_rows", "tile_cols", "reduce_blocks")
    cfg = dict(zip(keys, v[:8]))
    cfg["problems"] = [dict(zip(("co_tiles", "ci_tiles", "slices", "slice_len"), v[8 + 4 * q: 12 + 4 * q]))
                       for q in range(n)]
    cfg["workspace_bytes"] = int(lib().yb_conv_wgrad_workspace_bytes(probs, n))
    return cfg


def conv_wgrad(specs, device: torch.device) -> None:
    """yb_conv_wgrad on `device`'s current stream: writes dw (and db) of every (dy, x, dw, db) problem; the fp32
    workspace comes from torch's caching allocator.  Nothing is synchronised."""
    probs = wgrad_problems(specs)
    n = len(probs)
    ws_bytes = int(lib().yb_conv_wgrad_workspace_bytes(probs, n))
    if ws_bytes == 0:
        raise NativeLibraryError(f"conv_wgrad: {lib().yb_last_error().decode('utf-8', 'replace')}")
    with device_guard(device):
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
        check(lib().yb_conv_wgrad(probs, n, ws.data_ptr(), ws_bytes, current_stream_ptr(device)), "yb_conv_wgrad")


# ---------------------------------------------------------------------------------------------------
# AutoAnchor (csrc/autoanchor.cu)
YB_AA_MAX_ANCHORS = 64
YB_AA_METRIC_WORKSPACE = 65536


def anchor_metric(wh: torch.Tensor, anchors: torch.Tensor, thr: float, f64: bool):
    """(counts int64[2], sums float64[3]) of the ratio metric: labels with best > thr, (label, anchor) pairs with
    x > thr; sum x, sum best, sum of the x > thr.  wh: float32 [n, 2] on the device; anchors: float64 [na, 2] (holding
    float32 values when f64 is False)."""
    require_cuda(wh, "anchor_metric")
    dev = wh.device
    anchors = anchors.to(dev, torch.float64).contiguous()
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    sums = torch.empty(3, dtype=torch.float64, device=dev)
    ws = torch.empty(YB_AA_METRIC_WORKSPACE, dtype=torch.uint8, device=dev)
    with device_guard(dev):
        check(lib().yb_anchor_metric(wh.data_ptr(), wh.shape[0], anchors.data_ptr(), anchors.shape[0], int(f64),
                                     float(thr), counts.data_ptr(), sums.data_ptr(), ws.data_ptr(), ws.numel(),
                                     current_stream_ptr(dev)), "yb_anchor_metric")
    return counts, sums


def kmeans(obs: torch.Tensor, guesses: torch.Tensor, thresh: float = 1e-5, check_every: int = 8):
    """scipy.cluster.vq._kmeans from each starting book guesses[t] (float64 [trials, k, 2]) over the float64 [n, 2]
    observations on the device: (books [trials, k, 2], sizes int32 [trials], distortions float64 [trials], iterations)."""
    require_cuda(obs, "kmeans")
    dev = obs.device
    trials, k = int(guesses.shape[0]), int(guesses.shape[1])
    guesses = guesses.to(dev, torch.float64).contiguous()
    books = torch.empty_like(guesses)
    sizes = torch.empty(trials, dtype=torch.int32, device=dev)
    dist = torch.empty(trials, dtype=torch.float64, device=dev)
    nbytes = lib().yb_kmeans_workspace_bytes(obs.shape[0], k, trials)
    if nbytes == 0:
        raise ValueError(f"kmeans: {obs.shape[0]} observations, {k} codes, {trials} trials")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    iters = ctypes.c_int32(0)
    with device_guard(dev):
        check(lib().yb_kmeans(obs.data_ptr(), obs.shape[0], k, trials, guesses.data_ptr(), float(thresh), int(check_every),
                              books.data_ptr(), sizes.data_ptr(), dist.data_ptr(), ctypes.byref(iters), ws.data_ptr(),
                              nbytes, current_stream_ptr(dev)), "yb_kmeans")
    return books, sizes, dist, iters.value


def anchor_evolve(wh: torch.Tensor, k0: torch.Tensor, v: torch.Tensor, thr: float, unit_exp: int):
    """kmean_anchors' evolution on the device: (k float64 [na, 2], fitness float32 [gen + 1], accepted uint8 [gen])."""
    require_cuda(wh, "anchor_evolve")
    dev = wh.device
    k0 = k0.to(dev, torch.float64).contiguous()
    v = v.to(dev, torch.float64).contiguous()
    gen = int(v.shape[0])
    k = torch.empty_like(k0)
    fit = torch.empty(gen + 1, dtype=torch.float32, device=dev)
    acc = torch.empty(max(gen, 1), dtype=torch.uint8, device=dev)
    ws = torch.empty(gen + 1, dtype=torch.int64, device=dev)
    with device_guard(dev):
        check(lib().yb_anchor_evolve(wh.data_ptr(), wh.shape[0], k0.shape[0], k0.data_ptr(), v.data_ptr(), gen,
                                     float(thr), int(unit_exp), fit.data_ptr(), acc.data_ptr(), k.data_ptr(),
                                     ws.data_ptr(), ws.numel() * 8, current_stream_ptr(dev)), "yb_anchor_evolve")
    return k, fit, acc[:gen]


# ---------------------------------------------------------------------------------------------------
# YOLOv5 validation metrics (csrc/v5_metrics.cu)
YB_V5M_RECORD_INT32, YB_V5M_MAX_IOU, YB_V5M_CURVE_POINTS, YB_V5M_AP_POINTS, YB_V5M_NUM_PARAMS = 4, 31, 1000, 101, 1101
YB_V5M_ST_BAD_IMAGE, YB_V5M_ST_BAD_TARGET_CLASS, YB_V5M_ST_BAD_DET_CLASS = 1, 2, 4
YB_V5M_ST_BAD_COUNT, YB_V5M_ST_TP_EXCEEDS_LABELS = 8, 16


def v5m_match(boxes: torch.Tensor, scores: torch.Tensor, classes: torch.Tensor, counts: torch.Tensor,
              targets: torch.Tensor, order: torch.Tensor, start: torch.Tensor, nc: int, iouv: torch.Tensor,
              conf_thr: float, iou_thr: float, records: torch.Tensor, label_count: Optional[torch.Tensor],
              matrix: Optional[torch.Tensor], status: torch.Tensor, cm_empty_rows: bool = False) -> None:
    """yb_v5m_match on the current stream of `records`' device: boxes fp32 [n,d,4], scores / classes fp32 [n,d], counts
    int32 [n], targets fp32 [T,6], order int64 [T], start int64 [n+1], iouv fp32 [n_iou]; records int32 [n*d, 4],
    label_count int32 [nc] or None, matrix int64 [(nc+1)^2] or None, status int32 [1].  Nothing is synchronised."""
    dev = records.device
    if dev.type != "cuda":
        raise NativeLibraryError("v5m_match runs on a CUDA device only (no CPU fallback)")
    n, d = int(scores.shape[0]), int(scores.shape[1])
    T = int(targets.shape[0])
    ts = [(boxes, torch.float32), (scores, torch.float32), (classes, torch.float32), (counts, torch.int32),
          (targets, torch.float32), (order, torch.int64), (start, torch.int64), (iouv, torch.float32),
          (records, torch.int32), (status, torch.int32)]
    ts += [(t, dt) for t, dt in ((label_count, torch.int32), (matrix, torch.int64)) if t is not None]
    for t, dt in ts:
        if t.device != dev or t.dtype != dt or not t.is_contiguous():
            raise NativeLibraryError(f"v5m_match: every tensor must be a contiguous {dt} tensor on {dev}")
    if tuple(boxes.shape) != (n, d, 4) or tuple(classes.shape) != (n, d) or counts.numel() != n \
            or tuple(targets.shape) != (T, 6) or order.numel() != T or start.numel() != n + 1 \
            or tuple(records.shape) != (n * d, YB_V5M_RECORD_INT32):
        raise NativeLibraryError("v5m_match: shapes do not agree")
    ws_bytes = int(lib().yb_v5m_match_workspace_bytes(T))
    with device_guard(dev):
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        check(lib().yb_v5m_match(n, d, boxes.data_ptr(), scores.data_ptr(), classes.data_ptr(), counts.data_ptr(),
                                 targets.data_ptr(), T, order.data_ptr(), start.data_ptr(), nc, iouv.data_ptr(),
                                 iouv.numel(), conf_thr, iou_thr, int(cm_empty_rows), records.data_ptr(),
                                 label_count.data_ptr() if label_count is not None else None,
                                 matrix.data_ptr() if matrix is not None else None, status.data_ptr(), ws.data_ptr(),
                                 ws_bytes, current_stream_ptr(dev)), "yb_v5m_match")


def v5m_ap(records: torch.Tensor, nc: int, n_iou: int, label_count: torch.Tensor, params: torch.Tensor,
           status: torch.Tensor):
    """yb_v5m_ap: records int32 [n, 4], label_count int32 [nc], params float64 [1101], status int32 [1], on one CUDA
    device.  Returns float64 device tensors ap [nc, n_iou], p [nc, 1000], r [nc, 1000].  Nothing is synchronised."""
    dev = records.device
    if dev.type != "cuda":
        raise NativeLibraryError("v5m_ap runs on a CUDA device only (no CPU fallback)")
    for t, dt in ((records, torch.int32), (label_count, torch.int32), (params, torch.float64), (status, torch.int32)):
        if t.device != dev or t.dtype != dt or not t.is_contiguous():
            raise NativeLibraryError(f"v5m_ap: expected a contiguous {dt} tensor on {dev}")
    if label_count.numel() != nc or params.numel() != YB_V5M_NUM_PARAMS:
        raise NativeLibraryError("v5m_ap: label_count / params have the wrong size")
    n = int(records.shape[0])
    with device_guard(dev):
        ws_bytes = int(lib().yb_v5m_ap_workspace_bytes(n, nc))
        if ws_bytes == 0:
            raise NativeLibraryError(f"v5m_ap: no workspace size for {n} records and {nc} classes")
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        ap = torch.empty((nc, n_iou), dtype=torch.float64, device=dev)
        p = torch.empty((nc, YB_V5M_CURVE_POINTS), dtype=torch.float64, device=dev)
        r = torch.empty_like(p)
        check(lib().yb_v5m_ap(records.data_ptr() if n else None, n, nc, n_iou, label_count.data_ptr(),
                              params.data_ptr(), ap.data_ptr(), p.data_ptr(), r.data_ptr(), status.data_ptr(),
                              ws.data_ptr(), ws_bytes, current_stream_ptr(dev)), "yb_v5m_ap")
    return ap, p, r
