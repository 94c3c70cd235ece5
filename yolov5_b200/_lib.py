"""ctypes binding of liby5b200.so (the C ABI declared in include/y5b200.h).

There is no CPU or PyTorch fallback behind these calls: if the shared object is missing or a call fails, a
RuntimeError is raised with the library's own message.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("Y5B200_LIB") or os.path.join(_HERE, "liby5b200.so")  # env override: A/B experiments only

Y5_F16, Y5_BF16, Y5_F32, Y5_U8 = 0, 1, 2, 3
ACT_NONE, ACT_SILU, ACT_LEAKY = 0, 1, 2  # include/y5b200.h Y5_ACT_*
POOL_K2S2, POOL_K2S1_ZPAD = 0, 1  # include/y5b200.h Y5_POOL_*

_DTYPE = {torch.float16: Y5_F16, torch.bfloat16: Y5_BF16, torch.float32: Y5_F32, torch.uint8: Y5_U8}


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPE[dt]
    except KeyError:
        raise TypeError(f"y5b200: unsupported dtype {dt}") from None


class ConvDesc(C.Structure):
    _fields_ = [
        ("inp", C.c_void_p), ("in_pitch", C.c_int32),
        ("batch", C.c_int32), ("in_h", C.c_int32), ("in_w", C.c_int32), ("in_c", C.c_int32),
        ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("out", C.c_void_p), ("out_pitch", C.c_int32), ("out_c", C.c_int32),
        ("residual", C.c_void_p), ("res_pitch", C.c_int32),
        ("ksize", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("act", C.c_int32), ("dtype", C.c_int32), ("block_k", C.c_int32), ("block_n", C.c_int32),
        ("kw", C.c_int32), ("pad_w", C.c_int32),
        ("in_x_stride", C.c_int64), ("in_y_stride", C.c_int64), ("in_n_stride", C.c_int64),
        ("a_mode", C.c_int32), ("reserved", C.c_int32), ("act_slope", C.c_float),
    ]


class DetectDesc(C.Structure):
    _fields_ = [
        ("inp", C.c_void_p), ("in_pitch", C.c_int32),
        ("batch", C.c_int32), ("ny", C.c_int32), ("nx", C.c_int32), ("in_c", C.c_int32),
        ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("raw", C.c_void_p), ("z", C.c_void_p),
        ("z_rows", C.c_int32), ("z_row0", C.c_int32),
        ("na", C.c_int32), ("no", C.c_int32), ("nc", C.c_int32),
        ("stride", C.c_float), ("anchor_wh", C.c_float * 8),
        ("dtype", C.c_int32), ("block_k", C.c_int32),
    ]


class PlanInfo(C.Structure):
    _fields_ = [
        ("a_mode", C.c_int32), ("tw", C.c_int32), ("th", C.c_int32),
        ("block_k", C.c_int32), ("block_n", C.c_int32), ("mt", C.c_int32), ("cluster", C.c_int32),
        ("patch_pw", C.c_int32), ("b_grouped", C.c_int32), ("staged", C.c_int32), ("opt", C.c_int32), ("epi", C.c_int32),
        ("a_stages", C.c_int32), ("b_stages", C.c_int32), ("grid", C.c_int32),
        ("tma_epi", C.c_int32),
    ]

    def as_dict(self) -> dict:
        return {f: getattr(self, f) for f, _ in self._fields_}


class NmsParams(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("n_rows", C.c_int32), ("no", C.c_int32), ("nc", C.c_int32), ("nm", C.c_int32),
        ("dtype", C.c_int32), ("conf_thres", C.c_float), ("iou_thres", C.c_float),
        ("multi_label", C.c_int32), ("agnostic", C.c_int32), ("max_det", C.c_int32), ("max_nms", C.c_int32),
        ("max_wh", C.c_float), ("classes", C.c_void_p), ("n_classes", C.c_int32),
    ]


class LossParams(C.Structure):
    _fields_ = [
        ("nl", C.c_int32), ("batch", C.c_int32), ("na", C.c_int32), ("no", C.c_int32), ("nc", C.c_int32),
        ("ny", C.c_int32 * 5), ("nx", C.c_int32 * 5),
        ("dtype", C.c_int32), ("nt", C.c_int32),
        ("anchor_t", C.c_float), ("box_gain", C.c_float), ("obj_gain", C.c_float), ("cls_gain", C.c_float),
        ("cls_pw", C.c_float), ("obj_pw", C.c_float), ("cp", C.c_float), ("cn", C.c_float),
        ("balance", C.c_float * 5), ("grad_scale", C.c_float),
    ]


class WgradDesc(C.Structure):
    _fields_ = [
        ("inp", C.c_void_p), ("in_pitch", C.c_int32),
        ("batch", C.c_int32), ("in_h", C.c_int32), ("in_w", C.c_int32), ("in_c", C.c_int32),
        ("dout", C.c_void_p), ("dout_pitch", C.c_int32), ("out_c", C.c_int32),
        ("dweight", C.c_void_p),
        ("ksize", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("dtype", C.c_int32), ("accumulate", C.c_int32), ("reserved", C.c_int32),
        ("kw", C.c_int32), ("pad_w", C.c_int32),
        ("in_x_stride", C.c_int64), ("in_y_stride", C.c_int64), ("in_n_stride", C.c_int64),
    ]


class LetterboxImage(C.Structure):
    _fields_ = [
        ("data", C.c_void_p), ("src_h", C.c_int32), ("src_w", C.c_int32), ("row_bytes", C.c_int32),
        ("new_h", C.c_int32), ("new_w", C.c_int32), ("top", C.c_int32), ("left", C.c_int32),
    ]


class ValImage(C.Structure):
    _fields_ = [
        ("data", C.c_void_p), ("scratch", C.c_void_p), ("src_h", C.c_int32), ("src_w", C.c_int32), ("row_bytes", C.c_int32),
        ("res_h", C.c_int32), ("res_w", C.c_int32), ("interp", C.c_int32), ("new_h", C.c_int32), ("new_w", C.c_int32),
        ("top", C.c_int32), ("left", C.c_int32),
    ]


VAL_COPY, VAL_LINEAR, VAL_AREA = 0, 1, 2  # include/y5b200.h Y5_VAL_*


class ClsImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("side", C.c_int32), ("row_bytes", C.c_int32)]


class OptTensor(C.Structure):
    _fields_ = [
        ("param", C.c_void_p), ("grad", C.c_void_p), ("mom", C.c_void_p), ("ema", C.c_void_p),
        ("numel", C.c_int64), ("group", C.c_int32), ("reserved", C.c_int32),
    ]


class PackItem(C.Structure):
    _fields_ = [
        ("w", C.c_void_p), ("fwd", C.c_void_p), ("dgrad", C.c_void_p), ("w_dtype", C.c_int32),
        ("out_c", C.c_int32), ("in_c", C.c_int32), ("ksize", C.c_int32), ("in_c_pad", C.c_int32), ("out_c_pad", C.c_int32),
    ]


class AugTile(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("row_bytes", C.c_int32), ("pixel_stride", C.c_int32), ("channel_stride", C.c_int32),
        ("x1a", C.c_int32), ("y1a", C.c_int32), ("x2a", C.c_int32), ("y2a", C.c_int32), ("dx", C.c_int32), ("dy", C.c_int32),
        ("reserved", C.c_int32),
    ]


class AugImage(C.Structure):
    _fields_ = [
        ("inv_m", (C.c_double * 6) * 2), ("m", (C.c_double * 6) * 2), ("mix_r", C.c_double), ("scale", C.c_float * 2),
        ("clip_max", C.c_float), ("n_mosaic", C.c_int32), ("n_tiles", C.c_int32 * 2), ("canvas_w", C.c_int32), ("canvas_h", C.c_int32),
        ("warp", C.c_int32 * 2), ("hsv", C.c_int32), ("flipud", C.c_int32), ("fliplr", C.c_int32), ("reserved", C.c_int32),
        ("tiles", AugTile * 8), ("lut", (C.c_uint8 * 256) * 3),
    ]


class AugLabel(C.Structure):
    _fields_ = [
        ("cls", C.c_float), ("x", C.c_float), ("y", C.c_float), ("w", C.c_float), ("h", C.c_float),
        ("tile_w", C.c_float), ("tile_h", C.c_float), ("pad_w", C.c_float), ("pad_h", C.c_float),
        ("image", C.c_int32), ("mosaic", C.c_int32), ("flags", C.c_int32),
    ]


AUG_CLIP, AUG_IN_XYXY, AUG_OUT_XYXY = 1, 2, 4  # y5_aug_label.flags (include/y5b200.h Y5_AUG_*)


class AugSegment(C.Structure):
    _fields_ = [("point_offset", C.c_int32), ("n_points", C.c_int32)]


SEG_POINTS, SEG_I32 = 1000, 4  # include/y5b200.h Y5_SEG_POINTS, Y5_SEG_I32

# indices into the fused optimizer's `hyper` array (include/y5b200.h Y5_OPT_*)
OPT_INV_SCALE, OPT_MAX_NORM, OPT_EMA_DECAY, OPT_EMA_TAU, OPT_EMA_UPDATES, OPT_OUT_NORM, OPT_OUT_SKIPPED, OPT_GROUPS = 0, 1, 2, 3, 4, 5, 6, 8
# per-group block of y5_adam_step's fp64 `group_hyper` (include/y5b200.h Y5_ADAM_*)
ADAM_LR, ADAM_BETA1, ADAM_BETA2, ADAM_EPS, ADAM_WEIGHT_DECAY, ADAM_DECOUPLED, ADAM_STRIDE = 0, 1, 2, 3, 4, 5, 8

_P = C.c_void_p
_I32, _I64, _F = C.c_int32, C.c_int64, C.c_float
# name -> (restype, argtypes); mirrors include/y5b200.h one to one (tests/test_abi.py checks the header against this)
SIGNATURES = {
    "y5_version": (_I32, []),
    "y5_last_error": (C.c_char_p, []),
    "y5_launch_count": (_I64, []),
    "y5_conv_pick": (_I32, [_I32, _I32, _I64, C.POINTER(_I32), C.POINTER(_I32)]),
    "y5_conv_plan_create": (_I32, [C.POINTER(ConvDesc), C.POINTER(_P)]),
    "y5_conv_plan_run": (_I32, [_P, _P]),
    "y5_conv_plan_destroy": (None, [_P]),
    "y5_conv_plan_info": (_I32, [_P, C.POINTER(PlanInfo)]),
    "y5_conv_bn_silu_fwd": (_I32, [C.POINTER(ConvDesc), _P]),
    "y5_conv_direct_fwd": (_I32, [C.POINTER(ConvDesc), _P]),
    "y5_detect_plan_create": (_I32, [C.POINTER(DetectDesc), C.POINTER(_P)]),
    "y5_detect_plan_run": (_I32, [_P, _P]),
    "y5_detect_plan_run_to": (_I32, [_P, _P, _P, _P]),
    "y5_detect_plan_destroy": (None, [_P]),
    "y5_stem_s2d": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_sppf_pool": (_I32, [_P, _I32, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_upsample2x": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_copy_view": (_I32, [_P, _I32, _P, _I32, _I64, _I32, _I32, _P]),
    "y5_nhwc_to_nchw": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_nms_workspace_bytes": (_I64, [C.POINTER(NmsParams)]),
    "y5_nms_batched": (_I32, [C.POINTER(NmsParams), _P, _P, _P, _P, _P, _I64, _P]),
    "y5_box_iou": (_I32, [_P, _I32, _P, _I32, _F, _P, _P]),
    "y5_loss_workspace_bytes": (_I64, [C.POINTER(LossParams)]),
    "y5_loss_fwd_bwd": (_I32, [C.POINTER(LossParams), C.POINTER(_P), _P, _P, _P, C.POINTER(_P), _P, _I64, _P]),
    "y5_loss_read_targets": (_I32, [C.POINTER(LossParams), _P, _I32, _P, _P, _P, _P]),
    "y5_seg_loss_workspace_bytes": (_I64, [C.POINTER(LossParams)]),
    "y5_seg_loss_fwd_bwd_scaled": (_I32, [C.POINTER(LossParams), C.POINTER(_P), _P, _P, _P, _I32, _I64, _I64, _I64, _I64, _I32, _I32, _I32,
                                          _P, _I32, _I32, _I32, _I32, _P, C.POINTER(_P), _P, _P, _P, _I64, _P]),
    "y5_seg_loss_read_targets": (_I32, [C.POINTER(LossParams), _P, _I32, _P, _P, _P, _P]),
    "y5_conv_wgrad": (_I32, [C.POINTER(WgradDesc), _P]),
    "y5_bn_workspace_bytes": (_I64, [_I32]),
    "y5_bn_stats": (_I32, [_P, _I32, _I64, _I32, _I32, _P, _P]),
    "y5_bn_act_fwd": (_I32, [_P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _P, _F, _F, _P, _P, _P, _I32, _P]),
    "y5_upsample2x_bwd": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_sppf_bwd_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32]),
    "y5_sppf_pool_bwd": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P]),
    "y5_bn_act_bwd": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _P, _P, _P, _P]),
    "y5_col_sum": (_I32, [_P, _I32, _I64, _I32, _I32, _P, _P, _P]),
    "y5_bn_stats_sync": (_I32, [_P, _I32, _I64, _I32, _I32, _P, _P]),
    "y5_bn_act_fwd_sync": (_I32, [_P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _P, _F, _F, _P, _P, _P, _I32, _P]),
    "y5_bn_act_bwd_reduce": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _P, _P, _P, _P]),
    "y5_bn_act_bwd_apply": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _I32, _P, _P, _P]),
    "y5_bn_act_fwd_ex": (_I32, [_P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _F, _P, _F, _F, _P, _P, _P, _I32, _P]),
    "y5_bn_act_bwd_ex": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _F, _P, _P, _P, _P]),
    "y5_bn_act_fwd_sync_ex": (_I32, [_P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _F, _P, _F, _F, _P, _P, _P, _I32, _P]),
    "y5_bn_act_bwd_reduce_ex": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _F, _P, _P, _P, _P]),
    "y5_weight_pack": (_I32, [_P, _I32, _I32, _I32, _I32, _P, _I32, _P, _I32, _I32, _P]),
    "y5_weight_pack_chunk_elems": (_I32, []),
    "y5_weight_pack_multi": (_I32, [_P, _P, _P, _I32, _I32, _P]),
    "y5_zero_stuff2x": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_loss_fwd_bwd_scaled": (_I32, [C.POINTER(LossParams), C.POINTER(_P), _P, _P, _P, C.POINTER(_P), _P, _P, _I64, _P]),
    "y5_letterbox_max_images": (_I32, []),
    "y5_letterbox": (_I32, [C.POINTER(LetterboxImage), _I32, _I32, _I32, _I32, _I32, _P, _I32, _I32, _I32, _I32, _P]),
    "y5_val_letterbox": (_I32, [C.POINTER(ValImage), _I32, _I32, _I32, _P, _I32, _P]),
    "y5_cls_batch": (_I32, [_P, _I32, _I32, _I32, C.POINTER(_F), C.POINTER(_F), _P, _I32, _P]),
    "y5_process_mask_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32]),
    "y5_process_mask": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, C.POINTER(_I32), _P, _I32, _P, _I64,
                                _P]),
    "y5_crop_mask": (_I32, [_P, _P, _I32, _I32, _I32, _I32, _P, _P]),
    "y5_scale_boxes": (_I32, [_P, _I32, _I64, _P, _I32, _P, _P, _P]),
    "y5_labels_native": (_I32, [_P, _I32, _P, _P, _P]),
    "y5_match_batch": (_I32, [_P, _I64, _I32, _P, _I32, _I32, _P, _I32, _P, _I32, _F, _P, _P]),
    "y5_confusion_batch": (_I32, [_P, _I64, _I32, _P, _I32, _I32, _P, _I32, _I32, _F, _F, _F, _P, _P, _P]),
    "y5_mask_row_words": (_I32, [_I32, _I32]),
    "y5_mask_pack": (_I32, [_P, _I32, _I32, _I32, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P]),
    "y5_mask_iou": (_I32, [_P, _P, _P, _I32, _P, _P, _P, _I32, _I32, _I32, _I32, _F, _P, _P]),
    "y5_mask_match_batch": (_I32, [_P, _I64, _I32, _P, _I32, _I32, _P, _I32, _P, _I32, _P, _P, _I32, _P, _P]),
    "y5_opt_chunk_elems": (_I32, []),
    "y5_opt_step": (_I32, [_P, _P, _P, _I32, _P, _P, _I32, _I32, _I32, _P]),
    "y5_adam_step": (_I32, [_P, _I32, _P, _P, _I32, _P, _P, _I64, _P, _P, _I32, _I32, _P]),
    "y5_grad_pack": (_I32, [_P, _P, _P, _I32, _P, _P, _P, _P]),
    "y5_grad_bind": (_I32, [_P, _I32, _P, _P, _P, _P]),
    "y5_aug_gather": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _I32, _I32, _I32, _I32, _P]),
    "y5_aug_labels": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _P, _P, _P]),
    "y5_seg_warp": (_I32, [_P, _I32, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P, _P]),
    "y5_seg_raster": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _P, _P, _P]),
    "y5_seg_order": (_I32, [_P, _I32, _P, _P, _P, _I32, _P, _P, _P, _P]),
    "y5_seg_compose": (_I32, [_P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _I32, _P]),
    "y5_fold_pack": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _I32, _F, _P, _I32, _I32, _P, _I32, _P]),
    "y5_global_avg_pool": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_global_avg_pool_bwd": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_cross_entropy": (_I32, [_P, _I32, _I32, _I32, _I64, _P, _F, _P, _P, _I64, _P, _P, _P]),
    "y5_ap_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32, _I32]),
    "y5_ap_per_class": (_I32, [_P, _P, _I64, _I32, _P, _P, _I64, _I32, _P, _I32, _I32, _I32, _P, _I32, _P, C.c_double, _P, _I64, _P, _P, _P]),
    "y5_attention_fwd": (_I32, [_P, _P, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _F, _I32, _P]),
    "y5_attention_bwd": (_I32, [_P, _P, _P, _I32, _P, _I32, _P, _I32, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _F, _I32, _P]),
    "y5_image_nhwc": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_maxpool2d": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_maxpool2d_bwd": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "y5_spp_bwd_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32]),
    "y5_spp_pool_bwd": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P]),
    "y5_dwconv_fwd": (_I32, [_P, _I32, _P, _P, _P, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _F, _I32,
                             _I32, _P]),
    "y5_dwconv_wgrad": (_I32, [_P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
}

AP_META = 5  # include/y5b200.h Y5_AP_META

_lib = None


def lib():
    """Load liby5b200.so (once).  Fails loudly: there is no fallback implementation."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"y5b200: {LIB_PATH} not found -- build it with `python -m yolov5_b200.build` "
                "(or __graft_entry__.build()); this engine has no CPU / PyTorch fallback"
            )
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError here == header/library mismatch: also loud
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib().y5_last_error().decode(errors="replace")
        raise RuntimeError(f"y5b200 {what} failed (code {code}): {msg}")


def stream_ptr(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def on(device):
    """Device guard for the entry points: the C ABI launches on the CURRENT CUDA device, so a model / tensor living on
    cuda:1 while cuda:0 is current must switch first (per-device kernel attributes are handled inside the library)."""
    return torch.cuda.device(device)


def launch_count() -> int:
    return int(lib().y5_launch_count())
