"""ctypes binding of libstreamyolo_sm100.so (include/streamyolo_sm100.h) + NHWC view helper.

The library is the product; there is NO fallback: if it is missing or the device is not an
sm_90 part, every op raises RuntimeError.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libstreamyolo_sm100.so")

SY_CONV_RAW, SY_CONV_FUSED = 0, 1
SY_STORAGE_BF16, SY_STORAGE_F16 = 0, 1
SY_PACK_F16 = 0x100
SY_ACT_NONE, SY_ACT_SILU, SY_ACT_RELU, SY_ACT_LRELU = 0, 1, 2, 3
ACT_CODES = {"silu": SY_ACT_SILU, "relu": SY_ACT_RELU, "lrelu": SY_ACT_LRELU}    # [yolox] act name -> the kernels' act code
STORAGE = {torch.bfloat16: SY_STORAGE_BF16, torch.float16: SY_STORAGE_F16}    # activation dtype -> SyConvDesc.storage


class SyTensor(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
                ("pitch", C.c_int64)]


class SyBnSegment(C.Structure):
    _fields_ = [("gamma", C.c_void_p), ("beta", C.c_void_p), ("running_mean", C.c_void_p),
                ("running_var", C.c_void_p), ("num_batches_tracked", C.c_void_p), ("c_begin", C.c_int32)]


class SyConvDesc(C.Structure):
    _fields_ = [("x", SyTensor), ("y", SyTensor), ("w", C.c_void_p), ("kh", C.c_int32), ("kw", C.c_int32),
                ("stride", C.c_int32), ("mode", C.c_int32), ("act", C.c_int32), ("scale", C.c_void_p),
                ("shift", C.c_void_p), ("res", SyTensor), ("split_n", C.c_int32), ("stat_partials", C.c_void_p),
                ("n_partials", C.c_int32), ("rows_written", C.POINTER(C.c_int32)), ("bn", SyBnSegment * 2),
                ("momentum", C.c_float), ("eps", C.c_float), ("scale_shift", C.c_void_p), ("mean_invstd", C.c_void_p),
                ("sync", C.c_void_p), ("debug_timeline", C.c_void_p),
                ("debug_timeline_events", C.c_int32), ("debug_flags", C.c_int32), ("debug_f32", C.c_void_p),
                ("tile_mode", C.c_int32), ("tile_bn", C.c_int32), ("stat_updates", C.c_int32), ("storage", C.c_int32)]


class SyHeadPredDesc(C.Structure):
    _fields_ = [("cls_feat", SyTensor), ("reg_feat", SyTensor),
                ("w_reg", C.c_void_p), ("b_reg", C.c_void_p), ("w_obj", C.c_void_p), ("b_obj", C.c_void_p),
                ("w_cls", C.c_void_p), ("b_cls", C.c_void_p),
                ("num_classes", C.c_int32), ("stride", C.c_int32), ("anchor_offset", C.c_int32),
                ("a_total", C.c_int32), ("sigmoid", C.c_int32), ("decode", C.c_int32),
                ("out", C.c_void_p), ("origin", C.c_void_p), ("storage", C.c_int32)]


class SyTalLossDesc(C.Structure):
    _fields_ = [("b", C.c_int32), ("a_total", C.c_int32), ("max_labels", C.c_int32), ("num_classes", C.c_int32),
                ("n_levels", C.c_int32), ("level_h", C.c_int32 * 4), ("level_w", C.c_int32 * 4),
                ("level_stride", C.c_int32 * 4),
                ("outputs", C.c_void_p), ("origin", C.c_void_p), ("labels_fut", C.c_void_p),
                ("labels_cur", C.c_void_p), ("gamma", C.c_float), ("ignore_thr", C.c_float),
                ("ignore_value", C.c_float), ("use_l1", C.c_int32), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t), ("loss_out", C.c_void_p), ("fg_out", C.c_void_p),
                ("matched_out", C.c_void_p), ("pred_iou_out", C.c_void_p)]


class SyConvWgradDesc(C.Structure):
    _fields_ = [("x", SyTensor), ("dy", SyTensor), ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32),
                ("dw", C.c_void_p), ("accumulate", C.c_int32), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t)]


class SyNmsDesc(C.Structure):
    _fields_ = [("pred", C.c_void_p), ("b", C.c_int32), ("a_total", C.c_int32), ("num_classes", C.c_int32),
                ("max_det", C.c_int32), ("conf_thre", C.c_float), ("nms_thre", C.c_float), ("class_agnostic", C.c_int32),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("det_out", C.c_void_p),
                ("count_out", C.c_void_p)]


class SyBnActBwdDesc(C.Structure):
    _fields_ = [("raw", SyTensor), ("dy", SyTensor), ("draw", SyTensor), ("scale", C.c_void_p), ("shift", C.c_void_p),
                ("mean", C.c_void_p), ("invstd", C.c_void_p), ("split_n", C.c_int32), ("act", C.c_int32),
                ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("accumulate", C.c_int32), ("partials", C.c_void_p),
                ("n_partials", C.c_int32), ("coef", C.c_void_p)]


class SyHeadPredBwdDesc(C.Structure):
    _fields_ = [("grad_raw", C.c_void_p), ("cls_feat", SyTensor), ("reg_feat", SyTensor), ("d_cls_feat", SyTensor),
                ("d_reg_feat", SyTensor), ("w_reg", C.c_void_p), ("w_obj", C.c_void_p), ("w_cls", C.c_void_p),
                ("num_classes", C.c_int32), ("a_total", C.c_int32), ("anchor_offset", C.c_int32),
                ("dw_reg", C.c_void_p), ("dw_obj", C.c_void_p), ("dw_cls", C.c_void_p), ("db_reg", C.c_void_p),
                ("db_obj", C.c_void_p), ("db_cls", C.c_void_p), ("accumulate", C.c_int32), ("partials", C.c_void_p),
                ("n_partials", C.c_int32)]


class SySgdEmaDesc(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("momentum_buf", C.c_void_p), ("ema", C.c_void_p),
                ("n_param", C.c_int64), ("n_total", C.c_int64), ("decay_begin", C.c_int64),
                ("lr", C.c_float), ("momentum", C.c_float), ("weight_decay", C.c_float), ("inv_scale", C.c_float),
                ("nesterov", C.c_int32), ("ema_decay", C.c_float), ("ema_one_minus_decay", C.c_float),
                ("found_inf", C.c_void_p), ("hyper", C.c_void_p), ("found_inf_ema", C.c_int32)]


class SyPackItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("out", C.c_void_p), ("cout", C.c_int32), ("cin", C.c_int32), ("kh", C.c_int32),
                ("taps", C.c_int32), ("mode", C.c_int32), ("co_offset", C.c_int32), ("out_pitch", C.c_int64),
                ("begin", C.c_int64)]


class SyConvPlan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mode", "bn", "m_tiles", "n_tiles", "rounds", "kblocks", "patch_h", "patch_w",
                                               "walk", "grid")]


class SyTalLossBwdDesc(C.Structure):
    _fields_ = [("outputs", C.c_void_p), ("origin", C.c_void_p), ("labels_fut", C.c_void_p),
                ("b", C.c_int32), ("a_total", C.c_int32), ("max_labels", C.c_int32), ("num_classes", C.c_int32),
                ("n_levels", C.c_int32), ("level_h", C.c_int32 * 4), ("level_w", C.c_int32 * 4),
                ("level_stride", C.c_int32 * 4), ("gamma", C.c_float), ("use_l1", C.c_int32),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("grad_scale", C.c_float),
                ("grad_outputs", C.c_void_p), ("grad_origin", C.c_void_p), ("grad_raw", C.c_void_p)]


class SyPairLabelsDesc(C.Structure):
    _fields_ = [("ann", C.c_void_p), ("counts", C.c_void_p), ("mirror", C.c_void_p), ("n_items", C.c_int32),
                ("max_rows", C.c_int32), ("max_labels", C.c_int32), ("flip", C.c_int32), ("width", C.c_int32),
                ("r", C.c_double), ("labels_fut", C.c_void_p), ("labels_cur", C.c_void_p), ("flags_out", C.c_void_p)]


class SyFrameLabelsDesc(C.Structure):
    _fields_ = [("ann", C.c_void_p), ("counts", C.c_void_p), ("mirror", C.c_void_p), ("n", C.c_int32),
                ("max_rows", C.c_int32), ("max_labels", C.c_int32), ("flip", C.c_int32), ("width", C.c_int32),
                ("r", C.c_double), ("labels", C.c_void_p), ("flags_out", C.c_void_p)]


class SyLetterboxDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("mid_h", C.c_int32),
                ("mid_w", C.c_int32), ("dst_h", C.c_int32), ("dst_w", C.c_int32), ("out_h", C.c_int32),
                ("out_w", C.c_int32), ("flags", C.c_void_p), ("out", C.c_void_p)]


class SyJpegDecodeDesc(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("lengths", C.c_void_p), ("n", C.c_int32), ("max_bytes", C.c_int64),
                ("h", C.c_int32), ("w", C.c_int32), ("out", C.c_void_p), ("status", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class SyJpegDecodeSizedDesc(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("lengths", C.c_void_p), ("n", C.c_int32), ("max_bytes", C.c_int64),
                ("sizes", C.c_void_p), ("max_h", C.c_int32), ("max_w", C.c_int32), ("out", C.c_void_p),
                ("status", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class SyLetterboxSizedDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("n", C.c_int32), ("slot_h", C.c_int32), ("slot_w", C.c_int32),
                ("sizes", C.c_void_p), ("out_h", C.c_int32), ("out_w", C.c_int32), ("out", C.c_void_p)]


class SyResizeSizedDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("n", C.c_int32), ("slot_h", C.c_int32), ("slot_w", C.c_int32), ("sizes", C.c_void_p),
                ("out_h", C.c_int32), ("out_w", C.c_int32), ("out", C.c_void_p)]


class SyYuvToBgrSizedDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("n", C.c_int32), ("max_bytes", C.c_int64), ("sizes", C.c_void_p),
                ("format", C.c_int32), ("slot_h", C.c_int32), ("slot_w", C.c_int32), ("out", C.c_void_p)]


class SyBayerToBgrSizedDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("n", C.c_int32), ("max_bytes", C.c_int64), ("sizes", C.c_void_p),
                ("pattern", C.c_int32), ("algo", C.c_int32), ("slot_h", C.c_int32), ("slot_w", C.c_int32),
                ("out", C.c_void_p)]


class SyJpegEncodeDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("sizes", C.c_void_p), ("n", C.c_int32), ("max_h", C.c_int32), ("max_w", C.c_int32),
                ("quality", C.c_int32), ("out", C.c_void_p), ("max_bytes", C.c_int64), ("lengths", C.c_void_p),
                ("status", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class SyDrawBoxesDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("sizes", C.c_void_p), ("n", C.c_int32), ("max_h", C.c_int32), ("max_w", C.c_int32),
                ("boxes", C.c_void_p), ("labels", C.c_void_p), ("counts", C.c_void_p), ("K", C.c_int32),
                ("palette", C.c_void_p), ("P", C.c_int32), ("dst", C.c_void_p), ("dst_h", C.c_int32), ("dst_w", C.c_int32)]


class SyDrawOutlinesDesc(C.Structure):
    _fields_ = [("img", C.c_void_p), ("sizes", C.c_void_p), ("n", C.c_int32), ("max_h", C.c_int32), ("max_w", C.c_int32),
                ("boxes", C.c_void_p), ("counts", C.c_void_p), ("K", C.c_int32), ("points", C.c_void_p),
                ("n_points", C.c_void_p), ("M", C.c_int32), ("color", C.c_uint8 * 3)]


class SyVisDetBoxesDesc(C.Structure):
    _fields_ = [("det", C.c_void_p), ("count", C.c_void_p), ("S", C.c_int32), ("A", C.c_int32), ("score_th", C.c_float),
                ("boxes", C.c_void_p), ("labels", C.c_void_p), ("counts", C.c_void_p)]


class SySpliceFramesDesc(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("sizes", C.c_void_p), ("splits", C.c_void_p), ("n", C.c_int32),
                ("max_h", C.c_int32), ("max_w", C.c_int32), ("horizontal", C.c_int32), ("color", C.c_uint8 * 3)]


class SySelectImagesDesc(C.Structure):
    _fields_ = [("src", SyTensor * 3), ("dst", SyTensor * 3), ("n_pairs", C.c_int32), ("flags", C.c_void_p)]


class SyCocoRowsDesc(C.Structure):
    _fields_ = [("det", C.c_void_p), ("b", C.c_int32), ("max_det", C.c_int32), ("count", C.c_void_p), ("ratio", C.c_void_p),
                ("image_id", C.c_void_p), ("status", C.c_void_p), ("frames_per_image", C.c_int32),
                ("num_classes", C.c_int32), ("class_ids", C.c_void_p), ("bbox_out", C.c_void_p),
                ("score_out", C.c_void_p), ("image_id_out", C.c_void_p), ("category_out", C.c_void_p),
                ("total_out", C.c_void_p)]


class SyForecastState(C.Structure):
    _fields_ = [("x", C.c_void_p), ("P", C.c_void_p), ("label", C.c_void_p), ("score", C.c_void_p), ("track", C.c_void_p),
                ("meta", C.c_void_p), ("S", C.c_int32), ("T", C.c_int32)]


class SyForecastUpdateDesc(C.Structure):
    _fields_ = [("state", SyForecastState), ("det", C.c_void_p), ("max_det", C.c_int32), ("count", C.c_void_p),
                ("dt", C.c_void_p), ("start", C.c_void_p), ("keep", C.c_void_p), ("match_iou_th", C.c_double),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("clear_on_empty", C.c_int32)]


class SyForecastExtrapDesc(C.Structure):
    _fields_ = [("state", SyForecastState), ("dt", C.c_void_p), ("img_wh", C.c_void_p), ("box_out", C.c_void_p),
                ("score_out", C.c_void_p), ("label_out", C.c_void_p), ("track_out", C.c_void_p), ("count_out", C.c_void_p)]


class SyForecastExtrapQueriesDesc(C.Structure):
    _fields_ = [("state", SyForecastState), ("dt", C.c_void_p), ("n_query", C.c_void_p), ("Q", C.c_int32),
                ("img_wh", C.c_void_p), ("box_out", C.c_void_p), ("score_out", C.c_void_p), ("label_out", C.c_void_p),
                ("track_out", C.c_void_p), ("count_out", C.c_void_p)]


class SyForecastSequencesDesc(C.Structure):
    _fields_ = [("state", SyForecastState), ("det", C.c_void_p), ("det_start", C.c_void_p), ("det_n", C.c_void_p),
                ("frames", C.c_void_p), ("seq_frames", C.c_void_p), ("match_iou_th", C.c_double), ("box_out", C.c_void_p),
                ("score_out", C.c_void_p), ("label_out", C.c_void_p), ("track_out", C.c_void_p), ("rows_out", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


# every symbol include/streamyolo_sm100.h declares: (restype, argtypes)
_SIG = {
    "sy_last_error_string": (C.c_char_p, []),
    "sy_version": (C.c_int, []),
    "sy_check_device": (C.c_int, []),
    "sy_conv_stat_rows": (C.c_int, []),
    "sy_conv2d_tc": (C.c_int, [C.POINTER(SyConvDesc), C.c_void_p]),
    "sy_conv2d_plan": (C.c_int, [C.c_int32] * 10 + [C.POINTER(SyConvPlan)]),
    "sy_conv2d_simt": (C.c_int, [C.POINTER(SyConvDesc), C.c_void_p]),
    "sy_dwconv2d": (C.c_int, [C.POINTER(SyConvDesc), C.c_void_p]),
    "sy_focus_pack": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, SyTensor,
                                C.c_void_p]),
    "sy_focus_pack_f16": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, SyTensor,
                                    C.c_void_p]),
    "sy_stats_num_partials": (C.c_int, [C.c_int32, C.c_int32]),
    "sy_channel_stats": (C.c_int, [SyTensor, C.c_void_p, C.c_int32, C.c_void_p]),
    "sy_bn_finalize": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "sy_bn_act_apply": (C.c_int, [SyTensor, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, SyTensor, SyTensor,
                                  C.c_int64, C.c_int64, C.c_void_p]),
    "sy_upsample_nearest": (C.c_int, [SyTensor, SyTensor, C.c_void_p]),
    "sy_spp_maxpool": (C.c_int, [SyTensor, SyTensor, SyTensor, SyTensor, C.c_void_p]),
    "sy_spp_maxpool_f16": (C.c_int, [SyTensor, SyTensor, SyTensor, SyTensor, C.c_void_p]),
    "sy_copy": (C.c_int, [SyTensor, SyTensor, C.c_void_p]),
    "sy_select_images": (C.c_int, [C.POINTER(SySelectImagesDesc), C.c_void_p]),
    "sy_head_pred_decode": (C.c_int, [C.POINTER(SyHeadPredDesc), C.c_void_p]),
    "sy_tal_loss_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "sy_tal_loss": (C.c_int, [C.POINTER(SyTalLossDesc), C.c_void_p]),
    "sy_tal_loss_backward": (C.c_int, [C.POINTER(SyTalLossBwdDesc), C.c_void_p]),
    "sy_add": (C.c_int, [SyTensor, SyTensor, C.c_void_p]),
    "sy_spp_maxpool_backward_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "sy_spp_maxpool_backward": (C.c_int, [SyTensor, SyTensor, SyTensor, SyTensor, SyTensor, C.c_void_p, C.c_size_t,
                                          C.c_void_p]),
    "sy_dilate2": (C.c_int, [SyTensor, SyTensor, C.c_void_p]),
    "sy_upsample_nearest_backward": (C.c_int, [SyTensor, SyTensor, C.c_void_p]),
    "sy_head_pred_bwd_rows": (C.c_int, [C.c_int32, C.c_int32, C.c_int32]),
    "sy_head_pred_backward": (C.c_int, [C.POINTER(SyHeadPredBwdDesc), C.c_void_p]),
    "sy_head_pred_backward_wide": (C.c_int, [C.POINTER(SyHeadPredBwdDesc), C.c_void_p]),
    "sy_bn_act_bwd_rows": (C.c_int, [C.c_int32, C.c_int32]),
    "sy_bn_act_backward": (C.c_int, [C.POINTER(SyBnActBwdDesc), C.c_void_p]),
    "sy_postprocess_nms_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "sy_postprocess_nms": (C.c_int, [C.POINTER(SyNmsDesc), C.c_void_p]),
    "sy_stream_gate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sy_stream_rescale": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sy_coco_rows": (C.c_int, [C.POINTER(SyCocoRowsDesc), C.c_void_p]),
    "sy_forecast_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "sy_forecast_update": (C.c_int, [C.POINTER(SyForecastUpdateDesc), C.c_void_p]),
    "sy_forecast_extrap": (C.c_int, [C.POINTER(SyForecastExtrapDesc), C.c_void_p]),
    "sy_forecast_extrap_queries": (C.c_int, [C.POINTER(SyForecastExtrapQueriesDesc), C.c_void_p]),
    "sy_forecast_sequences": (C.c_int, [C.POINTER(SyForecastSequencesDesc), C.c_void_p]),
    "sy_conv2d_wgrad_workspace_bytes": (C.c_size_t, [C.POINTER(SyConvWgradDesc)]),
    "sy_conv2d_wgrad_tc": (C.c_int, [C.POINTER(SyConvWgradDesc), C.c_void_p]),
    "sy_pack_conv_weight": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_int64, C.c_int32, C.c_void_p]),
    "sy_pack_item_tiles": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "sy_pack_conv_weights_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p]),
    "sy_sgd_nesterov_ema_step": (C.c_int, [C.POINTER(SySgdEmaDesc), C.c_void_p]),
    "sy_nonfinite_flag": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sy_resize_bilinear": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_void_p]),
    "sy_scale_labels": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_void_p]),
    "sy_pair_labels": (C.c_int, [C.POINTER(SyPairLabelsDesc), C.c_void_p]),
    "sy_frame_labels": (C.c_int, [C.POINTER(SyFrameLabelsDesc), C.c_void_p]),
    "sy_letterbox": (C.c_int, [C.POINTER(SyLetterboxDesc), C.c_void_p]),
    "sy_letterbox_sized": (C.c_int, [C.POINTER(SyLetterboxSizedDesc), C.c_void_p]),
    "sy_resize_sized": (C.c_int, [C.POINTER(SyResizeSizedDesc), C.c_void_p]),
    "sy_jpeg_decode_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "sy_jpeg_decode": (C.c_int, [C.POINTER(SyJpegDecodeDesc), C.c_void_p]),
    "sy_jpeg_decode_sized_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "sy_jpeg_decode_sized": (C.c_int, [C.POINTER(SyJpegDecodeSizedDesc), C.c_void_p]),
    "sy_yuv_to_bgr_sized": (C.c_int, [C.POINTER(SyYuvToBgrSizedDesc), C.c_void_p]),
    "sy_bayer_to_bgr_sized": (C.c_int, [C.POINTER(SyBayerToBgrSizedDesc), C.c_void_p]),
    "sy_jpeg_encode_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int64]),
    "sy_jpeg_encode_max_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "sy_jpeg_encode": (C.c_int, [C.POINTER(SyJpegEncodeDesc), C.c_void_p]),
    "sy_draw_boxes": (C.c_int, [C.POINTER(SyDrawBoxesDesc), C.c_void_p]),
    "sy_vis_det_boxes": (C.c_int, [C.POINTER(SyVisDetBoxesDesc), C.c_void_p]),
    "sy_draw_outlines": (C.c_int, [C.POINTER(SyDrawOutlinesDesc), C.c_void_p]),
    "sy_splice_frames": (C.c_int, [C.POINTER(SySpliceFramesDesc), C.c_void_p]),
}
EXPORTED_SYMBOLS = tuple(_SIG)

_lib = None
_device_ok = False
LAUNCHES = 0      # kernels launched through this binding (bench.py reports it as gpu_launches)


def load_library():
    """dlopen the in-tree library (no GPU needed) and type every entry point."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -m streamyolo_b200.build` "
                               "(there is no fallback path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIG.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def lib():
    """Library handle for compute calls: also insists on a CUDA sm_90 device."""
    global _device_ok
    l = load_library()
    if not _device_ok:
        if not torch.cuda.is_available():
            raise RuntimeError("streamyolo_b200 needs a CUDA sm_90 (H100) device; there is no CPU path")
        rc = l.sy_check_device()
        if rc != 0:
            raise RuntimeError("streamyolo_b200: " + l.sy_last_error_string().decode())
        _device_ok = True
    return l


def _check(rc, kernels=1):
    global LAUNCHES
    LAUNCHES += kernels
    if rc != 0:
        raise RuntimeError(f"libstreamyolo_sm100 error {rc}: " + load_library().sy_last_error_string().decode())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


NULL_T = SyTensor(None, 0, 0, 0, 0, 0)


class View:
    """Channel-slice / image-slice view of an NHWC 16-bit buffer ``buf[N,H,W,Ctot]``: bf16, or fp16 for the eval /
    streaming forwards with fp16 activation storage."""
    __slots__ = ("buf", "n0", "n", "c0", "c", "off")

    def __init__(self, buf, c0=0, c=None, n0=0, n=None):
        assert buf.dtype in STORAGE and buf.dim() == 4 and buf.is_contiguous()
        self.buf, self.c0, self.n0, self.off = buf, c0, n0, 0
        self.c = buf.shape[3] - c0 if c is None else c
        self.n = buf.shape[0] - n0 if n is None else n

    @staticmethod
    def empty(n, h, w, c, device, dtype=torch.bfloat16):
        return View(torch.empty((n, h, w, c), dtype=dtype, device=device))

    @property
    def dtype(self):
        return self.buf.dtype

    @property
    def h(self):
        return self.buf.shape[1]

    @property
    def w(self):
        return self.buf.shape[2]

    def ch(self, c0, c):
        return View(self.buf, self.c0 + c0, c, self.n0, self.n)

    def imgs(self, n0, n):
        return View(self.buf, self.c0, self.c, self.n0 + n0, n)

    def img_elems(self):
        b = self.buf
        return b.shape[1] * b.shape[2] * b.shape[3]

    def shifted(self, elems):
        """Same shape, base address moved by ``elems`` elements (used for group-offset destinations)."""
        v = View(self.buf, self.c0, self.c, self.n0, self.n)
        v.off = getattr(self, "off", 0) + elems
        return v

    def st(self):
        b = self.buf
        ptr = b.data_ptr() + 2 * (self.n0 * b.shape[1] * b.shape[2] * b.shape[3] + self.c0 + self.off)
        return SyTensor(ptr, self.n, b.shape[1], b.shape[2], self.c, b.shape[3])

    def torch(self):
        """NHWC torch view (for tests)."""
        return self.buf[self.n0:self.n0 + self.n, :, :, self.c0:self.c0 + self.c]

    def nchw_float(self):
        return self.torch().permute(0, 3, 1, 2).float()


def from_nchw(x):
    """float NCHW torch tensor -> bf16 NHWC View (test helper)."""
    return View(x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16))


def _w32(w):
    w = w.detach()
    if w.dtype != torch.float32 or not w.is_contiguous():
        w = w.float().contiguous()
    return w


def _pack_flag(dtype):
    if dtype not in STORAGE:
        raise ValueError(f"conv operands are bf16 or fp16, not {dtype}")
    return SY_PACK_F16 if dtype == torch.float16 else 0


def pack_conv_weight(*ws, dtype=torch.bfloat16):
    """OIHW fp32 parameter(s) -> bf16 (or fp16) [sum O][kh*kw][I] contiguous (GEMM B operand, K-major), packed on the device
    (sy_pack_conv_weight).  Several weights with the same [I, kh, kw] (CSPLayer conv1 | conv2) land in one operand."""
    _, i, kh, kw = ws[0].shape
    flag = _pack_flag(dtype)
    out = torch.empty((sum(w.shape[0] for w in ws), kh * kw, i), dtype=dtype, device=ws[0].device)
    o0 = 0
    for w in ws:
        w = _w32(w)
        assert tuple(w.shape[1:]) == (i, kh, kw)
        _check(lib().sy_pack_conv_weight(w.data_ptr(), w.shape[0], i, kh, kw, flag, out.data_ptr() + 2 * o0 * kh * kw * i, 0,
                                         0, _stream()))
        o0 += w.shape[0]
    return out


def conv_out_hw(h, w, k, s):
    p = (k - 1) // 2
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def conv_stat_rows():
    return load_library().sy_conv_stat_rows()


def conv2d(x: View, wpk, y: View, k, s, mode, impl="tc", scale=None, shift=None, act=1, res: View = None,
           partials=None, split_n=0, timeline=None, debug_flags=0, bn=None, momentum=0.03, eps=1e-3, scale_shift=None,
           sync=None, mean_invstd=None, debug_f32=None, tile_mode=0, tile_bn=0, stat_updates=1):
    """``k`` is an int (square) or (kh, kw).  With ``partials`` (RAW mode, tensor-core path) returns the number
    of per-CTA statistic rows the launch writes.  ``tile_mode`` / ``tile_bn`` override the tensor-core tiling
    (0 = planner; see conv2d_plan).  ``stat_updates=2``: the single statistics group updates the running statistics
    twice (one pass standing for two identical ones; SyConvDesc.stat_updates).  The activation storage (bf16 | fp16) is
    that of the views: x, y, res and the packed weights must all have it."""
    dtypes = {x.dtype, y.dtype, wpk.dtype} | ({res.dtype} if res is not None else set())
    if len(dtypes) != 1:
        raise ValueError(f"conv2d: x, y, res and the packed weights must share one storage dtype, got {sorted(map(str, dtypes))}")
    d = SyConvDesc()
    d.x, d.y = x.st(), y.st()
    d.w = wpk.data_ptr()
    d.kh, d.kw = (k, k) if isinstance(k, int) else k
    d.stride, d.mode, d.act = s, mode, act
    d.scale = scale.data_ptr() if scale is not None else None
    d.shift = shift.data_ptr() if shift is not None else None
    d.res = res.st() if res is not None else NULL_T
    d.split_n = split_n
    rows = C.c_int32(0)
    if partials is not None:
        d.stat_partials, d.n_partials = partials.data_ptr(), partials.shape[0]
        d.rows_written = C.pointer(rows)
    if bn:
        for i, (g, b_, rm, rv, nbt, c0) in enumerate(bn):
            seg = d.bn[i]
            seg.gamma, seg.beta = g.data_ptr(), b_.data_ptr()
            seg.running_mean = rm.data_ptr() if rm is not None else None
            seg.running_var = rv.data_ptr() if rv is not None else None
            seg.num_batches_tracked = nbt.data_ptr() if nbt is not None else None
            seg.c_begin = c0
        d.momentum, d.eps = momentum, eps
        d.scale_shift, d.sync = scale_shift.data_ptr(), sync.data_ptr()
        d.mean_invstd = mean_invstd.data_ptr() if mean_invstd is not None else None
    d.debug_flags = debug_flags
    d.tile_mode, d.tile_bn = tile_mode, tile_bn
    d.stat_updates = stat_updates
    d.storage = STORAGE[x.dtype]
    d.debug_f32 = debug_f32.data_ptr() if debug_f32 is not None else None
    if timeline is not None:
        d.debug_timeline, d.debug_timeline_events = timeline.data_ptr(), timeline.numel() // 2
    fn = {"tc": lib().sy_conv2d_tc, "simt": lib().sy_conv2d_simt, "dw": lib().sy_dwconv2d}[impl]
    _check(fn(C.byref(d), _stream()))
    return rows.value


def focus_pack(x, frames, y: View):
    """Focus space-to-depth of the float frames into ``y`` (bf16, or fp16 for an fp16-storage forward)."""
    assert x.dtype == torch.float32 and x.is_contiguous()
    b, ch, h, w = x.shape
    fn = lib().sy_focus_pack_f16 if y.dtype == torch.float16 else lib().sy_focus_pack
    _check(fn(x.data_ptr(), b, ch, h, w, frames, y.st(), _stream()))


STEM_K = (3, 1)      # the stem runs as a 3x1 conv over the W-gathered 64-channel focus tensor


def pack_dw_weight(w, dtype=torch.bfloat16):
    """depthwise [C, 1, k, k] fp32 parameter -> bf16 (or fp16) [k*k][C] (sy_pack_conv_weight mode 0 on the [1, C, k, k]
    view)."""
    c, one, kh, kw = w.shape
    assert one == 1
    return pack_conv_weight(_w32(w).view(1, c, kh, kw), dtype=dtype).view(kh * kw, c)


def pack_stem_weight(w, dtype=torch.bfloat16):
    """[O,12,3,3] float -> bf16 (or fp16) [O][3 (row)][64 = 3 taps x (12 focus + 4 zero) + 16 zero] (sy_pack_conv_weight,
    mode 2)."""
    w = _w32(w)
    o, i, kh, kw = w.shape
    flag = _pack_flag(dtype)
    out = torch.empty((o, kh, 64), dtype=dtype, device=w.device)
    _check(lib().sy_pack_conv_weight(w.data_ptr(), o, i, kh, kw, 2 | flag, out.data_ptr(), 0, 0, _stream()))
    return out


def stats_num_partials(n, hw):
    return load_library().sy_stats_num_partials(n, hw)


def channel_stats(x: View, partials):
    _check(lib().sy_channel_stats(x.st(), partials.data_ptr(), partials.shape[0], _stream()))


def bn_finalize(partials, p_split, groups, count, gamma, beta, rmean, rvar, nbt, momentum, eps, scale, shift):
    c = gamma.numel()
    _check(lib().sy_bn_finalize(partials.data_ptr(), partials.shape[0], p_split, groups, count, c,
                                gamma.data_ptr(), beta.data_ptr(),
                                rmean.data_ptr() if rmean is not None else None,
                                rvar.data_ptr() if rvar is not None else None,
                                nbt.data_ptr() if nbt is not None else None,
                                momentum, eps, scale.data_ptr(), shift.data_ptr(), _stream()))


def bn_act_apply(x: View, scale_ptr, shift_ptr, split_n, act, res, y: View, y_goff1=0, res_goff1=0):
    """``scale_ptr`` / ``shift_ptr``: fp32 [groups][C] tensors (or their raw device addresses)"""
    if torch.is_tensor(scale_ptr):
        scale_ptr, shift_ptr = scale_ptr.data_ptr(), shift_ptr.data_ptr()
    _check(lib().sy_bn_act_apply(x.st(), scale_ptr, shift_ptr, split_n, act,
                                 res.st() if res is not None else NULL_T, y.st(), y_goff1, res_goff1, _stream()))


def _same_dtype(what, *views):
    if len({v.dtype for v in views}) != 1:
        raise ValueError(f"{what}: the views must share one storage dtype")


def upsample_nearest(x: View, y: View):
    """(moves 16-bit values: bf16 and fp16 views alike)"""
    _same_dtype("upsample_nearest", x, y)
    _check(lib().sy_upsample_nearest(x.st(), y.st(), _stream()))


def spp_maxpool(x: View, y5: View, y9: View, y13: View):
    _same_dtype("spp_maxpool", x, y5, y9, y13)
    fn = lib().sy_spp_maxpool_f16 if x.dtype == torch.float16 else lib().sy_spp_maxpool
    _check(fn(x.st(), y5.st(), y9.st(), y13.st(), _stream()))


def copy(x: View, y: View):
    """(moves 16-bit values: bf16 and fp16 views alike)"""
    _same_dtype("copy", x, y)
    _check(lib().sy_copy(x.st(), y.st(), _stream()))


def select_images(srcs, dsts, flags):
    """Image i of ``dsts[k]`` = image i of ``srcs[k]`` for every i whose int32 device flag ``flags[i]`` is set, for up to
    three view pairs in ONE launch (sy_select_images); images whose flag is clear are not touched.  The flags are read on
    the device: a captured launch follows what is written there before each replay.  (Moves 16-bit values: bf16 and fp16
    views alike.)"""
    _require(1 <= len(srcs) == len(dsts) <= 3, "select_images: 1 to 3 (src, dst) view pairs")
    _same_dtype("select_images", *srcs, *dsts)
    _require(torch.is_tensor(flags) and flags.dtype == torch.int32 and flags.is_contiguous()
             and flags.numel() == srcs[0].n, "select_images: flags must be int32 [n]")
    d = SySelectImagesDesc()
    for k, (s, t) in enumerate(zip(srcs, dsts)):
        d.src[k], d.dst[k] = s.st(), t.st()
    d.n_pairs, d.flags = len(srcs), flags.data_ptr()
    _check(lib().sy_select_images(C.byref(d), _stream()))


def stream_gate(status, flags, start, keep):
    """start[i] = flags[i] != 0 and status[i] == 0, keep[i] = status[i] == 0 (sy_stream_gate): int32 [n] device arrays;
    ``status`` None counts every stream as decoded."""
    n = flags.numel()
    for name, t in (("flags", flags), ("start", start), ("keep", keep)) + ((("status", status),) if status is not None else ()):
        _require(_tensor_ok(t, torch.int32, 1) and t.numel() == n and t.is_cuda, f"stream_gate: {name} must be CUDA int32 [n]")
    _check(lib().sy_stream_gate(status.data_ptr() if status is not None else None, flags.data_ptr(), n, start.data_ptr(),
                                keep.data_ptr(), _stream()))


def stream_rescale(det, count, status, ratio):
    """In place: the boxes of rows < count[i] of ``det`` [n, max_det, 7] divided by fp32 ``ratio[i]``, and count[i] = 0 where
    ``status[i]`` != 0 (sy_stream_rescale; ``status`` may be None)."""
    _require(_tensor_ok(det, torch.float32, 3) and det.shape[2] == 7, "stream_rescale: det must be float32 [n, max_det, 7]")
    n = det.shape[0]
    _require(_tensor_ok(count, torch.int32, 1) and count.numel() == n, "stream_rescale: count must be int32 [n]")
    _require(_tensor_ok(ratio, torch.float32, 1) and ratio.numel() == n, "stream_rescale: ratio must be float32 [n]")
    _require(status is None or (_tensor_ok(status, torch.int32, 1) and status.numel() == n),
             "stream_rescale: status must be int32 [n]")
    _check(lib().sy_stream_rescale(det.data_ptr(), n, det.shape[1], count.data_ptr(),
                                   status.data_ptr() if status is not None else None, ratio.data_ptr(), _stream()))


def coco_rows(det, count, ratio, image_id, class_ids, status=None, out=None):
    """COCO detection rows of a batch of NMS outputs (sy_coco_rows): ``det`` fp32 [B, max_det, 7] and ``count`` int32 [B]
    of postprocess_nms, ``ratio`` fp32 [B], ``image_id`` int32 [B] (< 0: the image emits nothing), ``class_ids`` int32
    [num_classes]; ``status`` int32 [B * F] decode status of each image's F frames (an image with a frame not decoded emits
    nothing), or None.  -> ``(bbox fp32 [B * max_det, 4] xywh, score fp32 [B * max_det], image_id int32 [B * max_det],
    category int32 [B * max_det], total int32 [1])``: the first ``total`` rows are valid.  ``out``: those five tensors of an
    earlier call to write into (static buffers for CUDA-graph capture).  Nothing is read back."""
    _require(_tensor_ok(det, torch.float32, 3) and det.shape[2] == 7 and det.is_cuda,
             "coco_rows: det must be contiguous CUDA float32 [B, max_det, 7]")
    b, max_det, _ = det.shape
    for name, t, dt in (("count", count, torch.int32), ("ratio", ratio, torch.float32), ("image_id", image_id, torch.int32)):
        _require(_tensor_ok(t, dt, 1) and t.numel() == b and t.device == det.device, f"coco_rows: {name} must be {dt} [{b}]")
    _require(_tensor_ok(class_ids, torch.int32, 1) and class_ids.numel() > 0 and class_ids.device == det.device,
             "coco_rows: class_ids must be int32 [num_classes]")
    _require(status is None or (_tensor_ok(status, torch.int32, 1) and status.numel() % b == 0 and status.numel() > 0
                                and status.device == det.device), f"coco_rows: status must be int32 [{b} * frames]")
    cap = b * max_det
    if out is None:
        out = (torch.empty((cap, 4), dtype=torch.float32, device=det.device),
               torch.empty((cap,), dtype=torch.float32, device=det.device),
               torch.empty((cap,), dtype=torch.int32, device=det.device),
               torch.empty((cap,), dtype=torch.int32, device=det.device),
               torch.empty((1,), dtype=torch.int32, device=det.device))
    bbox, score, ids, cat, total = out
    _require(_tensor_ok(bbox, torch.float32, 2) and tuple(bbox.shape) == (cap, 4) and _tensor_ok(score, torch.float32, 1)
             and _tensor_ok(ids, torch.int32, 1) and _tensor_ok(cat, torch.int32, 1) and _tensor_ok(total, torch.int32, 1)
             and score.numel() == ids.numel() == cat.numel() == cap and total.numel() == 1,
             f"coco_rows: out must be fp32 [{cap}, 4], fp32 [{cap}], int32 [{cap}], int32 [{cap}], int32 [1]")
    d = SyCocoRowsDesc(det.data_ptr(), b, max_det, count.data_ptr(), ratio.data_ptr(), image_id.data_ptr(),
                       status.data_ptr() if status is not None else None,
                       status.numel() // b if status is not None else 1, class_ids.numel(), class_ids.data_ptr(),
                       bbox.data_ptr(), score.data_ptr(), ids.data_ptr(), cat.data_ptr(), total.data_ptr())
    _check(lib().sy_coco_rows(C.byref(d), _stream()))
    return out


class ForecastState:
    """Device state of the sy_forecast_* entry points for ``streams`` streams (or sequences) of at most ``max_tracks``
    tracks, with the update's workspace: x fp32 [S, T, 8], P fp32 [S, T, 8, 8], label / track int32 [S, T], score fp32
    [S, T], meta int32 [S, 4] (n_tracks, n_matched, next track id, overflow).  Zeroed: no tracks."""

    def __init__(self, streams, max_tracks, device):
        _require(int(streams) == streams and 1 <= streams <= 65535, f"ForecastState: {streams} streams (1 to 65535)")
        _require(int(max_tracks) == max_tracks and 1 <= max_tracks <= 1 << 20,
                 f"ForecastState: max_tracks {max_tracks} (1 to 2^20)")
        s, t = int(streams), int(max_tracks)
        self.streams, self.max_tracks = s, t
        self.x = torch.zeros((s, t, 8), dtype=torch.float32, device=device)
        self.P = torch.zeros((s, t, 8, 8), dtype=torch.float32, device=device)
        self.label = torch.zeros((s, t), dtype=torch.int32, device=device)
        self.score = torch.zeros((s, t), dtype=torch.float32, device=device)
        self.track = torch.zeros((s, t), dtype=torch.int32, device=device)
        self.meta = torch.zeros((s, 4), dtype=torch.int32, device=device)
        self.workspace = torch.empty(load_library().sy_forecast_workspace_bytes(s, t), dtype=torch.uint8, device=device)

    def desc(self):
        return SyForecastState(self.x.data_ptr(), self.P.data_ptr(), self.label.data_ptr(), self.score.data_ptr(),
                               self.track.data_ptr(), self.meta.data_ptr(), self.streams, self.max_tracks)


def _on(t, dtype, shape, device):
    return _tensor_ok(t, dtype, len(shape)) and tuple(t.shape) == tuple(shape) and t.device == device


def forecast_update(state, det, count, dt, start=None, keep=None, match_iou_th=0.3, clear_on_empty=False):
    """One new detection per stream into ``state`` (sy_forecast_update): ``det`` fp32 [S, max_det, 7] and ``count`` int32
    [S] as postprocess_nms / stream_rescale leave them, ``dt`` int32 [S] frames since each stream's previous detection,
    ``start`` / ``keep`` int32 [S] or None.  Nothing is read back: a stream whose count exceeds max_tracks keeps its state
    and gets state.meta[s, 3] = 1.  An empty detection keeps the predicted tracks (pps_forecast_kf.py), or with
    ``clear_on_empty`` leaves the stream without tracks (the streamer, sAP/forecast/streamer.py)."""
    dev = state.x.device
    _require(_tensor_ok(det, torch.float32, 3) and det.shape[0] == state.streams and det.shape[2] == 7 and det.device == dev,
             f"forecast_update: det must be float32 [{state.streams}, max_det, 7] on {dev}")
    for name, t in (("count", count), ("dt", dt), ("start", start), ("keep", keep)):
        _require(t is None and name in ("start", "keep") or (t is not None and _on(t, torch.int32, (state.streams,), dev)),
                 f"forecast_update: {name} must be int32 [{state.streams}] on {dev}")
    d = SyForecastUpdateDesc(state.desc(), det.data_ptr(), det.shape[1], count.data_ptr(), dt.data_ptr(),
                             start.data_ptr() if start is not None else None, keep.data_ptr() if keep is not None else None,
                             float(match_iou_th), state.workspace.data_ptr(), state.workspace.numel(),
                             1 if clear_on_empty else 0)
    _check(lib().sy_forecast_update(C.byref(d), _stream()))


def forecast_extrap(state, dt, img_wh, out=None):
    """Each stream's tracks extrapolated ``dt`` (int32 [S]) frames ahead and cleaned up for its image size ``img_wh`` (int32
    [S, 2], (W, H)) (sy_forecast_extrap) -> ``(box fp32 [S, T, 4] ltwh, score fp32 [S, T], label int32 [S, T], track int32
    [S, T], count int32 [S])``: the first count[s] rows of stream s are valid.  ``out``: those five tensors of an earlier
    call to write into."""
    s, t, dev = state.streams, state.max_tracks, state.x.device
    _require(_on(dt, torch.int32, (s,), dev), f"forecast_extrap: dt must be int32 [{s}] on {dev}")
    _require(_on(img_wh, torch.int32, (s, 2), dev), f"forecast_extrap: img_wh must be int32 [{s}, 2] on {dev}")
    if out is None:
        out = (torch.empty((s, t, 4), dtype=torch.float32, device=dev), torch.empty((s, t), dtype=torch.float32, device=dev),
               torch.empty((s, t), dtype=torch.int32, device=dev), torch.empty((s, t), dtype=torch.int32, device=dev),
               torch.empty((s,), dtype=torch.int32, device=dev))
    box, score, label, track, count = out
    _require(_on(box, torch.float32, (s, t, 4), dev) and _on(score, torch.float32, (s, t), dev)
             and _on(label, torch.int32, (s, t), dev) and _on(track, torch.int32, (s, t), dev)
             and _on(count, torch.int32, (s,), dev), "forecast_extrap: out must be the five tensors of an earlier call")
    d = SyForecastExtrapDesc(state.desc(), dt.data_ptr(), img_wh.data_ptr(), box.data_ptr(), score.data_ptr(),
                             label.data_ptr(), track.data_ptr(), count.data_ptr())
    _check(lib().sy_forecast_extrap(C.byref(d), _stream()))
    return out


def forecast_extrap_queries(state, dt, n_query, img_wh, out=None):
    """Up to Q queries per stream in one launch (sy_forecast_extrap_queries): stream s's tracks extrapolated ``dt[s, k]``
    (fp32 [S, Q]) frames ahead for k < ``n_query[s]`` (int32 [S]), each cleaned up for ``img_wh`` (int32 [S, 2], (W, H)) ->
    ``(box fp32 [S, Q, T, 4] ltwh, score fp32 [S, Q, T], label int32 [S, Q, T], track int32 [S, Q, T], count int32 [S, Q])``:
    the first count[s, k] rows of query (s, k) are valid, count is 0 past n_query[s].  An integer dt gives forecast_extrap's
    rows bit for bit.  ``out``: those five tensors of an earlier call to write into.  Capturable."""
    s, t, dev = state.streams, state.max_tracks, state.x.device
    q = dt.shape[1] if _tensor_ok(dt, torch.float32, 2) else 0
    _require(q >= 1 and _on(dt, torch.float32, (s, q), dev), f"forecast_extrap_queries: dt must be float32 [{s}, Q] on {dev}")
    _require(q <= 65535, f"forecast_extrap_queries: {q} queries per stream (at most 65535)")
    _require(_on(n_query, torch.int32, (s,), dev), f"forecast_extrap_queries: n_query must be int32 [{s}] on {dev}")
    _require(_on(img_wh, torch.int32, (s, 2), dev), f"forecast_extrap_queries: img_wh must be int32 [{s}, 2] on {dev}")
    if out is None:
        out = (torch.empty((s, q, t, 4), dtype=torch.float32, device=dev),
               torch.empty((s, q, t), dtype=torch.float32, device=dev), torch.empty((s, q, t), dtype=torch.int32, device=dev),
               torch.empty((s, q, t), dtype=torch.int32, device=dev), torch.empty((s, q), dtype=torch.int32, device=dev))
    box, score, label, track, count = out
    _require(_on(box, torch.float32, (s, q, t, 4), dev) and _on(score, torch.float32, (s, q, t), dev)
             and _on(label, torch.int32, (s, q, t), dev) and _on(track, torch.int32, (s, q, t), dev)
             and _on(count, torch.int32, (s, q), dev), "forecast_extrap_queries: out must be the five tensors of an earlier call")
    d = SyForecastExtrapQueriesDesc(state.desc(), dt.data_ptr(), n_query.data_ptr(), q, img_wh.data_ptr(), box.data_ptr(),
                                    score.data_ptr(), label.data_ptr(), track.data_ptr(), count.data_ptr())
    _check(lib().sy_forecast_extrap_queries(C.byref(d), _stream()))
    return out


def forecast_sequences(state, det, det_start, det_n, frames, seq_frames, n_rows, match_iou_th=0.3):
    """The offline forecast of ``state.streams`` sequences (sy_forecast_sequences): ``det`` fp32 [R, 7] rows of every
    detection, detection k at rows det_start[k] .. + det_n[k] (int32 [D]); ``frames`` int32 [F, 6] (latest detection or
    -1, dt of its update, dt of the query, first output row, W, H); ``seq_frames`` int32 [S + 1]; ``n_rows`` the output
    room (the sum of the frames' track counts) -> ``(box fp32 [n_rows, 4] ltwh, score fp32, label int32, track int32
    [n_rows], rows int32 [F])``: frame f's rows start at frames[f, 3], rows[f] of them.  The state is cleared per sequence."""
    dev = state.x.device
    _require(_tensor_ok(det, torch.float32, 2) and det.shape[1] == 7 and det.shape[0] > 0 and det.device == dev,
             "forecast_sequences: det must be float32 [R, 7]")
    nd = det_start.shape[0] if torch.is_tensor(det_start) else -1
    _require(nd > 0 and _on(det_start, torch.int32, (nd,), dev) and _on(det_n, torch.int32, (nd,), dev),
             "forecast_sequences: det_start and det_n must be int32 [D]")
    _require(_tensor_ok(frames, torch.int32, 2) and frames.shape[1] == 6 and frames.device == dev,
             "forecast_sequences: frames must be int32 [F, 6]")
    _require(_on(seq_frames, torch.int32, (state.streams + 1,), dev),
             f"forecast_sequences: seq_frames must be int32 [{state.streams + 1}]")
    n_rows = max(int(n_rows), 1)
    box = torch.empty((n_rows, 4), dtype=torch.float32, device=dev)
    score = torch.empty((n_rows,), dtype=torch.float32, device=dev)
    label = torch.empty((n_rows,), dtype=torch.int32, device=dev)
    track = torch.empty((n_rows,), dtype=torch.int32, device=dev)
    rows = torch.empty((frames.shape[0],), dtype=torch.int32, device=dev)
    d = SyForecastSequencesDesc(state.desc(), det.data_ptr(), det_start.data_ptr(), det_n.data_ptr(), frames.data_ptr(),
                                seq_frames.data_ptr(), float(match_iou_th), box.data_ptr(), score.data_ptr(),
                                label.data_ptr(), track.data_ptr(), rows.data_ptr(), state.workspace.data_ptr(),
                                state.workspace.numel())
    _check(lib().sy_forecast_sequences(C.byref(d), _stream()))
    return box, score, label, track, rows


def head_pred_decode(cls_feat: View, reg_feat: View, w_reg, b_reg, w_obj, b_obj, w_cls, b_cls, stride,
                     anchor_offset, a_total, out, origin, sigmoid, decode):
    _same_dtype("head_pred_decode", cls_feat, reg_feat)
    d = SyHeadPredDesc()
    d.cls_feat, d.reg_feat = cls_feat.st(), reg_feat.st()
    d.storage = STORAGE[cls_feat.dtype]
    d.w_reg, d.b_reg, d.w_obj, d.b_obj = w_reg.data_ptr(), b_reg.data_ptr(), w_obj.data_ptr(), b_obj.data_ptr()
    d.w_cls, d.b_cls = w_cls.data_ptr(), b_cls.data_ptr()
    d.num_classes = w_cls.shape[0]
    d.stride, d.anchor_offset, d.a_total = stride, anchor_offset, a_total
    d.sigmoid, d.decode = int(sigmoid), int(decode)
    d.out = out.data_ptr()
    d.origin = origin.data_ptr() if origin is not None else None
    _check(lib().sy_head_pred_decode(C.byref(d), _stream()))


def tal_loss_workspace_bytes(b, a_total, max_labels, num_classes):
    return load_library().sy_tal_loss_workspace_bytes(b, a_total, max_labels, num_classes)


def tal_loss(outputs, origin, labels_fut, labels_cur, hw, strides, gamma, ignore_thr, ignore_value, use_l1,
             workspace, loss_out, fg_out=None, matched_out=None, pred_iou_out=None):
    d = SyTalLossDesc()
    b, a, no = outputs.shape
    d.b, d.a_total, d.max_labels, d.num_classes = b, a, labels_fut.shape[1], no - 5
    d.n_levels = len(hw)
    for i, ((h, w), s) in enumerate(zip(hw, strides)):
        d.level_h[i], d.level_w[i], d.level_stride[i] = h, w, s
    d.outputs = outputs.data_ptr()
    d.origin = origin.data_ptr() if origin is not None else None
    d.labels_fut, d.labels_cur = labels_fut.data_ptr(), labels_cur.data_ptr()
    d.gamma, d.ignore_thr, d.ignore_value, d.use_l1 = gamma, ignore_thr, ignore_value, int(use_l1)
    d.workspace, d.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    d.loss_out = loss_out.data_ptr()
    d.fg_out = fg_out.data_ptr() if fg_out is not None else None
    d.matched_out = matched_out.data_ptr() if matched_out is not None else None
    d.pred_iou_out = pred_iou_out.data_ptr() if pred_iou_out is not None else None
    _check(lib().sy_tal_loss(C.byref(d), _stream()), kernels=6)


def tal_loss_backward(outputs, origin, labels_fut, hw, strides, gamma, use_l1, workspace, grad_scale=1.0,
                      grad_outputs=None, grad_origin=None, grad_raw=None):
    """Gradient of total_loss w.r.t. the head outputs; run after tal_loss() on the same workspace."""
    d = SyTalLossBwdDesc()
    b, a, no = outputs.shape
    d.outputs = outputs.data_ptr()
    d.origin = origin.data_ptr() if origin is not None else None
    d.labels_fut = labels_fut.data_ptr()
    d.b, d.a_total, d.max_labels, d.num_classes = b, a, labels_fut.shape[1], no - 5
    d.n_levels = len(hw)
    for i, ((h, w), s) in enumerate(zip(hw, strides)):
        d.level_h[i], d.level_w[i], d.level_stride[i] = h, w, s
    d.gamma, d.use_l1 = gamma, int(use_l1)
    d.workspace, d.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    d.grad_scale = grad_scale
    d.grad_outputs = grad_outputs.data_ptr() if grad_outputs is not None else None
    d.grad_origin = grad_origin.data_ptr() if grad_origin is not None else None
    d.grad_raw = grad_raw.data_ptr() if grad_raw is not None else None
    _check(lib().sy_tal_loss_backward(C.byref(d), _stream()), kernels=1)


def pack_conv_weight_dgrad(*ws):
    """Weights for the data gradient of a stride-1 conv: dx = conv(dy, w') with w'[ci][kh-1-r][kw-1-s][co] = w[co][ci][r][s]
    (same padding), i.e. the forward tensor-core kernel on the flipped, channel-transposed filter; packed on the device
    (sy_pack_conv_weight, mode 1).  Several weights (CSPLayer conv1 | conv2) are concatenated along co."""
    _, i, kh, kw = ws[0].shape
    ot = sum(w.shape[0] for w in ws)
    out = torch.empty((i, kh * kw, ot), dtype=torch.bfloat16, device=ws[0].device)
    o0 = 0
    for w in ws:
        w = _w32(w)
        _check(lib().sy_pack_conv_weight(w.data_ptr(), w.shape[0], i, kh, kw, 1, out.data_ptr(), ot, o0, _stream()))
        o0 += w.shape[0]
    return out


def conv2d_wgrad(x: View, dy: View, k, s, dw, accumulate=False, workspace=None):
    """dw[cout, cin, kh, kw] (fp32) (+)= weight gradient of the conv that maps x to (the shape of) dy."""
    kh, kw = (k, k) if isinstance(k, int) else k
    assert dw.dtype == torch.float32 and dw.is_contiguous() and tuple(dw.shape) == (dy.c, x.c, kh, kw)
    d = SyConvWgradDesc()
    d.x, d.dy = x.st(), dy.st()
    d.kh, d.kw, d.stride = kh, kw, s
    d.dw, d.accumulate = dw.data_ptr(), int(accumulate)
    need = lib().sy_conv2d_wgrad_workspace_bytes(C.byref(d))
    if need == 0:
        raise RuntimeError("conv2d_wgrad: " + (lib().sy_last_error_string() or b"").decode())
    if workspace is None or workspace.numel() * workspace.element_size() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=dw.device)
    d.workspace, d.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    _check(lib().sy_conv2d_wgrad_tc(C.byref(d), _stream()), kernels=2)
    return workspace


def postprocess_nms(pred, num_classes, conf_thre, nms_thre, class_agnostic=False, max_det=None):
    """-> (det [B, max_det, 7] fp32, count [B] int32) on the device; rows [x1, y1, x2, y2, obj, class_conf, class_pred]."""
    assert pred.dtype == torch.float32 and pred.is_contiguous() and pred.shape[2] == 5 + num_classes
    b, a, _ = pred.shape
    max_det = a if max_det is None else max_det
    det = torch.empty((b, max_det, 7), dtype=torch.float32, device=pred.device)
    count = torch.empty((b,), dtype=torch.int32, device=pred.device)
    ws = torch.empty(load_library().sy_postprocess_nms_workspace_bytes(b, a), dtype=torch.uint8, device=pred.device)
    d = SyNmsDesc()
    d.pred, d.b, d.a_total, d.num_classes, d.max_det = pred.data_ptr(), b, a, num_classes, max_det
    d.conf_thre, d.nms_thre, d.class_agnostic = conf_thre, nms_thre, int(class_agnostic)
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    d.det_out, d.count_out = det.data_ptr(), count.data_ptr()
    _check(lib().sy_postprocess_nms(C.byref(d), _stream()), kernels=1)
    return det, count


def bn_act_backward(raw: View, dy: View, draw: View, scale, shift, mean, invstd, split_n, act, dgamma, dbeta,
                    accumulate=False):
    """BatchNorm(train) + SiLU backward of one BaseConv; scale/shift/mean/invstd: fp32 [2, C] (group-major)."""
    rows = load_library().sy_bn_act_bwd_rows(raw.n, raw.h * raw.w)
    partials = torch.empty((rows, 2 * raw.c), dtype=torch.float32, device=dgamma.device)
    coef = torch.empty((8 * raw.c,), dtype=torch.float32, device=dgamma.device)
    d = SyBnActBwdDesc()
    d.raw, d.dy, d.draw = raw.st(), dy.st(), draw.st()
    d.scale, d.shift, d.mean, d.invstd = scale.data_ptr(), shift.data_ptr(), mean.data_ptr(), invstd.data_ptr()
    d.split_n, d.act = split_n, int(act)
    d.dgamma, d.dbeta, d.accumulate = dgamma.data_ptr(), dbeta.data_ptr(), int(accumulate)
    d.partials, d.n_partials, d.coef = partials.data_ptr(), rows, coef.data_ptr()
    _check(lib().sy_bn_act_backward(C.byref(d), _stream()), kernels=3)


def dilate2(g: View, D: View):
    _check(lib().sy_dilate2(g.st(), D.st(), _stream()))


def conv2d_dgrad_stride2(dy: View, w, dx: View, k=3):
    """Data gradient of a stride-2 conv: zero-insert dy to dx's spatial size, then the stride-1 forward kernel on the
    flipped, channel-transposed filter (``w`` = the forward OIHW weights)."""
    D = View.empty(dx.n, dx.h, dx.w, dy.c, dy.buf.device)
    dilate2(dy, D)
    conv2d(D, pack_conv_weight_dgrad(w), dx, k, 1, SY_CONV_RAW)


def upsample_nearest_backward(dy: View, dx: View):
    _check(lib().sy_upsample_nearest_backward(dy.st(), dx.st(), _stream()))


def head_pred_backward(grad_raw, cls_feat: View, reg_feat: View, d_cls_feat: View, d_reg_feat: View, w_reg, w_obj, w_cls,
                       a_total, anchor_offset, dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate=False):
    """Backward of one head level's three prediction convs, 1 <= classes <= 27 (sy_head_pred_backward)."""
    _head_pred_bwd("sy_head_pred_backward", grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls,
                   a_total, anchor_offset, dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate)


def head_pred_backward_wide(grad_raw, cls_feat: View, reg_feat: View, d_cls_feat: View, d_reg_feat: View, w_reg, w_obj,
                            w_cls, a_total, anchor_offset, dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate=False):
    """The same for any class count the forward takes (sy_head_pred_backward_wide: 1 ... 251 classes, (5 + classes) x
    channels x 4 bytes <= 200 KiB)."""
    _head_pred_bwd("sy_head_pred_backward_wide", grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls,
                   a_total, anchor_offset, dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate)


def _head_pred_bwd(entry, grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total, anchor_offset,
                   dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate):
    nc = w_cls.shape[0]
    rows = load_library().sy_head_pred_bwd_rows(cls_feat.n, cls_feat.h, cls_feat.w)
    partials = torch.empty((rows, (5 + nc) * (cls_feat.c + 1)), dtype=torch.float32, device=grad_raw.device)
    d = SyHeadPredBwdDesc()
    d.grad_raw = grad_raw.data_ptr()
    d.cls_feat, d.reg_feat, d.d_cls_feat, d.d_reg_feat = cls_feat.st(), reg_feat.st(), d_cls_feat.st(), d_reg_feat.st()
    d.w_reg, d.w_obj, d.w_cls = w_reg.data_ptr(), w_obj.data_ptr(), w_cls.data_ptr()
    d.num_classes, d.a_total, d.anchor_offset = nc, a_total, anchor_offset
    d.dw_reg, d.dw_obj, d.dw_cls = dw_reg.data_ptr(), dw_obj.data_ptr(), dw_cls.data_ptr()
    d.db_reg, d.db_obj, d.db_cls = db_reg.data_ptr(), db_obj.data_ptr(), db_cls.data_ptr()
    d.accumulate, d.partials, d.n_partials = int(accumulate), partials.data_ptr(), rows
    _check(getattr(lib(), entry)(C.byref(d), _stream()), kernels=3)


def add_(x: View, y: View):
    """y += x"""
    _check(lib().sy_add(x.st(), y.st(), _stream()))


def spp_maxpool_backward(x: View, d5: View, d9: View, d13: View, dx: View):
    ws = torch.empty(load_library().sy_spp_maxpool_backward_workspace_bytes(x.n, x.h, x.w, x.c), dtype=torch.uint8,
                     device=x.buf.device)
    _check(lib().sy_spp_maxpool_backward(x.st(), d5.st(), d9.st(), d13.st(), dx.st(), ws.data_ptr(), ws.numel(), _stream()),
           kernels=2)


def conv2d_plan(n, h, w, cin, cout, k, s, tile_mode=0, tile_bn=0):
    """Tiling decisions of the tensor-core conv for a layer shape (host-only: works without a GPU).  ``tile_mode``:
    0 = planner, 1 = linear tiles, 2 = halo where the conv is 3x3 stride 1; ``tile_bn``: 0 = planner, 64 or 128."""
    kh, kw = (k, k) if isinstance(k, int) else k
    p = SyConvPlan()
    rc = load_library().sy_conv2d_plan(n, h, w, cin, cout, kh, kw, s, tile_mode, tile_bn, C.byref(p))
    if rc != 0:
        raise RuntimeError("conv2d_plan: " + (load_library().sy_last_error_string() or b"").decode())
    return {f: getattr(p, f) for f, _ in SyConvPlan._fields_}


def sgd_nesterov_ema_step(param, grad, momentum_buf, ema, n_param, decay_begin, lr, momentum=0.9, weight_decay=5e-4,
                          inv_scale=1.0, nesterov=True, ema_decay=0.0, found_inf=None, hyper=None, found_inf_ema=False):
    """One fused optimiser step over flat fp32 state (sy_sgd_nesterov_ema_step); ``ema`` may be None.  ``hyper``: device
    fp32 [lr, momentum, weight_decay, inv_scale, ema_decay, 1 - ema_decay] replacing the scalars (CUDA-graph replays).
    ``found_inf``: device fp32 [1]; non-zero skips the step, and with ``found_inf_ema`` only the parameter and momentum
    update (the EMA still follows the unchanged parameters, as ModelEMA.update does on a step GradScaler skipped)."""
    d = SySgdEmaDesc()
    d.param, d.grad, d.momentum_buf = param.data_ptr(), grad.data_ptr(), momentum_buf.data_ptr()
    d.ema = ema.data_ptr() if ema is not None else None
    d.n_param, d.n_total, d.decay_begin = n_param, param.numel(), decay_begin
    d.lr, d.momentum, d.weight_decay, d.inv_scale, d.nesterov = lr, momentum, weight_decay, inv_scale, int(nesterov)
    d.ema_decay, d.ema_one_minus_decay = ema_decay, 1.0 - ema_decay
    d.found_inf = found_inf.data_ptr() if found_inf is not None else None
    d.hyper = hyper.data_ptr() if hyper is not None else None
    d.found_inf_ema = int(found_inf_ema)
    _check(lib().sy_sgd_nesterov_ema_step(C.byref(d), _stream()))


def nonfinite_flag(x, flag, count):
    """GradScaler's inf / NaN check (sy_nonfinite_flag) of a flat fp32 CUDA tensor ``x``: ``flag`` (fp32 [1]) becomes 1.0
    if any element is NaN or +-inf, else 0.0, and ``count`` (int32 [1]) goes up by one when it is 1.0.  Nothing is read
    back; capturable."""
    _require(x.dtype == torch.float32 and x.is_cuda and x.is_contiguous() and x.numel() > 0 and x.data_ptr() % 16 == 0,
             "nonfinite_flag: x must be a non-empty contiguous 16-byte aligned fp32 CUDA tensor")
    _require(flag.dtype == torch.float32 and flag.numel() == 1 and count.dtype == torch.int32 and count.numel() == 1
             and flag.device == x.device == count.device, "nonfinite_flag: flag must be fp32 [1], count int32 [1], on x's device")
    _check(lib().sy_nonfinite_flag(x.data_ptr(), x.numel(), flag.data_ptr(), count.data_ptr(), _stream()))


def resize_bilinear(x, size, out=None):
    """F.interpolate(x, size=size, mode="bilinear", align_corners=False) of an NCHW fp32 batch on the device.  ``out``: a
    contiguous fp32 [B, C, size] tensor to write into (the static input of a CUDA graph) instead of a new one."""
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    b, c, hi, wi = x.shape
    if out is None:
        y = torch.empty((b, c, size[0], size[1]), dtype=torch.float32, device=x.device)
    else:
        _require(out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (b, c, size[0], size[1])
                 and out.device == x.device, f"resize_bilinear: out must be contiguous fp32 {(b, c, size[0], size[1])}")
        y = out
    _check(lib().sy_resize_bilinear(x.data_ptr(), b * c, hi, wi, y.data_ptr(), size[0], size[1], _stream()))
    return y


def scale_labels_(labels, sx, sy):
    """labels[..., 1::2] *= sx; labels[..., 2::2] *= sy (in place; [.., cols] fp32 contiguous)."""
    assert labels.dtype == torch.float32 and labels.is_contiguous()
    cols = labels.shape[-1]
    _check(lib().sy_scale_labels(labels.data_ptr(), labels.numel() // cols, cols, sx, sy, _stream()))
    return labels


def _require(cond, msg):
    if not cond:
        raise RuntimeError(msg)


def _tensor_ok(t, dtype, dim):
    return torch.is_tensor(t) and t.dtype == dtype and t.dim() == dim and t.is_contiguous()


def pair_labels(ann, counts, mirror, flip, width, r, labels_fut, labels_cur, flags):
    """Label half of DoubleTrainTransform on the device (sy_pair_labels): ``ann`` fp64 [B, 2, M, 5] (x1, y1, x2, y2, cls),
    ``counts`` int32 [B, 2], ``mirror`` int32 [B] (or None without flip); writes fp32 [B, max_labels, 5] ``labels_fut`` /
    ``labels_cur`` and the int32 [B, 2] effective mirror bits ``flags``."""
    _require(_tensor_ok(ann, torch.float64, 4) and ann.shape[1] == 2 and ann.shape[3] == 5,
             "pair_labels: annotations must be contiguous float64 [B, 2, M, 5]")
    b = ann.shape[0]
    _require(_tensor_ok(counts, torch.int32, 2) and tuple(counts.shape) == (b, 2), "pair_labels: counts must be int32 [B, 2]")
    _require(mirror is None or (_tensor_ok(mirror, torch.int32, 1) and mirror.shape[0] == b),
             "pair_labels: mirror must be int32 [B]")
    for t in (labels_fut, labels_cur):
        _require(_tensor_ok(t, torch.float32, 3) and t.shape[0] == b and t.shape[2] == 5 and t.shape == labels_fut.shape,
                 "pair_labels: labels must be float32 [B, max_labels, 5]")
    _require(_tensor_ok(flags, torch.int32, 2) and tuple(flags.shape) == (b, 2), "pair_labels: flags must be int32 [B, 2]")
    d = SyPairLabelsDesc()
    d.ann, d.counts = ann.data_ptr(), counts.data_ptr()
    d.mirror = mirror.data_ptr() if mirror is not None else None
    d.n_items, d.max_rows, d.max_labels, d.flip = b, ann.shape[2], labels_fut.shape[1], int(flip)
    d.width, d.r = width, r
    d.labels_fut, d.labels_cur, d.flags_out = labels_fut.data_ptr(), labels_cur.data_ptr(), flags.data_ptr()
    _check(lib().sy_pair_labels(C.byref(d), _stream()))


def frame_labels(ann, counts, mirror, flip, width, r, labels, flags):
    """Label half of TrainTransform on the device (sy_frame_labels): ``ann`` fp64 [B, M, 5] (x1, y1, x2, y2, cls),
    ``counts`` int32 [B], ``mirror`` int32 [B] (or None without flip); writes fp32 [B, max_labels, 5] ``labels`` and the
    int32 [B] effective mirror bits ``flags``."""
    _require(_tensor_ok(ann, torch.float64, 3) and ann.shape[2] == 5,
             "frame_labels: annotations must be contiguous float64 [B, M, 5]")
    b = ann.shape[0]
    _require(_tensor_ok(counts, torch.int32, 1) and counts.shape[0] == b, "frame_labels: counts must be int32 [B]")
    _require(mirror is None or (_tensor_ok(mirror, torch.int32, 1) and mirror.shape[0] == b),
             "frame_labels: mirror must be int32 [B]")
    _require(_tensor_ok(labels, torch.float32, 3) and labels.shape[0] == b and labels.shape[2] == 5,
             "frame_labels: labels must be float32 [B, max_labels, 5]")
    _require(_tensor_ok(flags, torch.int32, 1) and flags.shape[0] == b, "frame_labels: flags must be int32 [B]")
    d = SyFrameLabelsDesc()
    d.ann, d.counts = ann.data_ptr(), counts.data_ptr()
    d.mirror = mirror.data_ptr() if mirror is not None else None
    d.n, d.max_rows, d.max_labels, d.flip = b, ann.shape[1], labels.shape[1], int(flip)
    d.width, d.r = width, r
    d.labels, d.flags_out = labels.data_ptr(), flags.data_ptr()
    _check(lib().sy_frame_labels(C.byref(d), _stream()))


def letterbox(src, mid, dst, out, flags=None):
    """uint8 [n, h, w, 3] frames -> fp32 [n * 3 / C, C, H, W] ``out`` (sy_letterbox): cv2-exact resize to ``mid`` (h, w),
    mirror where int32 ``flags[i]`` is set, cv2-exact resize to ``dst``, top-left on a canvas of 114."""
    _require(_tensor_ok(src, torch.uint8, 4) and src.shape[3] == 3, "letterbox: frames must be contiguous uint8 [n, h, w, 3]")
    n, h, w, _ = src.shape
    _require(_tensor_ok(out, torch.float32, 4) and out.numel() == n * 3 * out.shape[2] * out.shape[3],
             "letterbox: out must be contiguous float32 holding [n, 3, H, W]")
    _require(flags is None or (torch.is_tensor(flags) and flags.dtype == torch.int32 and flags.is_contiguous()
                               and flags.numel() == n), "letterbox: flags must be int32 [n]")
    d = SyLetterboxDesc(src.data_ptr(), n, h, w, mid[0], mid[1], dst[0], dst[1], out.shape[2], out.shape[3],
                        flags.data_ptr() if flags is not None else None, out.data_ptr())
    _check(lib().sy_letterbox(C.byref(d), _stream()))


def letterbox_sized(src, sizes, out):
    """uint8 [n, slot_h, slot_w, 3] slots -> fp32 [n, 3, H, W] ``out`` (sy_letterbox_sized): frame k of ``sizes[k]`` = (h, w,
    dst_h, dst_w) (int32 [n, 4] on the device) at the slot's top-left, cv2-exact resize to dst, top-left on a canvas of 114."""
    _require(_tensor_ok(src, torch.uint8, 4) and src.shape[3] == 3 and src.is_cuda,
             "letterbox_sized: frames must be contiguous CUDA uint8 [n, slot_h, slot_w, 3]")
    n, sh, sw, _ = src.shape
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 4) and sizes.device == src.device,
             f"letterbox_sized: sizes must be int32 [{n}, 4] on the frames' device")
    _require(_tensor_ok(out, torch.float32, 4) and out.shape[0] == n and out.shape[1] == 3 and out.device == src.device,
             f"letterbox_sized: out must be contiguous float32 [{n}, 3, H, W] on the frames' device")
    d = SyLetterboxSizedDesc(src.data_ptr(), n, sh, sw, sizes.data_ptr(), out.shape[2], out.shape[3], out.data_ptr())
    _check(lib().sy_letterbox_sized(C.byref(d), _stream()))


def resize_sized(src, sizes, out):
    """uint8 [n, slot_h, slot_w, 3] slots -> uint8 [n, out_h, out_w, 3] ``out`` slots (sy_resize_sized): frame k of
    ``sizes[k]`` = (h, w, dst_h, dst_w) (int32 [n, 4] on the device) at the slot's top-left, cv2-exact INTER_LINEAR resize
    to dst at the top-left of out slot k; the rest of ``out`` is not written.  Enqueues only (capturable)."""
    _require(_tensor_ok(src, torch.uint8, 4) and src.shape[3] == 3 and src.is_cuda,
             "resize_sized: frames must be contiguous CUDA uint8 [n, slot_h, slot_w, 3]")
    n, sh, sw, _ = src.shape
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 4) and sizes.device == src.device,
             f"resize_sized: sizes must be int32 [{n}, 4] on the frames' device")
    _require(_tensor_ok(out, torch.uint8, 4) and out.shape[0] == n and out.shape[3] == 3 and out.device == src.device
             and out.data_ptr() != src.data_ptr(), f"resize_sized: out must be another contiguous uint8 [{n}, H, W, 3] "
             "on the frames' device")
    d = SyResizeSizedDesc(src.data_ptr(), n, sh, sw, sizes.data_ptr(), out.shape[1], out.shape[2], out.data_ptr())
    _check(lib().sy_resize_sized(C.byref(d), _stream()))
    return out


class PackBatch:
    """Every conv operand of a model re-packed in ONE launch (sy_pack_conv_weights_batch).  ``add`` the (fp32 parameter,
    bf16 destination, layout) pairs once -- the tensors must keep their addresses -- then ``run()`` after every update."""

    def __init__(self, device):
        self.device, self.items, self.total, self.table = device, [], 0, None

    def add(self, w, out, mode, out_pitch=0, co_offset=0):
        assert w.dtype == torch.float32 and w.is_contiguous() and out.dtype == torch.bfloat16
        o, i, kh, kw = w.shape
        it = SyPackItem(w.data_ptr(), out.data_ptr(), o, i, kh, kh * kw, mode, co_offset, out_pitch, self.total)
        self.items.append(it)
        self.total += load_library().sy_pack_item_tiles(o, i, mode)      # work tiles (see include/streamyolo_sm100.h)

    def run(self):
        if self.table is None:
            arr = (SyPackItem * len(self.items))(*self.items)
            self.table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.device)
        _check(lib().sy_pack_conv_weights_batch(self.table.data_ptr(), len(self.items), self.total, _stream()))


def jpeg_decode_workspace_bytes(n, max_bytes, h, w):
    """bytes of the sy_jpeg_decode workspace for n frames of h x w stored in rows of max_bytes (host-only)"""
    need = load_library().sy_jpeg_decode_workspace_bytes(n, max_bytes, h, w)
    _require(need > 0, f"jpeg_decode: bad sizes (n {n}, max_bytes {max_bytes}, {h}x{w})")
    return need


def jpeg_decode(streams, lengths, out, status, workspace):
    """Decode n JPEG files into uint8 BGR frames (sy_jpeg_decode): ``streams`` uint8 [n, max_bytes] file bytes, ``lengths``
    int32 [n], ``out`` uint8 [n, h, w, 3], ``status`` int32 [n] (SY_JPEG_*), ``workspace`` uint8 of at least
    jpeg_decode_workspace_bytes(n, max_bytes, h, w) bytes, all on one CUDA device.  Nothing is read back."""
    _require(_tensor_ok(streams, torch.uint8, 2), "jpeg_decode: streams must be contiguous uint8 [n, max_bytes]")
    n, max_bytes = streams.shape
    _require(_tensor_ok(lengths, torch.int32, 1) and lengths.shape[0] == n, "jpeg_decode: lengths must be int32 [n]")
    _require(_tensor_ok(out, torch.uint8, 4) and out.shape[0] == n and out.shape[3] == 3,
             "jpeg_decode: out must be contiguous uint8 [n, h, w, 3]")
    _require(_tensor_ok(status, torch.int32, 1) and status.shape[0] == n, "jpeg_decode: status must be int32 [n]")
    need = jpeg_decode_workspace_bytes(n, max_bytes, out.shape[1], out.shape[2])
    _require(_tensor_ok(workspace, torch.uint8, 1) and workspace.numel() >= need,
             f"jpeg_decode: workspace must be contiguous uint8 of at least {need} bytes")
    _require(len({t.device for t in (streams, lengths, out, status, workspace)}) == 1 and streams.is_cuda,
             "jpeg_decode: all tensors must be on one CUDA device")
    d = SyJpegDecodeDesc(streams.data_ptr(), lengths.data_ptr(), n, max_bytes, out.shape[1], out.shape[2], out.data_ptr(),
                         status.data_ptr(), workspace.data_ptr(), workspace.numel())
    _check(lib().sy_jpeg_decode(C.byref(d), _stream()), kernels=5)


def jpeg_decode_sized_workspace_bytes(n, max_bytes, max_h, max_w):
    """bytes of the sy_jpeg_decode_sized workspace for n frames in slots of max_h x max_w, stored in rows of max_bytes"""
    need = load_library().sy_jpeg_decode_sized_workspace_bytes(n, max_bytes, max_h, max_w)
    _require(need > 0, f"jpeg_decode_sized: bad sizes (n {n}, max_bytes {max_bytes}, slot {max_h}x{max_w})")
    return need


def jpeg_decode_sized(streams, lengths, sizes, out, status, workspace):
    """Decode n JPEG files of their own sizes (sy_jpeg_decode_sized): ``sizes`` int32 [n, 2] expected (h, w), ``out`` uint8
    [n, max_h, max_w, 3] slots, the rest as jpeg_decode.  Nothing is read back."""
    _require(_tensor_ok(streams, torch.uint8, 2), "jpeg_decode_sized: streams must be contiguous uint8 [n, max_bytes]")
    n, max_bytes = streams.shape
    _require(_tensor_ok(lengths, torch.int32, 1) and lengths.shape[0] == n, "jpeg_decode_sized: lengths must be int32 [n]")
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2), "jpeg_decode_sized: sizes must be int32 [n, 2]")
    _require(_tensor_ok(out, torch.uint8, 4) and out.shape[0] == n and out.shape[3] == 3,
             "jpeg_decode_sized: out must be contiguous uint8 [n, max_h, max_w, 3]")
    _require(_tensor_ok(status, torch.int32, 1) and status.shape[0] == n, "jpeg_decode_sized: status must be int32 [n]")
    need = jpeg_decode_sized_workspace_bytes(n, max_bytes, out.shape[1], out.shape[2])
    _require(_tensor_ok(workspace, torch.uint8, 1) and workspace.numel() >= need,
             f"jpeg_decode_sized: workspace must be contiguous uint8 of at least {need} bytes")
    _require(len({t.device for t in (streams, lengths, sizes, out, status, workspace)}) == 1 and streams.is_cuda,
             "jpeg_decode_sized: all tensors must be on one CUDA device")
    d = SyJpegDecodeSizedDesc(streams.data_ptr(), lengths.data_ptr(), n, max_bytes, sizes.data_ptr(), out.shape[1],
                              out.shape[2], out.data_ptr(), status.data_ptr(), workspace.data_ptr(), workspace.numel())
    _check(lib().sy_jpeg_decode_sized(C.byref(d), _stream()), kernels=5)


# frame_format -> SY_YUV_* of sy_yuv_to_bgr_sized (each the cv2.cvtColor code it replaces: COLOR_YUV2BGR_NV12, ...)
YUV_FORMATS = {"nv12": 0, "nv21": 1, "i420": 2, "yv12": 3, "yuyv": 4, "uyvy": 5}


def yuv_to_bgr_sized(src, sizes, fmt, out):
    """Raw YUV frames -> uint8 BGR slots (sy_yuv_to_bgr_sized), cv2.cvtColor(COLOR_YUV2BGR_*) bit for bit: ``src`` uint8
    [n, max_bytes], frame i in the first bytes of row i in cv2's layout of ``fmt`` (a YUV_FORMATS key); ``sizes`` int32
    [n, 2] (h, w), h = 0 for no frame; ``out`` uint8 [n, slot_h, slot_w, 3], frame i at the top-left of slot i.  A row
    with no frame, an odd size where the format subsamples, or a frame that does not fit leaves its slot untouched."""
    _require(fmt in YUV_FORMATS, f"yuv_to_bgr_sized: unknown format {fmt!r} (one of {', '.join(YUV_FORMATS)})")
    _require(_tensor_ok(src, torch.uint8, 2) and src.is_cuda, "yuv_to_bgr_sized: src must be contiguous CUDA uint8 [n, max_bytes]")
    n, max_bytes = src.shape
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == src.device,
             f"yuv_to_bgr_sized: sizes must be int32 [{n}, 2] on src's device")
    _require(_tensor_ok(out, torch.uint8, 4) and out.shape[0] == n and out.shape[3] == 3 and out.device == src.device,
             f"yuv_to_bgr_sized: out must be contiguous uint8 [{n}, slot_h, slot_w, 3] on src's device")
    d = SyYuvToBgrSizedDesc(src.data_ptr(), n, max_bytes, sizes.data_ptr(), YUV_FORMATS[fmt], out.shape[1], out.shape[2],
                            out.data_ptr())
    _check(lib().sy_yuv_to_bgr_sized(C.byref(d), _stream()))


# the colour order of a mosaic's top-left 2x2 -> SY_BAYER_* of sy_bayer_to_bgr_sized (cv2's COLOR_BayerRGGB2BGR, ... --
# the aliases of COLOR_BayerBG2BGR, _RG, _GR, _GB), and the demosaicing -> SY_DEMOSAIC_* (COLOR_Bayer*2BGR, ..._EA)
BAYER_PATTERNS = {"rggb": 0, "bggr": 1, "gbrg": 2, "grbg": 3}
DEMOSAIC = {"bilinear": 0, "ea": 1}


def bayer_to_bgr_sized(src, sizes, pattern, algo, out):
    """8-bit Bayer mosaics -> uint8 BGR slots (sy_bayer_to_bgr_sized), cv2.cvtColor(COLOR_Bayer*2BGR[_EA]) bit for bit:
    ``src`` uint8 [n, max_bytes], frame i the first h * w bytes of row i, row-major [h, w]; ``pattern`` a BAYER_PATTERNS
    key (the colour order of the top-left 2x2), ``algo`` a DEMOSAIC key; ``sizes`` int32 [n, 2] (h, w), h = 0 for no
    frame; ``out`` uint8 [n, slot_h, slot_w, 3], frame i at the top-left of slot i.  A row with no frame, or a frame that
    does not fit, leaves its slot untouched."""
    _require(pattern in BAYER_PATTERNS,
             f"bayer_to_bgr_sized: unknown pattern {pattern!r} (one of {', '.join(BAYER_PATTERNS)})")
    _require(algo in DEMOSAIC, f"bayer_to_bgr_sized: unknown demosaicing {algo!r} (one of {', '.join(DEMOSAIC)})")
    _require(_tensor_ok(src, torch.uint8, 2) and src.is_cuda, "bayer_to_bgr_sized: src must be contiguous CUDA uint8 [n, max_bytes]")
    n, max_bytes = src.shape
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == src.device,
             f"bayer_to_bgr_sized: sizes must be int32 [{n}, 2] on src's device")
    _require(_tensor_ok(out, torch.uint8, 4) and out.shape[0] == n and out.shape[3] == 3 and out.device == src.device,
             f"bayer_to_bgr_sized: out must be contiguous uint8 [{n}, slot_h, slot_w, 3] on src's device")
    d = SyBayerToBgrSizedDesc(src.data_ptr(), n, max_bytes, sizes.data_ptr(), BAYER_PATTERNS[pattern], DEMOSAIC[algo],
                              out.shape[1], out.shape[2], out.data_ptr())
    _check(lib().sy_bayer_to_bgr_sized(C.byref(d), _stream()))


def jpeg_encode_max_bytes(h, w):
    """a file length no h x w JPEG of sy_jpeg_encode exceeds, for any content and quality"""
    need = load_library().sy_jpeg_encode_max_bytes(h, w)
    _require(need > 0, f"jpeg_encode_max_bytes: bad size {h}x{w}")
    return need


def jpeg_encode_workspace_bytes(n, max_h, max_w, max_bytes):
    """bytes of the sy_jpeg_encode workspace for n images in slots of max_h x max_w and files of at most max_bytes"""
    need = load_library().sy_jpeg_encode_workspace_bytes(n, max_h, max_w, max_bytes)
    _require(need > 0, f"jpeg_encode: bad sizes (n {n}, slot {max_h}x{max_w}, max_bytes {max_bytes})")
    return need


def jpeg_encode(src, sizes, quality, out, lengths, status, workspace):
    """Encode n BGR images of their own sizes into what cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, quality])
    returns (sy_jpeg_encode): ``src`` uint8 [n, max_h, max_w, 3], image i at the top-left of slot i; ``sizes`` int32
    [n, 2] (h, w) on the device; ``out`` uint8 [n, max_bytes], file i in the first ``lengths[i]`` bytes of row i;
    ``lengths`` int64 [n]; ``status`` int32 [n] (0 ok, 1 the file does not fit in max_bytes, 2 a size row outside the
    slot); ``workspace`` uint8 of jpeg_encode_workspace_bytes.  Enqueues only (capturable)."""
    _require(isinstance(quality, int) and 1 <= quality <= 100,
             f"jpeg_encode: quality must be an integer in 1..100, not {quality!r}")
    _require(_tensor_ok(src, torch.uint8, 4) and src.shape[3] == 3 and src.is_cuda,
             "jpeg_encode: src must be contiguous CUDA uint8 [n, max_h, max_w, 3]")
    n, mh, mw, _ = src.shape
    dev = src.device
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == dev,
             f"jpeg_encode: sizes must be int32 [{n}, 2] on src's device")
    _require(_tensor_ok(out, torch.uint8, 2) and out.shape[0] == n and out.device == dev,
             f"jpeg_encode: out must be contiguous uint8 [{n}, max_bytes] on src's device")
    _require(_tensor_ok(lengths, torch.int64, 1) and lengths.shape[0] == n and lengths.device == dev,
             f"jpeg_encode: lengths must be int64 [{n}] on src's device")
    _require(_tensor_ok(status, torch.int32, 1) and status.shape[0] == n and status.device == dev,
             f"jpeg_encode: status must be int32 [{n}] on src's device")
    need = jpeg_encode_workspace_bytes(n, mh, mw, out.shape[1])
    _require(_tensor_ok(workspace, torch.uint8, 1) and workspace.numel() >= need and workspace.device == dev,
             f"jpeg_encode: workspace must be contiguous uint8 of at least {need} bytes on src's device")
    d = SyJpegEncodeDesc(src.data_ptr(), sizes.data_ptr(), n, mh, mw, int(quality), out.data_ptr(), out.shape[1],
                         lengths.data_ptr(), status.data_ptr(), workspace.data_ptr(), workspace.numel())
    _check(lib().sy_jpeg_encode(C.byref(d), _stream()), kernels=8)


def draw_boxes(src, sizes, boxes, labels, counts, palette, dst):
    """Draw the boxes of the sAP toolkit's vis_obj_fancy (vis_det_th.py:99-120, no text) on n images of their own sizes
    (sy_draw_boxes): ``src`` / ``dst`` uint8 [n, max_h, max_w, 3] (the same tensor draws in place), image i of
    ``sizes[i]`` = (h, w) (int32 [n, 2]) at the top-left of slot i; ``boxes`` int32 [n, K, 4] (x1, y1, x2, y2, rounded),
    ``labels`` int32 [n, K], ``counts`` int32 [n] (the first counts[i] boxes of row i are drawn); ``palette`` uint8
    [P, 3] in the images' channel order.  Only pixels a box touches are written.  Enqueues only (capturable)."""
    _require(_tensor_ok(src, torch.uint8, 4) and src.shape[3] == 3 and src.is_cuda,
             "draw_boxes: src must be contiguous CUDA uint8 [n, max_h, max_w, 3]")
    n, mh, mw, _ = src.shape
    dev = src.device
    _require(_tensor_ok(dst, torch.uint8, 4) and tuple(dst.shape) == tuple(src.shape) and dst.device == dev,
             f"draw_boxes: dst must be contiguous uint8 {list(src.shape)} on src's device")
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == dev,
             f"draw_boxes: sizes must be int32 [{n}, 2] on src's device")
    _require(_tensor_ok(boxes, torch.int32, 3) and boxes.shape[0] == n and boxes.shape[2] == 4 and boxes.shape[1] >= 1
             and boxes.device == dev and boxes.data_ptr() % 16 == 0,
             f"draw_boxes: boxes must be contiguous 16-byte aligned int32 [{n}, K, 4] on src's device")
    k = boxes.shape[1]
    _require(_tensor_ok(labels, torch.int32, 2) and tuple(labels.shape) == (n, k) and labels.device == dev,
             f"draw_boxes: labels must be int32 [{n}, {k}] on src's device")
    _require(_tensor_ok(counts, torch.int32, 1) and counts.shape[0] == n and counts.device == dev,
             f"draw_boxes: counts must be int32 [{n}] on src's device")
    _require(_tensor_ok(palette, torch.uint8, 2) and palette.shape[1] == 3 and 1 <= palette.shape[0] <= 65536
             and palette.device == dev, "draw_boxes: palette must be contiguous uint8 [P, 3] (1 <= P <= 65536) on src's "
             "device")
    d = SyDrawBoxesDesc(src.data_ptr(), sizes.data_ptr(), n, mh, mw, boxes.data_ptr(), labels.data_ptr(),
                        counts.data_ptr(), k, palette.data_ptr(), palette.shape[0], dst.data_ptr(), dst.shape[1],
                        dst.shape[2])
    _check(lib().sy_draw_boxes(C.byref(d), _stream()))
    return dst


def vis_det_boxes(det, count, score_th, boxes=None, labels=None, counts=None):
    """A streaming tick's NMS rows (fp32 [S, A, 7]: x1, y1, x2, y2 already divided by the ratio, obj, class_conf,
    class_pred; ``count`` int32 [S]) -> draw_boxes's (boxes int32 [S, A, 4], labels int32 [S, A], counts int32 [S]) for
    the rows whose fp32 score obj * class_conf is >= ``score_th`` (fp32; -inf keeps every row), in order, the boxes taken
    through the ltwh round trip and rounded half to even (sy_vis_det_boxes).  Writes into the given buffers (allocated
    when None).  Enqueues only (capturable)."""
    _require(_tensor_ok(det, torch.float32, 3) and det.shape[2] == 7 and det.is_cuda,
             "vis_det_boxes: det must be contiguous CUDA float32 [S, A, 7]")
    s, a, _ = det.shape
    dev = det.device
    _require(_tensor_ok(count, torch.int32, 1) and count.shape[0] == s and count.device == dev,
             f"vis_det_boxes: count must be int32 [{s}] on det's device")
    if boxes is None:
        boxes = torch.empty((s, a, 4), dtype=torch.int32, device=dev)
        labels = torch.empty((s, a), dtype=torch.int32, device=dev)
        counts = torch.empty((s,), dtype=torch.int32, device=dev)
    _require(_tensor_ok(boxes, torch.int32, 3) and tuple(boxes.shape) == (s, a, 4) and boxes.device == dev
             and boxes.data_ptr() % 16 == 0, f"vis_det_boxes: boxes must be 16-byte aligned int32 [{s}, {a}, 4]")
    _require(_tensor_ok(labels, torch.int32, 2) and tuple(labels.shape) == (s, a) and labels.device == dev,
             f"vis_det_boxes: labels must be int32 [{s}, {a}]")
    _require(_tensor_ok(counts, torch.int32, 1) and counts.shape[0] == s and counts.device == dev,
             f"vis_det_boxes: counts must be int32 [{s}]")
    d = SyVisDetBoxesDesc(det.data_ptr(), count.data_ptr(), s, a, float(score_th), boxes.data_ptr(),
                          labels.data_ptr(), counts.data_ptr())
    _check(lib().sy_vis_det_boxes(C.byref(d), _stream()))
    return boxes, labels, counts


def draw_outlines(img, sizes, boxes, counts, points, n_points, color):
    """The drawing of the sAP toolkit's vis_det (sAP/det/__init__.py:152-174) on n images of their own sizes, in place
    (sy_draw_outlines): ``img`` uint8 [n, max_h, max_w, 3], image i of ``sizes[i]`` = (h, w) (int32 [n, 2]) at the
    top-left of slot i; the 1-pixel rectangles of the first counts[i] boxes of ``boxes`` (int32 [n, K, 4] x1, y1, x2, y2,
    rounded) and the pixels y * w + x of the first n_points[i] entries of ``points`` (int32 [n, M]) become ``color`` (3
    values in the images' channel order).  Only those pixels are written.  Enqueues only (capturable)."""
    _require(_tensor_ok(img, torch.uint8, 4) and img.shape[3] == 3 and img.is_cuda,
             "draw_outlines: img must be contiguous CUDA uint8 [n, max_h, max_w, 3]")
    n, mh, mw, _ = img.shape
    dev = img.device
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == dev,
             f"draw_outlines: sizes must be int32 [{n}, 2] on img's device")
    _require(_tensor_ok(boxes, torch.int32, 3) and boxes.shape[0] == n and boxes.shape[2] == 4 and boxes.shape[1] >= 1
             and boxes.device == dev and boxes.data_ptr() % 16 == 0,
             f"draw_outlines: boxes must be contiguous 16-byte aligned int32 [{n}, K, 4] on img's device")
    _require(_tensor_ok(points, torch.int32, 2) and points.shape[0] == n and points.shape[1] >= 1 and points.device == dev,
             f"draw_outlines: points must be contiguous int32 [{n}, M] on img's device")
    for name, t in (("counts", counts), ("n_points", n_points)):
        _require(_tensor_ok(t, torch.int32, 1) and t.shape[0] == n and t.device == dev,
                 f"draw_outlines: {name} must be int32 [{n}] on img's device")
    col = [int(c) for c in color]
    _require(len(col) == 3 and all(0 <= c <= 255 for c in col), "draw_outlines: color must be 3 values in 0..255")
    d = SyDrawOutlinesDesc(img.data_ptr(), sizes.data_ptr(), n, mh, mw, boxes.data_ptr(), counts.data_ptr(),
                           boxes.shape[1], points.data_ptr(), n_points.data_ptr(), points.shape[1], (C.c_uint8 * 3)(*col))
    _check(lib().sy_draw_outlines(C.byref(d), _stream()))
    return img


def splice_frames(a, b, sizes, splits, horizontal, color):
    """The split screen of the sAP toolkit's vis_contrast.py (:148-165) on n pairs of images of their own sizes
    (sy_splice_frames), written into ``a`` in place: ``a`` / ``b`` uint8 [n, max_h, max_w, 3], pair i of ``sizes[i]`` =
    (h, w) (int32 [n, 2]) at the top-left of slot i; ``splits`` int32 [n, 3] (split, band_start, band_end) along the
    columns, or the rows with ``horizontal``: a pixel in [band_start, band_end) gets ``color`` (3 values in the images'
    channel order), else one at or past ``split`` gets B's pixel, else it keeps A's.  Enqueues only (capturable)."""
    _require(_tensor_ok(a, torch.uint8, 4) and a.shape[3] == 3 and a.is_cuda,
             "splice_frames: a must be contiguous CUDA uint8 [n, max_h, max_w, 3]")
    n, mh, mw, _ = a.shape
    dev = a.device
    _require(_tensor_ok(b, torch.uint8, 4) and tuple(b.shape) == tuple(a.shape) and b.device == dev,
             f"splice_frames: b must be contiguous uint8 {list(a.shape)} on a's device")
    _require(a.data_ptr() != b.data_ptr(), "splice_frames: a and b must be different buffers")
    _require(_tensor_ok(sizes, torch.int32, 2) and tuple(sizes.shape) == (n, 2) and sizes.device == dev,
             f"splice_frames: sizes must be int32 [{n}, 2] on a's device")
    _require(_tensor_ok(splits, torch.int32, 2) and tuple(splits.shape) == (n, 3) and splits.device == dev,
             f"splice_frames: splits must be int32 [{n}, 3] on a's device")
    col = [int(c) for c in color]
    _require(len(col) == 3 and all(0 <= c <= 255 for c in col), "splice_frames: color must be 3 values in 0..255")
    d = SySpliceFramesDesc(a.data_ptr(), b.data_ptr(), sizes.data_ptr(), splits.data_ptr(), n, mh, mw, int(bool(horizontal)),
                           (C.c_uint8 * 3)(*col))
    _check(lib().sy_splice_frames(C.byref(d), _stream()))
    return a
