"""ctypes binding of libyolov6_b200.so (C ABI declared in include/yv6.h).

The product path has no CPU or PyTorch fallback: if the shared library is missing, or was built
without the requested symbol, loading fails loudly with RuntimeError.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libyolov6_b200.so")

ACT_NONE, ACT_RELU, ACT_SILU, ACT_SIGMOID, ACT_HARDSWISH = 0, 1, 2, 3, 4
DT_BF16, DT_F32, DT_U8, DT_F16 = 0, 1, 2, 3
PAD_SAME = -1000000
ACT_CODES = {None: ACT_NONE, "none": ACT_NONE, "relu": ACT_RELU, "silu": ACT_SILU, "sigmoid": ACT_SIGMOID, "hardswish": ACT_HARDSWISH}


class ConvDesc(C.Structure):
    """Mirror of `yv6_conv_desc` (include/yv6.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32),
        ("x_c_total", C.c_int32), ("x_plane_stride", C.c_int64),
        ("w", C.c_void_p), ("w_plane_stride", C.c_int64), ("bias", C.c_void_p),
        ("Cout", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("act", C.c_int32),
        ("y", C.c_void_p), ("y_dtype", C.c_int32),
        ("y_img_stride", C.c_int64), ("y_h_stride", C.c_int64), ("y_w_stride", C.c_int64),
        ("y_plane_stride", C.c_int64),
        ("res", C.c_void_p), ("alpha", C.c_float),
        ("res_img_stride", C.c_int64), ("res_h_stride", C.c_int64), ("res_w_stride", C.c_int64),
        ("res_plane_stride", C.c_int64),
        ("nsplit", C.c_int32),
        ("force_bw", C.c_int32), ("force_bh", C.c_int32), ("force_bi", C.c_int32), ("force_bn", C.c_int32),
        ("force_stages", C.c_int32), ("force_grid", C.c_int32), ("force_direct", C.c_int32), ("force_halo", C.c_int32),
        ("pad_w", C.c_int32), ("out_h", C.c_int32), ("out_w", C.c_int32), ("force_groups", C.c_int32),
        ("trace", C.c_void_p), ("stride_w", C.c_int32), ("force_pair", C.c_int32), ("pair_view", C.c_int32),
        ("reserved0", C.c_int32),     # operand dtype: 0 = bf16, DT_F16 = fp16
    ]


class StemDesc(C.Structure):
    """Mirror of `yv6_stem_desc` (include/yv6.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("x_dtype", C.c_int32), ("in_scale", C.c_float),
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("w", C.c_void_p), ("bias", C.c_void_p),
        ("Cout", C.c_int32), ("act", C.c_int32),
        ("y", C.c_void_p), ("y_plane_stride", C.c_int64), ("nsplit", C.c_int32), ("fp32_math", C.c_int32),
        ("force_sync_loads", C.c_int32),
    ]


class LossDesc(C.Structure):
    """Mirror of `yv6_loss_desc` (include/yv6.h)."""
    _fields_ = [
        ("pred_scores", C.c_void_p), ("pred_distri", C.c_void_p), ("anc_points", C.c_void_p), ("strides", C.c_void_p),
        ("gt", C.c_void_p), ("gt_idx", C.c_void_p), ("fg", C.c_void_p), ("norm", C.c_void_p),
        ("B", C.c_int32), ("A", C.c_int32), ("G", C.c_int32), ("nc", C.c_int32), ("reg_ch", C.c_int32),
        ("iou_type", C.c_int32),
        ("w_cls", C.c_double), ("w_iou", C.c_double), ("w_dfl", C.c_double), ("grad_scale", C.c_double),
        ("grad_scores", C.c_void_p), ("grad_distri", C.c_void_p), ("out", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("norm_gt_zero", C.c_int32),
    ]


class WgradDesc(C.Structure):
    """Mirror of `yv6_wgrad_desc` (include/yv6.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32), ("x_c_total", C.c_int32),
        ("dy", C.c_void_p), ("Cout", C.c_int32), ("dy_c_total", C.c_int32),
        ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("dw", C.c_void_p), ("force_ksplit", C.c_int32), ("force_taps", C.c_int32),
    ]


class BnDesc(C.Structure):
    """Mirror of `yv6_bn_desc` (include/yv6.h)."""
    _fields_ = [
        ("nb", C.c_int32), ("act", C.c_int32), ("C", C.c_int32), ("pixels", C.c_int64),
        ("x", C.c_void_p * 3), ("x_pitch", C.c_int64 * 3),
        ("mean", C.c_void_p * 3), ("invstd", C.c_void_p * 3), ("scale", C.c_void_p * 3), ("shift", C.c_void_p * 3),
        ("y", C.c_void_p), ("y_pitch", C.c_int64),
        ("dy", C.c_void_p), ("dy_pitch", C.c_int64),
        ("s1", C.c_void_p), ("s2", C.c_void_p * 3),
        ("dx", C.c_void_p * 3), ("dx_pitch", C.c_int64 * 3), ("accumulate", C.c_int32 * 3),
        ("res", C.c_void_p), ("res_pitch", C.c_int64), ("res_alpha", C.c_float),
        ("dres", C.c_void_p), ("dres_pitch", C.c_int64), ("dalpha", C.c_void_p),
        ("res_alpha_dev", C.c_void_p),
        ("work", C.c_void_p), ("counter", C.c_void_p), ("coef", C.c_void_p), ("zeroed", C.c_int32), ("dres_assign", C.c_int32),
    ]


class BnStatsDesc(C.Structure):
    """Mirror of `yv6_bn_stats_desc` (include/yv6.h)."""
    _fields_ = [
        ("nb", C.c_int32), ("C", C.c_int32), ("pixels", C.c_int64),
        ("x", C.c_void_p * 3), ("x_pitch", C.c_int64 * 3),
        ("sums", C.c_void_p), ("counter", C.c_void_p), ("zeroed", C.c_int32),
        ("gamma", C.c_void_p * 3), ("beta", C.c_void_p * 3),
        ("running_mean", C.c_void_p * 3), ("running_var", C.c_void_p * 3),
        ("stats", C.c_void_p * 3),
        ("eps", C.c_float), ("momentum", C.c_float),
    ]


class XformSeg(C.Structure):
    """Mirror of `yv6_xform_seg` (include/yv6.h)."""
    _fields_ = [
        ("dst", C.c_void_p), ("src", C.c_void_p),
        ("n", C.c_int32 * 4), ("ds", C.c_int32 * 4), ("ss", C.c_int32 * 4),
        ("dst_dtype", C.c_int32), ("src_dtype", C.c_int32),
    ]


class FoldChan(C.Structure):
    """Mirror of `yv6_fold_chan` (include/yv6.h)."""
    _fields_ = [("bn", (C.c_int64 * 4) * 3), ("b", C.c_int64), ("coef", C.c_int64), ("layout", C.c_int32), ("n", C.c_int32)]


class FoldRec(C.Structure):
    """Mirror of `yv6_fold_rec` (include/yv6.h)."""
    _fields_ = [
        ("dst", C.c_void_p), ("plane_stride", C.c_int64), ("ds", C.c_int64 * 4), ("w", C.c_int64), ("w1", C.c_int64),
        ("coef", C.c_int64), ("blk0", C.c_int64), ("n", C.c_int32 * 4), ("layout", C.c_int32), ("fmt", C.c_int32),
        ("k", C.c_int32), ("cin", C.c_int32), ("r0", C.c_int32), ("s0", C.c_int32), ("cout", C.c_int32), ("flags", C.c_int32),
        ("check", C.c_int32), ("reserved0", C.c_int32),
    ]


class PrState(C.Structure):
    """Mirror of `yv6_pr_state` (include/yv6.h)."""
    _fields_ = [
        ("max_images", C.c_int32), ("max_det", C.c_int32), ("nc", C.c_int32), ("confusion", C.c_int32),
        ("conf", C.c_void_p), ("cls", C.c_void_p), ("correct", C.c_void_p), ("ndet", C.c_void_p),
        ("nt", C.c_void_p), ("npred", C.c_void_p), ("matrix", C.c_void_p), ("flags", C.c_void_p),
    ]


class CocoState(C.Structure):
    """Mirror of `yv6_coco_state` (include/yv6.h)."""
    _fields_ = [
        ("n_images", C.c_int32), ("n_cats", C.c_int32), ("max_det", C.c_int32), ("max_gts", C.c_int32),
        ("gt_off", C.c_void_p), ("gt_box", C.c_void_p), ("gt_area", C.c_void_p), ("gt_flags", C.c_void_p), ("npig", C.c_void_p),
        ("area_rng", C.c_void_p), ("iou_thrs", C.c_void_p), ("rec_thrs", C.c_void_p),
        ("score", C.c_void_p), ("cat", C.c_void_p), ("rank", C.c_void_p), ("tp", C.c_void_p), ("fp", C.c_void_p),
        ("ndet", C.c_void_p), ("flags", C.c_void_p),
    ]


class DwDesc(C.Structure):
    """Mirror of `yv6_dw_desc` (include/yv6.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("x_c_total", C.c_int32), ("y_c_total", C.c_int32), ("x_plane_stride", C.c_int64), ("y_plane_stride", C.c_int64),
        ("w", C.c_void_p), ("bias", C.c_void_p), ("k", C.c_int32), ("stride", C.c_int32), ("act", C.c_int32), ("nsplit", C.c_int32),
        ("y", C.c_void_p),
    ]


class SeDesc(C.Structure):
    """Mirror of `yv6_se_desc` (include/yv6.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int32), ("HW", C.c_int32), ("C", C.c_int32), ("Cr", C.c_int32),
        ("c_total", C.c_int64), ("plane_stride", C.c_int64),
        ("w1", C.c_void_p), ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p), ("nsplit", C.c_int32),
        ("reserved0", C.c_int32),     # operand dtype: 0 = bf16, DT_F16 = fp16
    ]


class QaDesc(C.Structure):
    """Mirror of `yv6_qa_desc` (include/yv6.h)."""
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("u", C.c_void_p), ("u_pitch", C.c_int64), ("v", C.c_void_p), ("v_pitch", C.c_int64),
        ("scale_d", C.c_void_p), ("shift_d", C.c_void_p), ("x", C.c_void_p), ("x_pitch", C.c_int64),
        ("avg", C.c_int32), ("accumulate", C.c_int32), ("t", C.c_void_p), ("t_pitch", C.c_int64),
        ("sums", C.c_void_p), ("counter", C.c_void_p), ("zeroed", C.c_int32), ("eps", C.c_float),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
        ("stats", C.c_void_p), ("momentum", C.c_float), ("reserved0", C.c_int32),
        ("dt", C.c_void_p), ("dt_pitch", C.c_int64), ("dx", C.c_void_p), ("dx_pitch", C.c_int64),
    ]


class LbSrc(C.Structure):
    """Mirror of `yv6_lb_src` (include/yv6.h): where one image of yv6_letterbox_frames lies and in which layout."""
    _fields_ = [
        ("base", C.c_void_p), ("row_pitch", C.c_int64), ("plane_pitch", C.c_int64), ("layout", C.c_int32), ("reserved0", C.c_int32),
    ]


class JpegHuff(C.Structure):
    """Mirror of `yv6_jpeg_huff` (include/yv6.h): one Huffman table in the decoder's form."""
    _fields_ = [("lut", C.c_uint16 * 512), ("maxcode", C.c_int32 * 18), ("valoff", C.c_int32 * 18), ("vals", C.c_uint8 * 256)]


class JpegComp(C.Structure):
    """Mirror of `yv6_jpeg_comp` (include/yv6.h)."""
    _fields_ = [("h", C.c_int32), ("v", C.c_int32), ("dc", C.c_int32), ("ac", C.c_int32), ("bw", C.c_int32), ("bh", C.c_int32),
                ("dw", C.c_int32), ("dh", C.c_int32), ("plane", C.c_int64), ("q", C.c_uint16 * 64)]


class JpegImage(C.Structure):
    """Mirror of `yv6_jpeg_image` (include/yv6.h): one image of a yv6_jpeg_decode call."""
    _fields_ = [
        ("data", C.c_void_p), ("len", C.c_int64), ("out", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32),
        ("ncomp", C.c_int32), ("orientation", C.c_int32), ("restart", C.c_int32), ("mcux", C.c_int32), ("mcuy", C.c_int32),
        ("nblk", C.c_int32), ("ws_bytes", C.c_int64), ("ws_rst", C.c_int64), ("ws_coef", C.c_int64), ("comp", JpegComp * 3),
    ]


LB_BGR_HWC, LB_RGB_CHW = 0, 1
VAL_COPY, VAL_LINEAR, VAL_AREA, VAL_AREA_FAST = 0, 1, 2, 3      # yv6_letterbox_val's per-image modes (geo[7])
XF_F32, XF_F64, XF_BF16 = 0, 1, 2
XFORM_CHUNK = 4096
FOLD_C_DP, FOLD_C_REP, FOLD_C_QA, FOLD_C_BN, FOLD_C_BIAS = 0, 1, 2, 3, 4
FOLD_W, FOLD_W_REP, FOLD_W_QA, FOLD_W_COPY, FOLD_W_CONVT, FOLD_BIAS, FOLD_COPY = 0, 1, 2, 3, 4, 5, 6
FOLD_F32, FOLD_BF16, FOLD_F16, FOLD_SPLIT3 = 0, 1, 2, 3
FOLD_IDENTITY, FOLD_AVG = 1, 2
FOLD_CHUNK = 4096


_lib = None
_lock = threading.Lock()
_handles = {}

_SIGNATURES = {
    "yv6_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "yv6_destroy": (C.c_int, [C.c_void_p]),
    "yv6_last_error": (C.c_char_p, []),
    "yv6_abi_version": (C.c_int, []),
    "yv6_conv_fwd": (C.c_int, [C.c_void_p, C.POINTER(ConvDesc), C.c_void_p]),
    "yv6_conv_plan": (C.c_int, [C.c_void_p, C.POINTER(ConvDesc), C.POINTER(C.c_int32)]),
    "yv6_conv_plan_host": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(ConvDesc), C.POINTER(C.c_int32)]),
    "yv6_stem_fwd": (C.c_int, [C.c_void_p, C.POINTER(StemDesc), C.c_void_p]),
    "yv6_stem_fwd_f16": (C.c_int, [C.c_void_p, C.POINTER(StemDesc), C.c_void_p]),
    "yv6_sppf_pool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                C.c_int32, C.c_int64, C.c_void_p]),
    "yv6_sppf_pool_f16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int64, C.c_void_p]),
    "yv6_head_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                  C.c_void_p]),
    "yv6_targets_pad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_assign_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "yv6_tal_assign": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "yv6_atss_assign": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "yv6_assign_expand": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "yv6_head_ab_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float),
                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_head_ab_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_ab_boxes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_ab_boxes_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "yv6_kl_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_int32, C.c_double,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_box_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_det_loss_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "yv6_det_loss": (C.c_int, [C.c_void_p, C.POINTER(LossDesc), C.c_void_p]),
    "yv6_conv_wgrad": (C.c_int, [C.c_void_p, C.POINTER(WgradDesc), C.c_void_p]),
    "yv6_wgrad_plan_host": (C.c_int, [C.c_int, C.c_int, C.POINTER(WgradDesc), C.POINTER(C.c_int32)]),
    "yv6_bn_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_bn_finalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_float, C.c_float,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "yv6_bn_apply_fwd": (C.c_int, [C.c_void_p, C.POINTER(BnDesc), C.c_void_p]),
    "yv6_bn_bwd": (C.c_int, [C.c_void_p, C.POINTER(BnDesc), C.c_void_p]),
    "yv6_head_grad_prep": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_maxpool5_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "yv6_stem_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_nms_batched_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.c_float, C.c_double,
                                       C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "yv6_eval_boxes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_letterbox": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_letterbox_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_letterbox_val": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_rescale_boxes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_void_p]),
    "yv6_aug_resize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p]),
    "yv6_aug_resize_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "yv6_augment": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "yv6_bn_stats_finalize": (C.c_int, [C.c_void_p, C.POINTER(BnStatsDesc), C.c_void_p]),
    "yv6_stem_wgrad2": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "yv6_stem_im2col": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_xform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "yv6_sgd_ema_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                   C.c_void_p, C.c_void_p]),
    "yv6_fold": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                           C.c_int32, C.c_void_p]),
    "yv6_pr_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "yv6_pr_match": (C.c_int, [C.c_void_p, C.POINTER(PrState), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                               C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "yv6_pr_metric": (C.c_int, [C.c_void_p, C.POINTER(PrState), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                C.c_void_p]),
    "yv6_coco_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "yv6_coco_update": (C.c_int, [C.c_void_p, C.POINTER(CocoState), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                  C.c_int32, C.c_int32, C.c_void_p]),
    "yv6_coco_load": (C.c_int, [C.c_void_p, C.POINTER(CocoState), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "yv6_coco_accumulate": (C.c_int, [C.c_void_p, C.POINTER(CocoState), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]),
    "yv6_dwconv_fwd": (C.c_int, [C.c_void_p, C.POINTER(DwDesc), C.c_void_p]),
    "yv6_dwconv_fwd_f16": (C.c_int, [C.c_void_p, C.POINTER(DwDesc), C.c_void_p]),
    "yv6_se_fwd": (C.c_int, [C.c_void_p, C.POINTER(SeDesc), C.c_void_p]),
    "yv6_qa_fwd": (C.c_int, [C.c_void_p, C.POINTER(QaDesc), C.c_void_p]),
    "yv6_qa_bwd": (C.c_int, [C.c_void_p, C.POINTER(QaDesc), C.c_void_p]),
    "yv6_channel_shuffle": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                      C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "yv6_upsample2x": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                 C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "yv6_jpeg_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32]),
    "yv6_jpeg_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "yv6_nms_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "yv6_nms_batched": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_double,
                                  C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
}


def exported_symbols():
    """Names every build of the library must export (checked by the CPU test-suite)."""
    return sorted(_SIGNATURES)


def lib():
    """Load the shared library once; raise RuntimeError if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                    "(yolov6_b200 has no CPU/PyTorch fallback for its CUDA path)")
            l = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGNATURES.items():
                try:
                    fn = getattr(l, name)
                except AttributeError as e:
                    raise RuntimeError(f"{LIB_PATH} does not export {name}; rebuild the library") from e
                fn.restype = res
                fn.argtypes = args
            _lib = l
    return _lib


def check(rc):
    if rc != 0:
        raise RuntimeError(f"yolov6_b200 kernel call failed ({rc}): {lib().yv6_last_error().decode()}")


def require_cuda(t, what):
    """RuntimeError unless tensor `t` lives on a CUDA device; `what` names the caller and its verb ("... runs")."""
    if t.device.type != "cuda":
        raise RuntimeError(f"{what} on CUDA tensors only (no CPU fallback)")


def handle(device_index=0):
    """Per-device `yv6_handle*` (created lazily, cached for the life of the process)."""
    h = _handles.get(device_index)
    if h is None:
        p = C.c_void_p()
        check(lib().yv6_create(int(device_index), C.byref(p)))
        h = _handles[device_index] = p
    return h


def stream_ptr(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)
