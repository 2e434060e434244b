"""ctypes binding of libryolo.so (the C-ABI declared in include/ryolo.h).

The library is the product: there is no Python/CPU fallback.  If it has not been built, importing this
module raises with the build instruction; if CUDA is unavailable, every compute entry point returns
RYOLO_E_CUDA and the wrappers raise RuntimeError."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libryolo.so")

RYOLO_OK = 0
IOU_MODE_IOU = 0
IOU_MODE_GIOU = 1
DT_BF16 = 0
DT_F32 = 1
DT_F16 = 2
DT_U8 = 3
MERGE_MAX_SCALES = 16          # RYOLO_MERGE_MAX_SCALES

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "rotate_yolov3_b200: %s is missing. Build it with `python -c \"import __graft_entry__ as g; g.build()\"` "
        "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)

lib = ctypes.CDLL(LIB_PATH)

_vp, _i, _f, _sz, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_double


class ConvDesc(ctypes.Structure):
    """mirror of ryolo_conv_desc (include/ryolo.h)"""
    _fields_ = [("batch", ctypes.c_int32), ("in_h", ctypes.c_int32), ("in_w", ctypes.c_int32),
                ("cin", ctypes.c_int32), ("cin_stride", ctypes.c_int32), ("cout", ctypes.c_int32),
                ("cout_stride", ctypes.c_int32), ("ksize", ctypes.c_int32), ("stride", ctypes.c_int32),
                ("has_act", ctypes.c_int32), ("slope", ctypes.c_float), ("has_residual", ctypes.c_int32),
                ("res_stride", ctypes.c_int32), ("upsample2x", ctypes.c_int32), ("out_dtype", ctypes.c_int32)]


class PackJob(ctypes.Structure):
    """mirror of ryolo_pack_job"""
    _fields_ = [("weight", ctypes.c_void_p), ("packed", ctypes.c_void_p), ("cout", ctypes.c_int32), ("cin", ctypes.c_int32),
                ("ks", ctypes.c_int32), ("cout_pad", ctypes.c_int32), ("cin_pad", ctypes.c_int32), ("mode", ctypes.c_int32)]


class UnpackJob(ctypes.Structure):
    """mirror of ryolo_unpack_job"""
    _fields_ = [("dw", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("cout_pad", ctypes.c_int32), ("cin_pad", ctypes.c_int32),
                ("mode", ctypes.c_int32), ("cout", ctypes.c_int32), ("cin", ctypes.c_int32), ("ks", ctypes.c_int32)]


class HaloJob(ctypes.Structure):
    """mirror of ryolo_halo_job"""
    _fields_ = [("ptr", ctypes.c_void_p), ("batch", ctypes.c_int32), ("h", ctypes.c_int32), ("w", ctypes.c_int32),
                ("c_real", ctypes.c_int32), ("c_stride", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class LetterboxJob(ctypes.Structure):
    """mirror of ryolo_letterbox_job"""
    _fields_ = [("src", ctypes.c_void_p), ("src_stride", ctypes.c_int64), ("src_h", ctypes.c_int32),
                ("src_w", ctypes.c_int32), ("dst_h", ctypes.c_int32), ("dst_w", ctypes.c_int32), ("top", ctypes.c_int32),
                ("left", ctypes.c_int32), ("kind", ctypes.c_int32), ("kx", ctypes.c_int32), ("ky", ctypes.c_int32),
                ("xtab", ctypes.c_int32), ("ytab", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class WarpJob(ctypes.Structure):
    """mirror of ryolo_warp_job"""
    _fields_ = [("src", ctypes.c_void_p), ("dst", ctypes.c_void_p), ("src_stride", ctypes.c_int64),
                ("m", ctypes.c_double * 6), ("warp", ctypes.c_int32), ("image", ctypes.c_int32)]


class FinishJob(ctypes.Structure):
    """mirror of ryolo_finish_job"""
    _fields_ = [("src", ctypes.c_void_p), ("src_stride", ctypes.c_int64), ("gamma", ctypes.c_double),
                ("hsv_s", ctypes.c_float), ("hsv_v", ctypes.c_float), ("flags", ctypes.c_int32),
                ("reserved", ctypes.c_int32)]


class JpegImage(ctypes.Structure):
    """mirror of ryolo_jpeg_image"""
    _fields_ = [("out_off", ctypes.c_int64), ("coef_off", ctypes.c_int64), ("plane_off", ctypes.c_int64 * 3),
                ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("out_w", ctypes.c_int32),
                ("out_h", ctypes.c_int32), ("orient", ctypes.c_int32), ("ncomp", ctypes.c_int32),
                ("color", ctypes.c_int32), ("hmax", ctypes.c_int32), ("vmax", ctypes.c_int32), ("mcux", ctypes.c_int32),
                ("mcuy", ctypes.c_int32), ("bpm", ctypes.c_int32)]
    _fields_ += [(n, ctypes.c_int32 * 3) for n in ("h", "v", "boff", "pitch", "dw", "dh", "qtab", "dctab", "actab")]
    _fields_ += [("reserved", ctypes.c_int32)]


class JpegSegment(ctypes.Structure):
    """mirror of ryolo_jpeg_segment"""
    _fields_ = [("start", ctypes.c_int64), ("end", ctypes.c_int64), ("image", ctypes.c_int32),
                ("first_mcu", ctypes.c_int32), ("nmcu", ctypes.c_int32), ("first_chunk", ctypes.c_int32),
                ("nchunk", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class JpegHuff(ctypes.Structure):
    """mirror of ryolo_jpeg_huff"""
    _fields_ = [("lut", ctypes.c_uint16 * 512), ("maxcode", ctypes.c_int32 * 18), ("valoff", ctypes.c_int32 * 18),
                ("vals", ctypes.c_uint8 * 256)]


# name -> (restype, argtypes); must list every symbol include/ryolo.h declares (tests/test_abi.py checks it)
SIGNATURES = {
    "ryolo_abi_version": (_i, []),
    "ryolo_last_error": (ctypes.c_char_p, []),
    "ryolo_launch_count": (ctypes.c_uint64, []),
    "ryolo_set_reserved_sms": (_i, [_i]),
    "ryolo_rnms_workspace_bytes": (_sz, [_i]),
    "ryolo_rnms": (_i, [_vp, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "ryolo_rnms_full_mask": (_i, [_vp, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "ryolo_rnms_batched_workspace_bytes": (_sz, [_i, _i]),
    "ryolo_rnms_batched": (_i, [_vp, _i, _i, _vp, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "ryolo_detect_select_workspace_bytes": (_sz, [_i, _i]),
    "ryolo_detect_select": (_i, [_vp, _i, _i, _i, _f, _f, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "ryolo_detect_select_classes": (_i, [_vp, _i, _i, _i, _f, _f, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "ryolo_rnms_batched_classes_workspace_bytes": (_sz, [_i, _i]),
    "ryolo_rnms_batched_classes": (_i, [_vp, _i, _i, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    "ryolo_merge_scales": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp), _i, _i, _i, _vp, _vp, _vp]),
    "ryolo_rnms_debug_views": (_i, [_vp, _i, ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp)]),
    "ryolo_riou_paired": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_riou_pairwise": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _vp, _vp]),
    "ryolo_riou_paired_grad": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "ryolo_match_detections": (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _f, _vp, _vp, _vp]),
    "ryolo_match_batched": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp,
                                 ctypes.POINTER(_sz), _vp]),
    "ryolo_ap_per_class": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, ctypes.POINTER(_sz), _vp]),
    "ryolo_nms_filter_workspace_bytes": (_sz, [_i]),
    "ryolo_nms_filter": (_i, [_vp, _i, _i, _f, _f, _vp, _i, _vp, _vp, _sz, _vp]),
    "ryolo_yolo_decode": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _f, _f, _i, _vp, _i, _i, _vp, _vp]),
    "ryolo_conv_packed_weight_bytes": (_sz, [ctypes.POINTER(ConvDesc)]),
    "ryolo_conv_pack_weights_ex": (_i, [ctypes.POINTER(ConvDesc), _vp, _vp, _vp, _i, _vp]),
    "ryolo_conv_unpack_wgrad": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_conv_pack_weights_multi": (_i, [_vp, _i, _vp, ctypes.c_longlong, _vp]),
    "ryolo_zero_halo_multi": (_i, [_vp, _i, _vp]),
    "ryolo_letterbox": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    "ryolo_augment_warp": (_i, [_vp, _i, _vp, _i, _i, _vp]),
    "ryolo_augment_finish": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    "ryolo_jpeg_workspace_bytes": (_sz, [_i, ctypes.c_longlong]),
    "ryolo_jpeg_decode": (_i, [_vp, _i, _vp, _i, _vp, _i, _i, _vp, ctypes.c_longlong, _vp, _vp, _i, _i, _vp, _vp, _vp,
                               _sz, ctypes.c_longlong, _i, _vp]),
    "ryolo_conv_unpack_wgrad_multi": (_i, [_vp, _i, _vp, ctypes.c_longlong, _vp]),
    "ryolo_conv_bn_act_fwd": (_i, [ctypes.POINTER(ConvDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "ryolo_conv_first_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _f, _vp, _i, _vp]),
    "ryolo_conv_first_s2d_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _f, _vp, _i, _vp]),
    "ryolo_head_grad_nchw_to_padded": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp]),
    "ryolo_head_bias_grad": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_loss_rows_gather": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp]),
    "ryolo_loss_rows_scatter_add": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i,
                                         _vp, _vp, _vp]),
    "ryolo_loss_rows_set_tobj": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "ryolo_obj_bce_fwd": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp]),
    "ryolo_obj_bce_bwd": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp, _vp]),
    "ryolo_obj_focal_fwd": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _i, _vp, _f, _f, _vp, _vp]),
    "ryolo_obj_focal_bwd": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), _i, _i, _i, _i, _i, _i, _vp, _f, _f, _vp, _vp, _vp]),
    "ryolo_conv_wgrad": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_bn_stats_finalize": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ryolo_bn_act_fwd": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _f, _i, _vp, _i, _vp, _i, _i, _vp, _vp]),
    "ryolo_bn_act_fwd_s2d": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _f, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _vp]),
    "ryolo_bn_act_bwd": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "ryolo_zero_insert2x": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "ryolo_space_to_depth": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "ryolo_depth_to_space": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "ryolo_dilate_split": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "ryolo_dilate_merge": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _vp]),
    "ryolo_se_block": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "ryolo_se_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "ryolo_se_fwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ryolo_se_bwd": (_i, [_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                          _vp, _sz, _vp]),
    "ryolo_maxpool2x2": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "ryolo_im2col_first": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "ryolo_px_packed_weight_bytes": (_sz, [_i, _i, _i, _i]),
    "ryolo_px_pack_weights": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_px_conv": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "ryolo_px_unpack_wgrad": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_px_wgrad": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_px_bn_stats": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "ryolo_px_bn_finalize": (_i, [_vp, _i, _d, _f, _f, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ryolo_px_bn_act_fwd": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _vp]),
    "ryolo_px_bn_act_bwd": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i,
                                 _vp, _i, _i, _i, _vp]),
    "ryolo_px_im2col_first": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "ryolo_px_to_nchw": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "ryolo_px_head_grad": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "ryolo_px_depth_to_space": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "ryolo_px_split_from_nchw": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
}
for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)
    _fn.restype = _res
    _fn.argtypes = _args


def last_error():
    s = lib.ryolo_last_error()
    return s.decode() if s else ""


def check(status, what):
    if status != RYOLO_OK:
        raise RuntimeError("%s failed (status %d): %s" % (what, status, last_error()))


def stream_ptr(device=None):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())
