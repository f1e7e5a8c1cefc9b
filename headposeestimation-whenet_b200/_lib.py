"""ctypes binding of ``include/whenet_b200.h``.  No CPU fallback: if the shared
library is missing or CUDA is unavailable every call raises."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))

PRECISIONS = {"fp32": 0, "bf16": 1, "fp16": 2}

EXPORTS = [
    "whenet_create", "whenet_load_weights", "whenet_export_packed", "whenet_import_packed", "whenet_set_stream", "whenet_forward_u8", "whenet_forward_u8_async", "whenet_forward_f32",
    "whenet_crop_resize_u8", "whenet_crop_boxes_u8", "whenet_debug_enlarge_boxes", "whenet_synchronize", "whenet_host_alloc", "whenet_host_free", "whenet_debug_enable_taps", "whenet_debug_tap_crops", "whenet_debug_tap",
    "whenet_debug_conv1x1", "whenet_debug_decode", "whenet_debug_raise_timeout", "whenet_debug_set_k1_plan", "whenet_profile_enable", "whenet_profile_read", "whenet_launch_count", "whenet_set_option",
    "whenet_last_error", "whenet_version", "whenet_destroy",
    "whenet_det_create", "whenet_det_load_weights", "whenet_det_num_classes", "whenet_det_set_stream", "whenet_det_detect_u8",
    "whenet_det_synchronize", "whenet_det_destroy", "whenet_det_debug_tap", "whenet_det_debug_conv", "whenet_det_debug_maxpool",
    "whenet_det_debug_decode", "whenet_det_create_ex", "whenet_det_precision", "whenet_det_detect_ragged_u8", "whenet_crop_boxes_ragged_u8",
    "whenet_det_detect_yuv_u8", "whenet_det_detect_ragged_yuv_u8", "whenet_crop_boxes_yuv_u8", "whenet_crop_boxes_ragged_yuv_u8",
    "whenet_det_create_large", "whenet_det_debug_force_large_decode",
    "whenet_draw_heads_u8", "whenet_draw_heads_ragged_u8", "whenet_debug_overlay_segments",
    "whenet_draw_heads_ex_u8", "whenet_draw_heads_ex_ragged_u8", "whenet_put_text_u8", "whenet_put_text_ragged_u8",
    "whenet_debug_text_segments", "whenet_debug_label_text",
    "whenet_encode_jpeg_u8", "whenet_encode_jpeg_ragged_u8", "whenet_debug_jpeg_header",
    "whenet_encode_jpeg_ex_u8", "whenet_debug_jpeg_header_ex", "whenet_debug_jpeg_optimal_table", "whenet_debug_jpeg_optimal_table_gpu",
    "whenet_jpeg_info", "whenet_decode_jpeg_u8", "whenet_debug_jpeg_piece_bits", "whenet_jpeg_info_ex", "whenet_decode_jpeg_ex_u8",
    "whenet_det_detect_yuv422_u8", "whenet_det_detect_ragged_yuv422_u8", "whenet_crop_boxes_yuv422_u8", "whenet_crop_boxes_ragged_yuv422_u8",
    "whenet_yuv_to_bgr_u8", "whenet_yuv_to_bgr_ragged_u8",
]

# pixel_format -> the ABI's yuv_layout (WHENET_YUV_NV12 / WHENET_YUV_I420); "bgr" is packed 8-bit BGR, the *_u8 entries
YUV_LAYOUTS = {"nv12": 1, "i420": 2}
# pixel_format -> the ABI's yuv422_layout (WHENET_YUV_YUYV / WHENET_YUV_UYVY), the *_yuv422_u8 entries
YUV422_LAYOUTS = {"yuyv": 3, "uyvy": 4}


class WhenetError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("whenet_b200 error %d: %s" % (code, msg))
        self.code = code


class JpegOptions(C.Structure):
    """``whenet_jpeg_options``"""
    _fields_ = [("quality", C.c_int), ("chroma_quality", C.c_int), ("sampling", C.c_int), ("restart_interval", C.c_int),
                ("optimize", C.c_int), ("progressive", C.c_int)]


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("ndim", C.c_int32), ("dims", C.c_int64 * 4)]


class KernelStat(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("ms", C.c_float), ("launches", C.c_int), ("bytes", C.c_double),
                ("flops", C.c_double)]


def lib_path() -> str:
    return os.environ.get("WHENET_B200_LIB", os.path.join(HERE, "libwhenet_b200.so"))


_lib = None


def load():
    """dlopen the C-ABI library (building it first if the source is newer and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if "WHENET_B200_LIB" not in os.environ:
        from . import build
        try:
            build.build_lib()
        except FileNotFoundError:
            # no nvcc on this machine: a prebuilt library is acceptable.  A COMPILE or LINK failure is not - loading the
            # stale binary next to edited sources would run old kernels against new host code.
            if not os.path.exists(path):
                raise
    if not os.path.exists(path):
        raise WhenetError(-2, "shared library %s not found; run `python -m whenet_b200.build`" % path)
    L = C.CDLL(path)
    P = C.c_void_p
    L.whenet_create.argtypes = [C.POINTER(P), C.c_int, C.c_int, C.c_int]
    L.whenet_load_weights.argtypes = [P, C.POINTER(Tensor), C.c_int]
    L.whenet_export_packed.argtypes = [P, P, P, P, C.POINTER(C.c_int64)]
    L.whenet_import_packed.argtypes = [P, P, C.c_int64, P, C.c_int64, P, C.c_int64]
    L.whenet_set_stream.argtypes = [P, P]
    L.whenet_forward_u8.argtypes = [P, P, C.c_int, C.c_int, P, P, C.c_int]
    L.whenet_forward_f32.argtypes = [P, P, C.c_int, C.c_int, P, P, C.c_int]
    L.whenet_forward_u8_async.argtypes = [P, P, C.c_int, P, P]
    L.whenet_crop_resize_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, C.c_int, C.c_int, P]
    L.whenet_crop_boxes_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P, P, C.c_int, C.c_int, P, P, P]
    L.whenet_crop_boxes_ragged_u8.argtypes = [P, P, P, C.c_int, C.c_int, P, P, C.c_int, C.c_int, P, P, P]
    L.whenet_crop_boxes_yuv_u8.argtypes = L.whenet_crop_boxes_u8.argtypes
    L.whenet_crop_boxes_ragged_yuv_u8.argtypes = L.whenet_crop_boxes_ragged_u8.argtypes
    L.whenet_crop_boxes_yuv422_u8.argtypes = L.whenet_crop_boxes_u8.argtypes
    L.whenet_crop_boxes_ragged_yuv422_u8.argtypes = L.whenet_crop_boxes_ragged_u8.argtypes
    L.whenet_yuv_to_bgr_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P]
    L.whenet_yuv_to_bgr_ragged_u8.argtypes = [P, P, P, C.c_int, C.c_int, C.c_int, P]
    L.whenet_debug_enlarge_boxes.argtypes = [P, C.c_int, C.c_int, C.c_int, P, P]
    L.whenet_draw_heads_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, P, P, C.c_int, P]
    L.whenet_draw_heads_ragged_u8.argtypes = [P, P, P, C.c_int, P, P, P, C.c_int, P]
    L.whenet_debug_overlay_segments.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, P]
    L.whenet_draw_heads_ex_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, P, P, C.c_int, C.c_int, P]
    L.whenet_draw_heads_ex_ragged_u8.argtypes = [P, P, P, C.c_int, P, P, P, C.c_int, C.c_int, P]
    L.whenet_put_text_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, C.c_int]
    L.whenet_put_text_ragged_u8.argtypes = [P, P, P, C.c_int, P, P, P, P, P, P, C.c_int]
    L.whenet_debug_text_segments.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_double, C.c_int, P, C.c_int, P]
    L.whenet_debug_label_text.argtypes = [P, C.c_int, P, C.c_int]
    L.whenet_encode_jpeg_u8.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(P), P]
    L.whenet_encode_jpeg_ragged_u8.argtypes = [P, P, P, C.c_int, C.c_int, C.c_int, C.POINTER(P), P]
    L.whenet_debug_jpeg_header.argtypes = [C.c_int, C.c_int, C.c_int, P, C.c_int, P]
    L.whenet_encode_jpeg_ex_u8.argtypes = [P, P, P, C.c_int, C.c_int, C.c_int, P, C.POINTER(P), P]
    L.whenet_debug_jpeg_header_ex.argtypes = [C.c_int, C.c_int, C.c_int, P, P, C.c_int, P]
    L.whenet_debug_jpeg_optimal_table.argtypes = [P, P, P, P]
    L.whenet_debug_jpeg_optimal_table_gpu.argtypes = [P, P, P, P, P]
    L.whenet_jpeg_info.argtypes = [P, C.c_int64, P, C.c_char_p, C.c_int]
    L.whenet_decode_jpeg_u8.argtypes = [P, P, P, C.c_int, P, P]
    L.whenet_debug_jpeg_piece_bits.argtypes = [P, C.c_int]
    L.whenet_jpeg_info_ex.argtypes = [P, C.c_int64, C.c_int, C.c_int, P, C.c_char_p, C.c_int]
    L.whenet_decode_jpeg_ex_u8.argtypes = [P, P, P, C.c_int, C.c_int, C.c_int, P, P]
    L.whenet_synchronize.argtypes = [P]
    L.whenet_host_alloc.argtypes = [C.c_size_t]
    L.whenet_host_alloc.restype = P
    L.whenet_host_free.argtypes = [P]
    L.whenet_host_free.restype = None
    L.whenet_debug_enable_taps.argtypes = [P, C.c_int]
    L.whenet_debug_tap.argtypes = [P, C.c_char_p, P, C.c_size_t, C.POINTER(C.c_size_t)]
    L.whenet_debug_tap_crops.argtypes = [P, P, C.c_int]
    L.whenet_debug_conv1x1.argtypes = [P, C.c_int, P, P, P, P, P, P, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]
    L.whenet_debug_decode.argtypes = [P, P, C.c_int, P]
    L.whenet_debug_raise_timeout.argtypes = [P]
    L.whenet_debug_set_k1_plan.argtypes = [P] + [C.c_int] * 7
    L.whenet_profile_enable.argtypes = [P, C.c_int]
    L.whenet_profile_read.argtypes = [P, C.POINTER(KernelStat), C.c_int]
    L.whenet_launch_count.argtypes = [P]
    L.whenet_launch_count.restype = C.c_int64
    L.whenet_set_option.argtypes = [P, C.c_char_p, C.c_int]
    L.whenet_last_error.restype = C.c_char_p
    L.whenet_version.restype = C.c_char_p
    L.whenet_destroy.argtypes = [P]
    L.whenet_destroy.restype = None
    I = C.c_int
    L.whenet_det_create.argtypes = [C.POINTER(P), I, I, I, I]
    L.whenet_det_create_ex.argtypes = [C.POINTER(P), I, I, I, I, I]
    L.whenet_det_create_large.argtypes = [C.POINTER(P), I, I, I, I, I]
    L.whenet_det_debug_force_large_decode.argtypes = [P, I]
    L.whenet_det_precision.argtypes = [P]
    L.whenet_det_load_weights.argtypes = [P, C.POINTER(Tensor), I, P, I]
    L.whenet_det_num_classes.argtypes = [P]
    L.whenet_det_set_stream.argtypes = [P, P]
    L.whenet_det_detect_u8.argtypes = [P, P, I, I, I, I, I, C.c_float, C.c_float, I, P, P, P, P]
    L.whenet_det_detect_ragged_u8.argtypes = [P, P, P, I, I, I, C.c_float, C.c_float, I, P, P, P, P]
    L.whenet_det_detect_yuv_u8.argtypes = L.whenet_det_detect_u8.argtypes
    L.whenet_det_detect_ragged_yuv_u8.argtypes = L.whenet_det_detect_ragged_u8.argtypes
    L.whenet_det_detect_yuv422_u8.argtypes = L.whenet_det_detect_u8.argtypes
    L.whenet_det_detect_ragged_yuv422_u8.argtypes = L.whenet_det_detect_ragged_u8.argtypes
    L.whenet_det_synchronize.argtypes = [P]
    L.whenet_det_destroy.argtypes = [P]
    L.whenet_det_destroy.restype = None
    L.whenet_det_debug_tap.argtypes = [P, I, P, C.c_size_t, C.POINTER(C.c_size_t)]
    L.whenet_det_debug_conv.argtypes = [P, P, P, I, I, I, I, I, P, P, I, I, I, I, P, P]
    L.whenet_det_debug_maxpool.argtypes = [P, P, I, I, I, I, I, P]
    L.whenet_det_debug_decode.argtypes = [P, P, P, P, I, I, I, C.c_float, C.c_float, I, P, P, P, P]
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise WhenetError(rc, load().whenet_last_error().decode("utf-8", "replace"))
