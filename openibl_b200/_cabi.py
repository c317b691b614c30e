"""ctypes binding of libiblb200.so (include/iblb200.h).

The library is the product: if it cannot be loaded, or there is no sm_90 GPU, every
operation raises -- there is no PyTorch / CPU fallback behind these calls."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libiblb200.so")

IBL_OK = 0
STATUS_NAMES = {0: "IBL_OK", 1: "IBL_ERR_BAD_ARG", 2: "IBL_ERR_NOT_READY", 3: "IBL_ERR_CUDA",
                4: "IBL_ERR_NO_DEVICE", 5: "IBL_ERR_OOM", 6: "IBL_ERR_UNSUPPORTED"}
OUT_VLAD, OUT_PCA, OUT_POOL = 0x1, 0x2, 0x4
CONV_SIMT_FP32, CONV_TC_BF16X3 = 0, 1
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"

_P = c_void_p


class JpegInfo(Structure):
    """ibl_jpeg_info (include/iblb200.h)."""
    _fields_ = [("width", c_int), ("height", c_int), ("components", c_int), ("h_samp", c_int), ("v_samp", c_int),
                ("restart_interval", c_int), ("intervals", c_int), ("mcus", c_int), ("entropy_bytes", c_uint64),
                ("reason", c_char * 120)]


class JpegScan(Structure):
    """ibl_jpeg_scan (include/iblb200.h)."""
    _fields_ = [("components", c_int), ("comp", c_int * 3), ("ss", c_int), ("se", c_int), ("ah", c_int), ("al", c_int),
                ("restart_interval", c_int), ("intervals", c_int)]


class PngInfo(Structure):
    """ibl_png_info (include/iblb200.h)."""
    _fields_ = [("width", c_int), ("height", c_int), ("color_type", c_int), ("bit_depth", c_int),
                ("palette_size", c_int), ("zlib_bytes", c_uint64), ("reason", c_char * 120)]


class ColorJitterParams(Structure):
    """ibl_color_jitter_params (include/iblb200.h)."""
    _fields_ = [("order", c_int * 4), ("brightness", c_float), ("contrast", c_float), ("saturation", c_float),
                ("hue", c_float)]


# name -> (restype, argtypes); mirrors include/iblb200.h one to one
SIGNATURES = {
    "ibl_abi_version": (c_int, []),
    "ibl_status_string": (c_char_p, [c_int]),
    "ibl_last_error": (c_char_p, []),
    "ibl_engine_create": (c_int, [c_int, POINTER(c_void_p)]),
    "ibl_engine_destroy": (c_int, [_P]),
    "ibl_engine_set_conv_mode": (c_int, [_P, c_int]),
    "ibl_engine_set_gemm_mode": (c_int, [_P, c_int]),
    "ibl_engine_get_conv_mode": (c_int, [_P, POINTER(c_int)]),
    "ibl_engine_launch_count": (c_int, [_P, POINTER(c_uint64)]),
    "ibl_engine_set_vgg16": (c_int, [_P, POINTER(c_void_p), POINTER(c_void_p), _P]),
    "ibl_engine_set_netvlad": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "ibl_engine_set_pca": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "ibl_vgg16_forward": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P, _P]),
    "ibl_vgg16_prefix_forward": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "ibl_vgg16_layer_forward": (c_int, [_P, c_int, _P, c_int, c_int, c_int, _P, _P]),
    "ibl_maxpool2x2_forward": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "ibl_maxpool2x2_backward": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "ibl_vgg16_layer_backward": (c_int, [_P, c_int, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P]),
    "ibl_netvlad_forward": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, _P, _P]),
    "ibl_netvlad_backward": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, _P, _P, _P, _P]),
    "ibl_vlad_normalize": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "ibl_pca_l2": (c_int, [_P, _P, c_int, c_int, _P, _P, c_int, _P, _P]),
    "ibl_pca_forward_train": (c_int, [_P, _P, c_int, c_int, _P, _P, c_int, _P, _P]),
    "ibl_pca_backward": (c_int, [_P, _P, c_int, c_int, _P, c_int, _P, _P, _P, _P, _P]),
    "ibl_l2_normalize_rows": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "ibl_extract": (c_int, [_P, _P, c_int, c_int, c_int, c_uint, _P, _P, _P]),
    "ibl_extract_host": (c_int, [_P, _P, c_int, c_int, c_int, c_uint, _P, _P, _P]),
    "ibl_extract_host_submit": (c_int, [_P, c_int, _P, c_int, c_int, c_int, c_uint, _P, _P, _P]),
    "ibl_extract_host_wait": (c_int, [_P, c_int]),
    "ibl_preprocess_u8": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P, _P]),
    "ibl_resize_bilinear_u8": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, c_int, _P, _P]),
    "ibl_extract_host_u8": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_uint, _P, _P, _P]),
    "ibl_jpeg_parse": (c_int, [c_char_p, c_size_t, POINTER(JpegInfo)]),
    "ibl_jpeg_decode_u8": (c_int, [_P, _P, _P, c_int, _P, _P, _P, _P, _P]),
    "ibl_jpeg_parse_progressive": (c_int, [c_char_p, c_size_t, POINTER(JpegInfo), POINTER(c_int), POINTER(JpegScan),
                                           c_int]),
    "ibl_jpeg_decode_progressive_u8": (c_int, [_P, _P, _P, c_int, _P, _P, _P, _P, _P]),
    "ibl_png_parse": (c_int, [c_char_p, c_size_t, POINTER(PngInfo)]),
    "ibl_png_decode_u8": (c_int, [_P, _P, _P, c_int, _P, _P, _P, _P, _P]),
    "ibl_color_jitter_u8": (c_int, [_P, _P, _P, _P, _P, POINTER(ColorJitterParams), c_int, _P]),
    "ibl_l2dist_dense": (c_int, [_P, _P, c_int, _P, c_int, c_int, _P, _P]),
    "ibl_l2dist_self": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "ibl_l2dist_topk": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int64, _P, _P, _P]),
    "ibl_db_prepare": (c_int, [_P, _P, c_int, c_int, _P, _P, _P, _P]),
    "ibl_db_topk": (c_int, [_P, _P, c_int, _P, _P, _P, _P, c_int, c_int, c_int, c_int64, _P, _P, _P]),
    "ibl_topk_rows": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "ibl_argsort_rows": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "ibl_topk_merge": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "ibl_l2dist_topk_host": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, _P, _P, _P]),
    "ibl_knn_rowmax": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P]),
    "ibl_rerank_topk": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, c_float, _P, c_int,
                                c_int, _P, _P, _P]),
    "ibl_rerank_dense": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_double, _P, _P]),
    "ibl_debug_rerank_workspace_bytes": (c_int, [_P, POINTER(c_uint64)]),
    "ibl_debug_knn_flagged": (c_int, [_P, POINTER(c_int), _P]),
    "ibl_gemm_nt": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_float, _P, c_int, _P]),
    "ibl_debug_dist_flagged": (c_int, [_P, POINTER(c_int), _P]),
    "ibl_debug_dist_path": (c_int, [_P, POINTER(c_int)]),
    "ibl_selftest_tc": (c_int, [_P, POINTER(c_float)]),
    "ibl_debug_gemm_tn": (c_int, [_P, _P, _P, _P, _P]),
    "ibl_debug_umma_strided": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, _P, _P]),
    "ibl_debug_umma_halo_view": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, _P, _P]),
    "ibl_debug_wgmma_rs_halo_view": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "ibl_debug_set_conv3x3_variant": (c_int, [_P, c_int]),
    "ibl_debug_conv1_fused": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "ibl_debug_time_layer": (c_int, [_P, c_int, _P, c_int, c_int, c_int, c_int, c_int, POINTER(c_float)]),
    "ibl_debug_conv3x3": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, c_int, c_int,
                                  c_int, _P, _P]),
}

_lib = None


class IblError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str):
        self.status = status
        super().__init__(f"{where}: {STATUS_NAMES.get(status, status)}: {detail}")


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """Load (building in-tree with nvcc if absent) and type every exported symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise ImportError(f"{LIB_PATH} is missing; run `python -m openibl_b200.build`")
        from . import build as _build
        _build.build()
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def jpeg_parse(data: bytes) -> dict:
    """ibl_jpeg_parse on one in-memory file; runs on the host, no device needed."""
    lib = load()
    info = JpegInfo()
    data = bytes(data)
    st = lib.ibl_jpeg_parse(data, len(data), ctypes.byref(info))
    return {"ok": st == IBL_OK, "status": st, "width": info.width, "height": info.height,
            "components": info.components, "h_samp": info.h_samp, "v_samp": info.v_samp,
            "restart_interval": info.restart_interval, "intervals": info.intervals, "mcus": info.mcus,
            "entropy_bytes": info.entropy_bytes, "reason": info.reason.decode()}


def jpeg_parse_progressive(data: bytes) -> dict:
    """ibl_jpeg_parse_progressive on one in-memory file (host only): jpeg_parse's fields plus `scans`, the scan
    script as a list of dicts (components, ss, se, ah, al, restart_interval, intervals)."""
    lib = load()
    info = JpegInfo()
    data = bytes(data)
    n = c_int(0)
    st = lib.ibl_jpeg_parse_progressive(data, len(data), ctypes.byref(info), ctypes.byref(n), None, 0)
    scans = (JpegScan * max(n.value, 1))()
    if n.value:
        lib.ibl_jpeg_parse_progressive(data, len(data), ctypes.byref(info), ctypes.byref(n), scans, n.value)
    return {"ok": st == IBL_OK, "status": st, "width": info.width, "height": info.height,
            "components": info.components, "h_samp": info.h_samp, "v_samp": info.v_samp,
            "restart_interval": info.restart_interval, "intervals": info.intervals, "mcus": info.mcus,
            "entropy_bytes": info.entropy_bytes, "reason": info.reason.decode(),
            "scans": [{"components": tuple(s.comp[:s.components]), "ss": s.ss, "se": s.se, "ah": s.ah, "al": s.al,
                       "restart_interval": s.restart_interval, "intervals": s.intervals}
                      for s in scans[:n.value]]}


def png_parse(data: bytes) -> dict:
    """ibl_png_parse on one in-memory file; runs on the host, no device needed."""
    lib = load()
    info = PngInfo()
    data = bytes(data)
    st = lib.ibl_png_parse(data, len(data), ctypes.byref(info))
    return {"ok": st == IBL_OK, "status": st, "width": info.width, "height": info.height,
            "color_type": info.color_type, "bit_depth": info.bit_depth, "palette_size": info.palette_size,
            "zlib_bytes": info.zlib_bytes, "reason": info.reason.decode()}


def check(status: int, where: str) -> None:
    if status != IBL_OK:
        lib = load()
        detail = lib.ibl_last_error().decode() or lib.ibl_status_string(status).decode()
        raise IblError(status, where, detail)
