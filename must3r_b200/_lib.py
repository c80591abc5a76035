"""ctypes binding of libm3r_b200.so (the C ABI declared in include/must3r_b200.h).

There is no CPU fallback: if the library is missing or no CUDA device is present, the ops raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libm3r_b200.so")
_lib = None


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("W", C.c_void_p), ("ldw", C.c_int64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("is_bf16", C.c_int32),
        ("bias", C.c_void_p),
        ("act", C.c_int32),
        ("residual", C.c_void_p), ("ldr", C.c_int64),
        ("rowbias", C.c_void_p), ("rb_period", C.c_int32), ("rb_first", C.c_int32),
        ("rope_tab", C.c_void_p), ("rope_cols", C.c_int32), ("rope_period", C.c_int32),
        ("out", C.c_void_p), ("ldc", C.c_int64),
        ("out_dtype", C.c_int32),
        ("rows_per_batch", C.c_int32),
        ("batch_stride_rows", C.c_int64),
        ("n_peer_out", C.c_int32),
        ("peer_out", C.c_void_p * 8),
        ("w_static", C.c_int32),
        ("norm_out", C.c_void_p), ("ldn", C.c_int64), ("norm_eps", C.c_float),
    ]


class GemmE4M3Args(C.Structure):
    _fields_ = [("a_e4m3", C.c_int32), ("w_scale", C.c_void_p), ("norm_e4m3", C.c_int32)]


class GemmGroup(C.Structure):
    _fields_ = [("groups", C.c_int32), ("w_group_rows", C.c_int64), ("bias_group", C.c_int64),
                ("out", C.c_void_p * 16), ("peer_out", C.c_void_p * (16 * 8)), ("max_ctas", C.c_int32)]


class AttnArgs(C.Structure):
    _fields_ = [
        ("Q", C.c_void_p), ("ldq", C.c_int64),
        ("K0", C.c_void_p), ("V0", C.c_void_p), ("ldk0", C.c_int64), ("kv_bstride0", C.c_int64), ("Nk0", C.c_int32),
        ("K1", C.c_void_p), ("V1", C.c_void_p), ("ldk1", C.c_int64), ("kv_bstride1", C.c_int64), ("Nk1", C.c_int32),
        ("O", C.c_void_p), ("ldo", C.c_int64),
        ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32),
        ("kv_group", C.c_int32),
        ("skip_lo", C.c_int32), ("skip_step", C.c_int32), ("skip_len", C.c_int32),
        ("is_bf16", C.c_int32),
        ("scale", C.c_float),
        ("export_o", C.c_void_p), ("export_ml", C.c_void_p),
    ]


class JpegInfo(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("ncomp", C.c_int32), ("eligible", C.c_int32),
                ("orientation", C.c_int32), ("orientation_exact", C.c_int32), ("restart_interval", C.c_int32),
                ("hs", C.c_int32 * 3), ("vs", C.c_int32 * 3), ("scan_offset", C.c_int64), ("prep_bytes", C.c_int64)]


class JpegDesc(C.Structure):
    _fields_ = [("tables_off", C.c_int64), ("segs_off", C.c_int64), ("subs_off", C.c_int64), ("stream_off", C.c_int64),
                ("stream_bytes", C.c_int64), ("out", C.c_void_p),
                ("width", C.c_int32), ("height", C.c_int32), ("ncomp", C.c_int32), ("orientation", C.c_int32),
                ("mcux", C.c_int32), ("mcuy", C.c_int32), ("bpm", C.c_int32), ("restart_interval", C.c_int32),
                ("nseg", C.c_int32), ("nsub", C.c_int32), ("hs", C.c_int32 * 3), ("vs", C.c_int32 * 3),
                ("sub_base", C.c_int64), ("blk_base", C.c_int64), ("pix_base", C.c_int64), ("coef_off", C.c_int64),
                ("plane_off", C.c_int64 * 3)]


class PngInfo(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("bit_depth", C.c_int32), ("color_type", C.c_int32),
                ("interlace", C.c_int32), ("channels", C.c_int32), ("palette_entries", C.c_int32), ("eligible", C.c_int32),
                ("has_exif", C.c_int32), ("has_text", C.c_int32), ("text_bytes", C.c_int64), ("idat_bytes", C.c_int64),
                ("prep_bytes", C.c_int64)]


class PngDesc(C.Structure):
    _fields_ = [("plte_off", C.c_int64), ("stream_off", C.c_int64), ("stream_bytes", C.c_int64), ("out", C.c_void_p),
                ("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("color_type", C.c_int32),
                ("palette_entries", C.c_int32), ("orientation", C.c_int32), ("raw_off", C.c_int64), ("raw_bytes", C.c_int64)]


# name -> (restype, argtypes); must list every symbol include/must3r_b200.h declares
SIGNATURES = {
    "m3r_last_error": (C.c_char_p, []),
    "m3r_abi_version": (C.c_int, []),
    "m3r_debug_trace": (C.c_int, [C.c_void_p]),
    "m3r_launch_count": (C.c_longlong, []),
    "m3r_prof_enable": (None, [C.c_int]),
    "m3r_prof_read": (C.c_int, [C.POINTER(C.c_double)]),
    "m3r_gemm": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p]),
    "m3r_gemm_grouped": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(GemmGroup), C.c_void_p]),
    "m3r_gemm_e4m3": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(GemmE4M3Args), C.c_void_p]),
    "m3r_gemm_grouped_e4m3": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(GemmGroup), C.POINTER(GemmE4M3Args), C.c_void_p]),
    "m3r_normalize16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "m3r_normalize8": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_layernorm": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float,
                                C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    "m3r_cast16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "m3r_layernorm16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_int64, C.c_int32, C.c_void_p]),
    "m3r_add_cast16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                 C.c_int32, C.c_void_p]),
    "m3r_rope_table": (C.c_int, [C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "m3r_rope_2d": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                              C.c_int64, C.c_void_p, C.c_float, C.c_float, C.c_void_p]),
    "m3r_attention": (C.c_int, [C.POINTER(AttnArgs), C.c_void_p]),
    "m3r_attention_ragged": (C.c_int, [C.POINTER(AttnArgs), C.c_void_p, C.c_void_p]),
    "m3r_mem_commit": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.POINTER(C.c_int64), C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_mem_commit_rows": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_mem_commit_ordered": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_mem_compact_rows": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_int64,
                                       C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p]),
    "m3r_attn_merge": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                 C.c_int32, C.c_void_p]),
    "m3r_attn_state_fill": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "m3r_im2col16": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "m3r_unpatchify": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "m3r_postprocess": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "m3r_nn_min_dist": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "m3r_pointgrid_keys": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]),
    "m3r_pointgrid_query": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                      C.c_int32, C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "m3r_slam_pose": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_void_p]),
    "m3r_slam_keyframe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                    C.c_double, C.c_float, C.c_int32, C.c_void_p, C.c_void_p]),
    "m3r_slam_pose_views": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                      C.c_float, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_void_p,
                                      C.c_void_p]),
    "m3r_slam_keyframe_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_int32, C.c_double, C.c_double, C.c_float, C.POINTER(C.c_int32), C.c_void_p,
                                           C.c_void_p]),
    "m3r_scene_count": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "m3r_scene_points": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "m3r_resample_pil_u8": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p, C.c_void_p]),
    "m3r_resize_aa_bilinear_u8": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                            C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "m3r_jpeg_parse": (C.c_int, [C.c_char_p, C.c_int64, C.POINTER(JpegInfo)]),
    "m3r_jpeg_prepare": (C.c_int, [C.c_char_p, C.c_int64, C.POINTER(JpegInfo), C.c_int32, C.c_void_p, C.c_int64,
                                   C.POINTER(JpegDesc)]),
    "m3r_jpeg_plan": (C.c_int64, [C.POINTER(JpegDesc), C.c_int32]),
    "m3r_jpeg_decode": (C.c_int, [C.POINTER(JpegDesc), C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                  C.c_void_p]),
    "m3r_png_parse": (C.c_int, [C.c_char_p, C.c_int64, C.POINTER(PngInfo)]),
    "m3r_png_prepare": (C.c_int, [C.c_char_p, C.c_int64, C.POINTER(PngInfo), C.c_int32, C.c_void_p, C.c_int64,
                                  C.POINTER(PngDesc)]),
    "m3r_png_plan": (C.c_int64, [C.POINTER(PngDesc), C.c_int32]),
    "m3r_png_decode": (C.c_int, [C.POINTER(PngDesc), C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.c_void_p]),
    "m3r_peer_alloc": (C.c_int, [C.c_int64, C.POINTER(C.c_void_p)]),
    "m3r_peer_free": (C.c_int, [C.c_void_p]),
    "m3r_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "m3r_ipc_open": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "m3r_ipc_close": (C.c_int, [C.c_void_p]),
    "m3r_peer_bcast": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_int64, C.c_void_p]),
    "m3r_peer_signal": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_uint32, C.c_void_p]),
    "m3r_peer_wait": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
}


def lib():
    """Load the shared library once; raise (never fall back) if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} not found: build it with `python -m must3r_b200.build` "
                               "(must3r_b200 has no CPU / PyTorch fallback)")
        _lib = C.CDLL(LIB_PATH)
        apply_signatures()
    return _lib


def apply_signatures():
    """(Re)apply SIGNATURES to the loaded library (model/common.py registers the whole-model entry points)."""
    if _lib is None:
        return
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(_lib, name)
        fn.restype = res
        fn.argtypes = args


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().m3r_last_error()
        raise RuntimeError(f"must3r_b200 {what} failed: {msg.decode() if msg else rc}")
