"""ctypes binding of libfast3r_b200.so (include/fast3r_b200.h).

There is NO fallback: if the library is missing or a call fails this raises (the reference's own native
precedent, curope, surfaces TORCH_CHECK failures as RuntimeError the same way —
fast3r/croco/models/curope/curope.cpp:54-59).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfast3r_b200.so")

EPI_STORE, EPI_ROPE, EPI_IDXEMB, EPI_CONVT, EPI_FINAL = range(5)
ACT_NONE, ACT_RELU, ACT_GELU = range(3)
# element-type codes of f3r_layernorm / f3r_im2col_patch / f3r_upsample2x
ELT_BF16, ELT_F32, ELT_F16 = range(3)


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("wt", C.c_void_p),
        ("n", C.c_int32), ("k", C.c_int32), ("taps", C.c_int32),
        ("w", C.c_int32), ("h", C.c_int32), ("nb", C.c_int32),
        ("a_ld", C.c_int32),
        ("epi", C.c_int32), ("act", C.c_int32),
        ("out0_f32", C.c_int32), ("res0_f32", C.c_int32),
        ("ldo", C.c_int32),
        ("split_col", C.c_int32), ("ldo_b", C.c_int32),
        ("tok_per_img", C.c_int32), ("grid_w", C.c_int32), ("rope_cols", C.c_int32),
        ("ct_k", C.c_int32), ("ct_cout", C.c_int32),
        ("f16", C.c_int32),
        ("bias", C.c_void_p), ("res0", C.c_void_p), ("res1", C.c_void_p),
        ("out0", C.c_void_p), ("out0b", C.c_void_p), ("out1", C.c_void_p),
        ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p),
        ("emb_table", C.c_void_p), ("emb_ids", C.c_void_p),
        ("w4", C.c_void_p), ("b4", C.c_void_p), ("pts", C.c_void_p), ("conf", C.c_void_p),
    ]


ABI_VERSION = 3


JPEG_SUPPORTED, JPEG_UNSUPPORTED, JPEG_MALFORMED = range(3)


# one row of the hypothesis table of f3r_pnp_score / f3r_pnp_inliers (f3r_pnp_hyp), as a numpy record
PNP_HYP = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,)), ("fx", "<f8"), ("fy", "<f8"), ("cx", "<f8"), ("cy", "<f8"),
                    ("view", "<i4"), ("reserved", "<i4")])


# f3r_pose_metric's counts row: [0..2] rotation angle < 5 / 15 / 30, [3..5] translation angle < 5 / 15 / 30, [6] bad
# traces, [7] pairs, [PM_HIST + b] histogram bin b
PM_HIST, PM_MAX_BINS = 8, 64
PM_COUNTS = PM_HIST + PM_MAX_BINS


# f3r_view_param of f3r_view_geometry (one (view, item) of fast3r_b200.views), as a numpy record
VIEW_PARAM = np.dtype([("depth", "<u8"), ("out_offset", "<i8"), ("src_w", "<i4"), ("src_h", "<i4"), ("crop_x", "<i4"),
                       ("crop_y", "<i4"), ("crop_w", "<i4"), ("crop_h", "<i4"), ("rs_w", "<i4"), ("rs_h", "<i4"),
                       ("box_x", "<i4"), ("box_y", "<i4"), ("out_w", "<i4"), ("out_h", "<i4"), ("transpose", "<i4"),
                       ("reserved", "<i4"), ("k", "<f4", (4,)), ("pose", "<f4", (12,))])


class JpegInfo(C.Structure):
    _fields_ = [("status", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("components", C.c_int32),
                ("h_samp", C.c_int32), ("v_samp", C.c_int32), ("restart_interval", C.c_int32), ("segments", C.c_int32),
                ("scan_offset", C.c_size_t), ("scan_bytes", C.c_size_t), ("workspace_bytes", C.c_size_t)]


# name -> (restype, argtypes), one entry per prototype of include/fast3r_b200.h, in header order.  ctypes does not check
# these against the C side: tests/test_cabi_bindings_cpu.py compares every entry with the header.  Device pointers and
# the cudaStream_t are void*.
_P, _I32, _F32, _SIZE = C.c_void_p, C.c_int32, C.c_float, C.c_size_t
_API = {
    "f3r_last_error": (C.c_char_p, []),
    "f3r_abi_version": (C.c_int, []),
    "f3r_gemm_desc_size": (_SIZE, []),
    "f3r_launch_count": (C.c_uint64, []),
    "f3r_set_option": (C.c_int, [C.c_char_p, _I32]),
    "f3r_gemm": (C.c_int, [C.POINTER(GemmDesc), _P]),
    "f3r_attention": (C.c_int, [_P, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _F32, _P]),
    "f3r_attention_partial": (C.c_int, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _I32, _I32, _I32, _I32,
                                        _F32, _P]),
    "f3r_attention_segments": (C.c_int, [_P, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _F32, _I32, _P, _P, _P]),
    "f3r_attention_merge": (C.c_int, [_P, _P, _I32, _P, _I32, _I32, _I32, _I32, _P]),
    "f3r_attention_f16": (C.c_int, [_P, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _F32, _P]),
    "f3r_attention_partial_f16": (C.c_int, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _I32, _I32, _I32, _I32,
                                            _F32, _P]),
    "f3r_attention_segments_f16": (C.c_int, [_P, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _I32, _F32, _I32, _P, _P,
                                             _P]),
    "f3r_attention_merge_f16": (C.c_int, [_P, _P, _I32, _P, _I32, _I32, _I32, _I32, _P]),
    "f3r_layernorm": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _I32, _F32, _P]),
    "f3r_im2col_patch": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _P]),
    "f3r_im2col3x3s2": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "f3r_upsample2x": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "f3r_cast_bf16": (C.c_int, [_P, _P, _SIZE, _P]),
    "f3r_cast_f16": (C.c_int, [_P, _P, _SIZE, _P]),
    "f3r_resample_ksize": (C.c_int, [_I32, _I32, _I32]),
    "f3r_resample_coeffs": (C.c_int, [_I32, _I32, _I32, _P, _P]),
    "f3r_ingest_rgb8": (C.c_int, [_P, _I32, _I32, _I32, _I32, _P, _P, _I32, _I32, _P, _P, _I32, _P, _I32, _I32, _I32,
                                  _I32, _P, _P]),
    "f3r_jpeg_probe": (C.c_int, [_P, _SIZE, C.POINTER(JpegInfo)]),
    "f3r_jpeg_decode": (C.c_int, [_P, _SIZE, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _SIZE, _P]),
    "f3r_conf_quantile": (C.c_int, [_P, _I32, _I32, _F32, _P, _P]),
    "f3r_similarity_fit_workspace": (_SIZE, [_I32]),
    "f3r_similarity_fit": (C.c_int, [_P, _P, _P, _P, _P, _I32, _I32, _P, _P, _SIZE, _P]),
    "f3r_similarity_apply": (C.c_int, [_P, _P, _P, _I32, _I32, _P]),
    "f3r_focal_workspace": (_SIZE, [_I32]),
    "f3r_focal_weiszfeld": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _SIZE, _P]),
    "f3r_split3": (C.c_int, [_P, _P, _SIZE, _I32, _I32, _P]),
    "f3r_add_f32": (C.c_int, [_P, _P, _SIZE, _P]),
    "f3r_attention_x3_workspace": (_SIZE, [_I32, _I32, _I32, _I32]),
    "f3r_attention_x3": (C.c_int, [_P, _I32, _P, _I32, _P, _I32, _P, _P, _SIZE, _I32, _I32, _I32, _I32, _F32, _P]),
    "f3r_pc_index_workspace": (_SIZE, [_I32]),
    "f3r_pc_index_build": (C.c_int, [_P, _I32, _I32, _P, _SIZE, _P]),
    "f3r_pc_query_workspace": (_SIZE, [_I32]),
    "f3r_pc_nearest": (C.c_int, [_P, _SIZE, _I32, _P, _I32, _I32, _P, _P, _P, _SIZE, _P]),
    "f3r_pc_knn_normals": (C.c_int, [_P, _SIZE, _I32, _I32, _P, _P]),
    "f3r_pc_count_nonfinite": (C.c_int, [_P, _I32, _I32, _P, _P]),
    "f3r_pc_abs_dot": (C.c_int, [_P, _P, _P, _P, _I32, _P, _P]),
    "f3r_f64_reduce_workspace": (_SIZE, []),
    "f3r_f64_mean": (C.c_int, [_P, _I32, _P, _P, _SIZE, _P]),
    "f3r_f64_median": (C.c_int, [_P, _I32, _P, _P, _SIZE, _P]),
    "f3r_f64_count_below": (C.c_int, [_P, _I32, _P, _P, _P]),
    "f3r_pnp_gather_workspace": (_SIZE, [_I32, _I32, _I32]),
    "f3r_pnp_gather": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _P, _P, _P, _P, _SIZE, _P]),
    "f3r_pnp_score_workspace": (_SIZE, [_I32, _I32]),
    "f3r_pnp_score": (C.c_int, [_P, _P, _P, _P, _I32, _P, _I32, _F32, _P, _P, _SIZE, _P]),
    "f3r_pnp_inliers_workspace": (_SIZE, [_I32, _I32]),
    "f3r_pnp_inliers": (C.c_int, [_P, _P, _P, _P, _I32, _P, _I32, _F32, _P, _P, _P, _P, _SIZE, _P]),
    "f3r_pose_metric_workspace": (_SIZE, [_I32, _I32, _I32]),
    "f3r_pose_metric": (C.c_int, [_I32, _P, _P, _I32, _I32, _I32, _P, _P, _P, _P, _SIZE, _P]),
    "f3r_pose_metric_counts": (C.c_int, [_I32, _P, _P, _SIZE, _I32, _P, _P]),
    "f3r_val_loss_workspace": (_SIZE, [_I32, _I32, _I32]),
    "f3r_val_loss": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _F32, _I32, _I32, _I32, _I32, _P, _P, _SIZE,
                               _P]),
    "f3r_sky_mask_workspace": (_SIZE, [_I32, _I32, _I32]),
    "f3r_sky_mask": (C.c_int, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _SIZE, _P]),
    "f3r_scene_sort_workspace": (_SIZE, [_I32]),
    "f3r_scene_sort": (C.c_int, [_P, _P, _P, _P, _P, _I32, _I32, _P, _P, _P, _P, _P, _SIZE, _P]),
    "f3r_scene_visible_workspace": (_SIZE, [_I32, _SIZE]),
    "f3r_scene_visible": (C.c_int, [_P, _I32, _SIZE, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _P, _SIZE, _P]),
    "f3r_ply_pack": (C.c_int, [_P, _P, _SIZE, _P, _P]),
    "f3r_extent_percentiles_workspace": (_SIZE, []),
    "f3r_extent_percentiles": (C.c_int, [_P, _SIZE, _SIZE, _SIZE, _F32, _F32, _P, _P, _SIZE, _P]),
    "f3r_view_geometry": (C.c_int, [_P, _P, _I32, _P, _P, _P, _SIZE, _P]),
}
EXPORTS = list(_API)

_lib = None


def load() -> C.CDLL:
    """Loads the shared library (no CUDA call is made); raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m fast3r_b200.build` (or __graft_entry__.build()). "
            "fast3r_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _API.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.f3r_abi_version() != ABI_VERSION or lib.f3r_gemm_desc_size() != C.sizeof(GemmDesc):
        raise RuntimeError("libfast3r_b200.so ABI mismatch (rebuild: python -m fast3r_b200.build --force)")
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise RuntimeError(f"fast3r_b200 {what} failed: {load().f3r_last_error().decode()}")


def set_option(name: str, value: int) -> None:
    check(load().f3r_set_option(name.encode(), int(value)), "f3r_set_option")


def launch_count() -> int:
    return int(load().f3r_launch_count())
