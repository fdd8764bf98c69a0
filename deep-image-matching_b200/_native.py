"""ctypes binding of libdimb200.so (the C ABI in include/dimb200.h).

There is no CPU fallback: importing this module without the built library, or
creating a context without a CUDA device, raises.  Build with
``python -c "import __graft_entry__ as g; g.build()"`` (or ``make -C csrc``).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DIMB_LIB") or os.path.join(_HERE, "libdimb200.so")  # DIMB_LIB: A/B builds of tools/ only

OK, ERR_CUDA, ERR_OOM, ERR_ARG, ERR_UNSUPPORTED, ERR_CAPACITY = 0, -1, -2, -3, -4, -5
PRECISION_EXACT, PRECISION_FAST = 0, 1
NN_MODES = {"nn": 0, "mnn": 1, "snn": 2, "smnn": 3}

EXPORTS = [
    "dimb_version", "dimb_ctx_create", "dimb_ctx_destroy", "dimb_last_error", "dimb_ctx_set_precision",
    "dimb_ctx_launch_count", "dimb_read_dev",
    "dimb_sp_create", "dimb_sp_destroy", "dimb_sp_extract", "dimb_sp_extract_dev", "dimb_sp_debug_read",
    "dimb_lg_create", "dimb_lg_destroy", "dimb_lg_match", "dimb_lg_match_dev", "dimb_lg_debug_read",
    "dimb_nn_match", "dimb_nn_match_dev", "dimb_nn_match_batch_dev", "dimb_ctx_profile", "dimb_ctx_profile_read", "dimb_pipe_create", "dimb_pipe_destroy",
    "dimb_pipe_match_image_pairs", "dimb_pipe_match_image_pairs_u8", "dimb_pipe_match_image_pairs_dev", "dimb_pipe_outputs_dev", "dimb_pipe_features_dev", "dimb_sp_ctx",
    "dimb_sg_weight_count", "dimb_sg_create", "dimb_sg_destroy", "dimb_sg_match", "dimb_sg_match_dev", "dimb_fstore_sg_feats_dev",
    "dimb_aliked_create", "dimb_aliked_destroy", "dimb_aliked_extract", "dimb_aliked_extract_dev", "dimb_aliked_debug_read",
    "dimb_fstore_create", "dimb_fstore_destroy", "dimb_fstore_put_dev", "dimb_fstore_put", "dimb_fstore_count", "dimb_fstore_get",
    "dimb_fstore_feats_dev", "dimb_fstore_block_dev", "dimb_gv_fundamental", "dimb_gv_estimate", "dimb_gv_fundamental_batch_dev", "dimb_gv_verify_dev",
    "dimb_tile_grid", "dimb_tile_cut_dev", "dimb_tile_merge_dev", "dimb_tile_views_dev", "dimb_tile_match_merge_dev",
    "dimb_resize_area_tab", "dimb_resize_area_dev", "dimb_kpts_extent_dev", "dimb_tile_preselect_dev",
    "dimb_resize_area_linear_tab", "dimb_resize_area_linear_dev", "dimb_resize_area_rgb_dev", "dimb_pyr_size", "dimb_pyr_dev", "dimb_fstore_rescale_dev",
    "dimb_tile_preselect_pairs_dev", "dimb_rot90_dev", "dimb_fstore_unrotate_dev",
    "dimb_sift_create", "dimb_sift_destroy", "dimb_sift_extract", "dimb_sift_extract_dev", "dimb_sift_debug_read",
    "dimb_orb_create", "dimb_orb_destroy", "dimb_orb_extract", "dimb_orb_extract_dev", "dimb_orb_debug_read",
]


class DimbError(RuntimeError):
    pass


class SpConf(C.Structure):
    _fields_ = [("nms_radius", C.c_int), ("keypoint_threshold", C.c_float), ("max_keypoints", C.c_int),
                ("remove_borders", C.c_int), ("fix_sampling", C.c_int), ("max_batch", C.c_int),
                ("max_height", C.c_int), ("max_width", C.c_int)]


class AlikedConf(C.Structure):
    _fields_ = [("max_num_keypoints", C.c_int), ("detection_threshold", C.c_float), ("nms_radius", C.c_int),
                ("max_height", C.c_int), ("max_width", C.c_int)]


class SiftConf(C.Structure):
    _fields_ = [("n_features", C.c_int), ("n_octave_layers", C.c_int), ("contrast_threshold", C.c_double),
                ("edge_threshold", C.c_double), ("sigma", C.c_double), ("max_batch", C.c_int), ("max_height", C.c_int),
                ("max_width", C.c_int)]


class OrbConf(C.Structure):
    _fields_ = [("n_features", C.c_int), ("scale_factor", C.c_double), ("nlevels", C.c_int), ("edge_threshold", C.c_int),
                ("first_level", C.c_int), ("wta_k", C.c_int), ("score_type", C.c_int), ("patch_size", C.c_int),
                ("fast_threshold", C.c_int), ("max_batch", C.c_int), ("max_height", C.c_int), ("max_width", C.c_int)]


class SgConf(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("cross_mask", C.c_ulonglong), ("sinkhorn_iterations", C.c_int), ("match_threshold", C.c_float),
                ("max_kpts", C.c_int), ("max_pairs", C.c_int)]


class SgFeats(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("descriptors", C.c_void_p), ("scores", C.c_void_p), ("n", C.c_int), ("desc_ld", C.c_int),
                ("height", C.c_int), ("width", C.c_int)]


class SgFeatsDev(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("descriptors", C.c_void_p), ("scores", C.c_void_p), ("n", C.c_void_p), ("n_cap", C.c_int),
                ("desc_ld", C.c_int), ("f16", C.c_int), ("round_fp16", C.c_int), ("height", C.c_int), ("width", C.c_int),
                ("size_dev", C.c_void_p)]


class LgConf(C.Structure):
    _fields_ = [("input_dim", C.c_int), ("descriptor_dim", C.c_int), ("n_layers", C.c_int), ("num_heads", C.c_int),
                ("depth_confidence", C.c_double), ("width_confidence", C.c_double), ("filter_threshold", C.c_double),
                ("prune_min_kpts", C.c_int), ("max_pairs", C.c_int), ("max_kpts", C.c_int)]


class Feats(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("descriptors", C.c_void_p), ("n", C.c_int), ("desc_layout", C.c_int),
                ("desc_ld", C.c_int), ("has_size", C.c_int), ("size0", C.c_float), ("size1", C.c_float)]


class FeatsDev(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("descriptors", C.c_void_p), ("n", C.c_void_p), ("n_cap", C.c_int),
                ("desc_layout", C.c_int), ("desc_ld", C.c_int), ("size0", C.c_float), ("size1", C.c_float),
                ("round_fp16", C.c_int), ("f16", C.c_int), ("size_dev", C.c_void_p), ("size_f32_dev", C.c_void_p)]


class GvConf(C.Structure):
    _fields_ = [("threshold", C.c_float), ("max_iters", C.c_int), ("min_inliers", C.c_int), ("min_inlier_ratio", C.c_float),
                ("estimator", C.c_int), ("confidence", C.c_float)]


GV_ESTIMATORS = {"ransac8": 0, "lo-ransac": 1, "degensac": 3}


def gv_estimator(name) -> int:
    """dimb_gv_conf.estimator of an estimator name in GV_ESTIMATORS; ValueError otherwise."""
    if name not in GV_ESTIMATORS:
        raise ValueError(f"unknown geometric verification estimator {name!r}; expected one of {list(GV_ESTIMATORS)}")
    return GV_ESTIMATORS[name]


_lib = None


def load_library():
    """Load libdimb200.so and declare prototypes. Raises DimbError if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DimbError(f"{LIB_PATH} is missing: build the CUDA extension first (__graft_entry__.build()); "
                        "this package has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    vp, ip, fp = C.c_void_p, C.c_int, C.c_float
    lib.dimb_version.restype = C.c_char_p
    lib.dimb_ctx_create.argtypes = [ip, C.POINTER(vp)]
    lib.dimb_ctx_destroy.argtypes = [vp]
    lib.dimb_ctx_destroy.restype = None
    lib.dimb_last_error.argtypes = [vp]
    lib.dimb_last_error.restype = C.c_char_p
    lib.dimb_ctx_set_precision.argtypes = [vp, ip]
    lib.dimb_ctx_launch_count.argtypes = [vp]
    lib.dimb_ctx_launch_count.restype = C.c_ulonglong
    lib.dimb_read_dev.argtypes = [vp, vp, vp, C.c_size_t]
    lib.dimb_sp_create.argtypes = [vp, vp, C.c_size_t, C.POINTER(SpConf), C.POINTER(vp)]
    lib.dimb_sp_destroy.argtypes = [vp]
    lib.dimb_sp_destroy.restype = None
    lib.dimb_sp_extract.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, ip]
    lib.dimb_sp_extract_dev.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, ip, vp]
    lib.dimb_sp_debug_read.argtypes = [vp, ip, vp, C.c_size_t]
    lib.dimb_lg_create.argtypes = [vp, vp, C.c_size_t, C.POINTER(LgConf), C.POINTER(vp)]
    lib.dimb_lg_destroy.argtypes = [vp]
    lib.dimb_lg_destroy.restype = None
    lib.dimb_lg_match.argtypes = [vp, ip, C.POINTER(Feats), C.POINTER(Feats), vp, vp, vp, vp, ip]
    lib.dimb_lg_match_dev.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev), vp, vp, vp, vp, ip, vp]
    lib.dimb_lg_debug_read.argtypes = [vp, ip, ip, vp, C.c_size_t]
    lib.dimb_nn_match.argtypes = [vp, vp, ip, vp, ip, ip, ip, fp, vp, vp, C.POINTER(ip), ip]
    lib.dimb_nn_match_dev.argtypes = [vp, vp, ip, ip, vp, ip, ip, ip, ip, ip, fp, vp, vp, vp, ip, vp]
    lib.dimb_nn_match_batch_dev.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev), ip, ip, fp, vp, vp, vp, ip, vp]
    lib.dimb_ctx_profile.argtypes = [vp, ip]
    lib.dimb_ctx_profile_read.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.dimb_pipe_create.argtypes = [vp, vp, ip, ip, ip, ip, C.POINTER(vp)]
    lib.dimb_pipe_destroy.argtypes = [vp]
    lib.dimb_pipe_destroy.restype = None
    lib.dimb_pipe_match_image_pairs.argtypes = [vp, vp, ip, vp, vp, vp, vp, vp, vp]
    lib.dimb_pipe_match_image_pairs_u8.argtypes = [vp, vp, ip, vp, vp, vp, vp, vp, vp]
    lib.dimb_pipe_match_image_pairs_dev.argtypes = [vp, vp, ip, vp]
    lib.dimb_pipe_outputs_dev.argtypes = [vp] + [C.POINTER(vp)] * 6
    lib.dimb_pipe_features_dev.argtypes = [vp] + [C.POINTER(vp)] * 4
    lib.dimb_sp_ctx.argtypes = [vp]
    lib.dimb_sg_weight_count.argtypes = [ip]
    lib.dimb_sg_weight_count.restype = C.c_size_t
    lib.dimb_sg_create.argtypes = [vp, vp, C.c_size_t, C.POINTER(SgConf), C.POINTER(vp)]
    lib.dimb_sg_destroy.argtypes = [vp]
    lib.dimb_sg_destroy.restype = None
    lib.dimb_sg_match.argtypes = [vp, C.POINTER(SgFeats), C.POINTER(SgFeats), vp, vp, C.POINTER(ip), ip]
    lib.dimb_sg_match_dev.argtypes = [vp, ip, C.POINTER(SgFeatsDev), C.POINTER(SgFeatsDev), vp, vp, vp, ip, vp]
    lib.dimb_aliked_create.argtypes = [vp, vp, C.c_size_t, C.POINTER(AlikedConf), C.POINTER(vp)]
    lib.dimb_aliked_destroy.argtypes = [vp]
    lib.dimb_aliked_destroy.restype = None
    lib.dimb_aliked_extract.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, ip]
    lib.dimb_aliked_extract_dev.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, ip, vp]
    lib.dimb_aliked_debug_read.argtypes = [vp, ip, vp, C.c_size_t]
    lib.dimb_sift_create.argtypes = [vp, C.POINTER(SiftConf), C.POINTER(vp)]
    lib.dimb_sift_destroy.argtypes = [vp]
    lib.dimb_sift_destroy.restype = None
    lib.dimb_sift_extract.argtypes = [vp, vp, ip, ip, vp, vp, vp, vp, vp, ip]
    lib.dimb_sift_extract_dev.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, vp, ip, vp]
    lib.dimb_sift_debug_read.argtypes = [vp, ip, ip, ip, vp, C.c_size_t]
    lib.dimb_orb_create.argtypes = [vp, C.POINTER(OrbConf), C.POINTER(vp)]
    lib.dimb_orb_destroy.argtypes = [vp]
    lib.dimb_orb_destroy.restype = None
    lib.dimb_orb_extract.argtypes = [vp, vp, ip, ip, vp, vp, vp, vp, vp, ip]
    lib.dimb_orb_extract_dev.argtypes = [vp, vp, ip, ip, ip, vp, vp, vp, vp, vp, ip, vp]
    lib.dimb_orb_debug_read.argtypes = [vp, ip, ip, ip, vp, C.c_size_t]
    lib.dimb_sp_ctx.restype = vp
    lib.dimb_fstore_create.argtypes = [vp, ip, ip, ip, C.POINTER(vp)]
    lib.dimb_fstore_destroy.argtypes = [vp]
    lib.dimb_fstore_destroy.restype = None
    lib.dimb_fstore_put_dev.argtypes = [vp, ip, vp, vp, vp, vp, ip, vp, ip, ip, vp]
    lib.dimb_fstore_put.argtypes = [vp, ip, vp, vp, vp, vp, ip, ip, ip]
    lib.dimb_fstore_count.argtypes = [vp, ip, C.POINTER(ip), vp]
    lib.dimb_fstore_get.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(ip), vp, ip]
    lib.dimb_fstore_feats_dev.argtypes = [vp, ip, C.POINTER(FeatsDev)]
    lib.dimb_fstore_sg_feats_dev.argtypes = [vp, ip, C.POINTER(SgFeatsDev)]
    lib.dimb_gv_fundamental.argtypes = [vp, vp, vp, ip, fp, ip, C.c_uint, vp, vp, C.POINTER(ip)]
    lib.dimb_gv_estimate.argtypes = [vp, vp, vp, ip, C.POINTER(GvConf), C.c_uint, vp, vp, C.POINTER(ip), C.POINTER(ip)]
    lib.dimb_gv_fundamental_batch_dev.argtypes = [vp, ip, vp, vp, vp, vp, ip, fp, ip, C.c_uint, vp, vp, vp, vp]
    lib.dimb_gv_verify_dev.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev), vp, vp, ip, C.POINTER(C.c_uint),
                                       C.POINTER(GvConf), vp, vp, vp, vp, vp, vp]
    lib.dimb_fstore_block_dev.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t), C.POINTER(ip), C.POINTER(ip)]
    lib.dimb_tile_grid.argtypes = [ip] * 6 + [vp]
    lib.dimb_tile_cut_dev.argtypes = [vp, vp] + [ip] * 8 + [vp, vp]
    lib.dimb_tile_merge_dev.argtypes = [vp, ip, vp] + [ip] * 6 + [vp, vp, vp, vp, ip, vp]
    lib.dimb_tile_views_dev.argtypes = [vp, ip, vp, ip, vp, vp, vp, vp]
    lib.dimb_tile_match_merge_dev.argtypes = [vp, ip, vp, vp, vp, vp, ip, vp, vp, ip, vp, vp, ip, vp]
    lib.dimb_resize_area_tab.argtypes = [ip, ip, vp, vp, vp, ip, C.POINTER(ip)]
    lib.dimb_resize_area_dev.argtypes = [vp, vp, ip, ip, ip, vp, ip, ip, vp]
    lib.dimb_resize_area_linear_tab.argtypes = [ip, ip, vp, vp, C.POINTER(ip)]
    lib.dimb_resize_area_linear_dev.argtypes = [vp, vp, ip, ip, ip, vp, ip, ip, vp]
    lib.dimb_resize_area_rgb_dev.argtypes = [vp, vp, ip, ip, ip, vp, ip, ip, vp]
    lib.dimb_pyr_size.argtypes = [ip, ip, ip, C.POINTER(ip), C.POINTER(ip)]
    lib.dimb_pyr_dev.argtypes = [vp, vp, ip, ip, ip, ip, ip, vp, vp]
    lib.dimb_fstore_rescale_dev.argtypes = [vp, ip, vp, ip, ip, ip, vp]
    lib.dimb_rot90_dev.argtypes = [vp, vp, ip, ip, ip, ip, vp, vp, vp]
    lib.dimb_fstore_unrotate_dev.argtypes = [vp, ip, vp, vp, vp, vp, vp]
    lib.dimb_kpts_extent_dev.argtypes = [vp, ip, vp, ip, vp, vp, vp]
    lib.dimb_tile_preselect_dev.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev), vp, vp, ip] + [ip] * 6 + \
        [C.c_double, C.c_double, ip, vp, vp, vp]
    lib.dimb_tile_preselect_pairs_dev.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev), vp, vp, ip, vp] + [ip] * 4 + \
        [vp, ip, vp, vp, vp]
    _lib = lib
    return lib


_selftest = None


def load_selftest_library():
    """libdimb200_selftest.so: the production GEMM template behind a C = A B^T entry, the flash-attention kernels behind an
    attention entry, keypoint detection (simple_nms, compaction, top-k), the SuperPoint head kernels, the matching heads (LightGlue
    assignment and tail, SuperGlue Sinkhorn), the SIFT stages (extrema, orientation, selection, descriptors), the ALIKED stages
    (convolutions, fusion, DKD, SDDH) and the brute-force NN engine (row statistics, mode logic) behind their own entries, and the
    host drive of the RANSAC arithmetic.
    Test / tool infrastructure - the product library exports none of it.  Its context is its own (dimb_ctx_create of
    THIS library); never mix handles of the two libraries."""
    global _selftest
    if _selftest is None:
        path = os.path.join(_HERE, "libdimb200_selftest.so")
        if not os.path.exists(path):
            raise DimbError(f"{path} is missing: build the CUDA extension first (__graft_entry__.build())")
        lib = C.CDLL(path)
        vp, ip = C.c_void_p, C.c_int
        lib.dimb_ctx_create.argtypes = [ip, C.POINTER(vp)]
        lib.dimb_ctx_destroy.argtypes = [vp]
        lib.dimb_ctx_destroy.restype = None
        lib.dimb_last_error.argtypes = [vp]
        lib.dimb_last_error.restype = C.c_char_p
        lib.dimb_ctx_set_precision.argtypes = [vp, ip]
        fp = C.c_float
        lib.dimb_selftest_gemm.argtypes = [vp, vp, vp, vp, vp, ip, ip, ip, ip, ip, fp, vp]
        lib.dimb_selftest_gemm_plan.argtypes = [ip] * 8 + [vp]
        lib.dimb_selftest_conv3x3.argtypes = [vp, vp, vp, vp, vp] + [ip] * 7 + [fp, fp, vp]
        lib.dimb_selftest_conv_mode.argtypes = [ip] * 5 + [vp]
        lib.dimb_selftest_conv3x3_time.argtypes = [vp] + [ip] * 9 + [vp, vp]
        lib.dimb_selftest_attention.argtypes = [vp, ip, vp, vp, vp, vp, ip, ip, ip, ip, vp, vp, ip, fp, fp, fp]
        lib.dimb_selftest_nms_plan.argtypes = [ip, ip, vp]
        lib.dimb_selftest_detect.argtypes = [vp, vp] + [ip] * 5 + [fp, vp, ip, ip, ip, fp] + [vp] * 8
        lib.dimb_selftest_select.argtypes = [vp, vp] + [ip] * 5 + [fp, vp] + [ip] * 5 + [fp] + [vp] * 7 + [ip, vp]
        lib.dimb_selftest_sp_softmax.argtypes = [vp, vp, ip, ip, ip, fp, vp]
        lib.dimb_selftest_sp_describe.argtypes = [vp] * 5 + [ip] * 5 + [fp, vp, vp, vp]
        lib.dimb_selftest_lg_assign.argtypes = [vp, ip, ip] + [vp] * 6 + [fp, ip, fp] + [vp] * 8
        lib.dimb_selftest_lg_tail.argtypes = [vp, ip, ip, vp, vp, fp, vp, fp] + [vp] * 6 + [ip, fp, fp, fp, ip, ip, ip, fp] + [vp] * 6
        lib.dimb_selftest_lgx_assign.argtypes = [vp, ip, ip, ip] + [vp] * 5 + [fp, ip, fp] + [vp] * 11
        lib.dimb_selftest_sg_sinkhorn.argtypes = [vp, ip, vp, vp, vp, fp, fp, vp, vp, ip, ip, fp, ip, fp] + [vp] * 9
        lib.dimb_selftest_sift_extrema.argtypes = [vp, vp, ip, ip, ip, vp, vp, fp, fp, fp, ip, fp, vp, vp]
        lib.dimb_selftest_sift_ori.argtypes = [vp, vp, ip, ip, ip, vp, vp, fp, vp, vp, ip, ip, fp, vp, vp]
        lib.dimb_selftest_sift_select.argtypes = [vp, vp, vp, ip, ip, ip, ip, fp] + [vp] * 5
        lib.dimb_selftest_sift_desc.argtypes = [vp, vp, ip, ip, ip] + [vp] * 5 + [ip, ip, fp, vp]
        lib.dimb_selftest_aliked_conv_plan.argtypes = [ip, ip, ip, vp]
        lib.dimb_selftest_aliked_conv3x3.argtypes = [vp, ip, vp, ip, ip, ip, vp, vp, vp, vp, ip, ip, fp, vp, vp]
        lib.dimb_selftest_aliked_conv1x1.argtypes = [vp, vp, ip, ip, vp, vp, ip, ip, fp, vp]
        lib.dimb_selftest_aliked_avgpool.argtypes = [vp, vp, ip, ip, ip, ip, fp, vp]
        lib.dimb_selftest_aliked_pad.argtypes = [vp, vp, ip, ip, ip, fp, vp, vp]
        lib.dimb_selftest_aliked_crop.argtypes = [vp, vp] + [ip] * 6 + [fp, vp]
        lib.dimb_selftest_aliked_deform.argtypes = [vp, vp, ip, ip, ip, vp, fp, vp, vp, vp, vp, vp, ip, ip, fp, vp, vp]
        lib.dimb_selftest_aliked_fuse.argtypes = [vp] * 7 + [ip] * 6 + [fp, vp, vp]
        lib.dimb_selftest_aliked_dkd.argtypes = [vp, vp, ip, ip, ip, vp, ip, ip, fp, vp, vp, vp]
        lib.dimb_selftest_aliked_sddh.argtypes = [vp, vp, ip, ip, vp, ip, ip] + [vp] * 7 + [fp, vp, vp, vp]
        lib.dimb_selftest_aliked_threshold.argtypes = [vp, vp, ip, vp, fp, fp, vp]
        lib.dimb_selftest_nn_stats.argtypes = [vp, ip, C.POINTER(FeatsDev), C.POINTER(FeatsDev)] + [ip] * 5 + [fp] + [vp] * 5
        lib.dimb_selftest_nn_select.argtypes = [vp, ip, fp, ip, ip] + [vp] * 4 + [ip, fp] + [vp] * 3
        lib.dimb_gv_host.argtypes = [vp, vp, ip, C.c_float, ip, C.c_uint, vp, vp]
        lib.dimb_gv_lo_host.argtypes = [vp, vp, ip, C.c_float, ip, C.c_float, C.c_uint, vp, vp, C.POINTER(ip)]
        lib.dimb_gv_seven_point_host.argtypes = [vp, vp, vp]
        lib.dimb_gv_degensac_host.argtypes = [vp, vp, ip, C.c_float, ip, C.c_float, C.c_uint, vp, vp, C.POINTER(ip)]
        lib.dimb_gv_h_from_f3_host.argtypes = [vp, vp, vp, ip, vp, vp]
        lib.dimb_gv_degenerate_host.argtypes = [vp, vp, vp, ip, vp, C.c_float, vp]
        lib.dimb_gv_plane_parallax_host.argtypes = [vp, vp, vp, ip, ip, ip, vp]
        _selftest = lib
    return _selftest


def gemm_plan(conv: int, bn: int, split: bool, const_b: bool, num_kb: int, m_tiles: int, n_tiles: int, num_sms: int):
    """Launch plan (resb, sa, sb, smem_bytes, grid) of the persistent tensor-core kernel for one call shape, as launch_gemm computes
    it (dimb_selftest_gemm_plan).  Host only: needs neither a context nor a GPU."""
    out = np.zeros(5, np.int32)
    rc = load_selftest_library().dimb_selftest_gemm_plan(conv, bn, int(bool(split)), int(bool(const_b)), num_kb, m_tiles, n_tiles,
                                                         num_sms, _ptr(out))
    if rc != OK:
        raise DimbError(f"gemm_plan({conv}, {bn}, ...) failed (code {rc})")
    return tuple(int(p) for p in out)


def conv_mode(cout: int, B: int, H: int, W: int, num_sms: int) -> int:
    """Tile shape the SuperPoint 3x3 conv launch picks on the tensor-core kernel, as the csrc/gemm.cuh CONV mode: 1 = 8 x 16 pixels,
    2 = 16 x 16 pixels (dimb_selftest_conv_mode).  Host only."""
    out = np.zeros(1, np.int32)
    rc = load_selftest_library().dimb_selftest_conv_mode(cout, B, H, W, num_sms, _ptr(out))
    if rc != OK:
        raise DimbError(f"conv_mode({cout}, {B}, {H}, {W}, {num_sms}) failed (code {rc})")
    return int(out[0])


def aliked_conv_plan(H: int, W: int, cout: int) -> int:
    """The al_conv3x3_kernel instantiation ALIKED's conv3 runs on an H x W map with cout output channels: 1 = <8,1>, 2 = <16,4>, 3 =
    <8,4> (dimb_selftest_aliked_conv_plan).  Host only."""
    out = np.zeros(1, np.int32)
    rc = load_selftest_library().dimb_selftest_aliked_conv_plan(int(H), int(W), int(cout), _ptr(out))
    if rc != OK:
        raise DimbError(f"aliked_conv_plan({H}, {W}, {cout}) failed (code {rc})")
    return int(out[0])


def nms_plan(r: int, cut: int = 0):
    """Launch plan (kernel, tile, threads, smem_bytes) of simple_nms at radius r (dimb_selftest_nms_plan): kernel 1 = first cut, 2 =
    bit-mask kernel.  cut 0 = the production choice, 1 = first cut (radii 0..8), 2 = bit-mask kernel (radii 1..5).  Host only."""
    out = np.zeros(4, np.int32)
    rc = load_selftest_library().dimb_selftest_nms_plan(int(r), int(cut), _ptr(out))
    if rc != OK:
        raise DimbError(f"nms_plan({r}, {cut}) failed (code {rc})")
    return tuple(int(p) for p in out)


DET_TAIL = 1024  # elements past the valid ones in every output buffer of the detection / head self-tests


class SelfTest:
    """Context of the self-test library (tests/test_gemm_conv_kernel.py, tests/test_attention_kernel.py, tests/test_detect_kernel.py,
    tests/test_match_heads.py, tests/test_sift_kernels.py, tests/test_aliked_kernels.py, tests/test_nn_kernels.py)."""

    def __init__(self, device: int = 0):
        self.lib = load_selftest_library()
        h = C.c_void_p()
        if self.lib.dimb_ctx_create(device, C.byref(h)) != OK:
            raise DimbError("selftest: dimb_ctx_create failed (an H100 is required)")
        self.h = h

    def check(self, rc, what):
        if rc != OK:
            raise DimbError(f"{what} failed (code {rc}): {self.lib.dimb_last_error(self.h).decode()}")

    def set_precision(self, precision: str):
        self.check(self.lib.dimb_ctx_set_precision(self.h, {"exact": 0, "fast": 1}[precision]), "set_precision")

    def gemm(self, A: np.ndarray, B: np.ndarray, bn: int = 128, bias=None, k32: bool = False, guard: float = 0.0):
        """C = A B^T (+ bias) through the production GEMM launch (dimb_selftest_gemm), precision of the context.  A [M][K], B [N][K],
        K a multiple of 64; k32: 32-wide K blocks (bn 256).  Rows of the operand allocations past M / N, and the output buffer, hold
        `guard`.  Returns (C [M][N], tail [128][N] of the output buffer past the last row, plan
        {resb, sa, sb, smem_bytes, grid} of the launch)."""
        A = np.ascontiguousarray(A, np.float32)
        B = np.ascontiguousarray(B, np.float32)
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
        M, K = A.shape
        N = B.shape[0]
        Cm = np.zeros((M + 128, N), np.float32)
        plan = np.zeros(5, np.int32)
        self.check(self.lib.dimb_selftest_gemm(self.h, _ptr(A), _ptr(B), None if bias is None else _ptr(bias), _ptr(Cm), M, N, K, bn,
                                               int(bool(k32)), float(guard), _ptr(plan)), "selftest_gemm")
        return Cm[:M], Cm[M:], tuple(int(p) for p in plan)

    def conv3x3(self, x: np.ndarray, w: np.ndarray, bias: np.ndarray, pool: bool, guard: float = 0.0, sentinel: float = 0.0):
        """One SuperPoint 3x3 conv layer (zero padding, bias, ReLU, optional 2x2 max pool) through its production launch
        (dimb_selftest_conv3x3), precision of the context.  x NHWC [B][H][W][cin], w OIHW [cout][cin][3][3].  The input allocation
        holds one more image of `guard`; the output buffer starts as `sentinel`.  Returns (out [B][Ho][Wo][cout], tail: one more
        output image of the buffer, plan as gemm())."""
        return self.conv3x3_tiles(x, w, bias, pool, 0, guard, sentinel)[:3]

    def conv3x3_tiles(self, x: np.ndarray, w: np.ndarray, bias: np.ndarray, pool: bool, tile: int, guard: float = 0.0,
                      sentinel: float = 0.0):
        """conv3x3() on one tile shape: tile 8 = 8 x 16 pixels, 16 = 16 x 16 pixels (cout 64), 0 = the shape production picks.
        Returns (out, tail, plan, the csrc/gemm.cuh CONV mode that ran)."""
        x = np.ascontiguousarray(x, np.float32)
        w = np.ascontiguousarray(w, np.float32)
        bias = np.ascontiguousarray(bias, np.float32)
        B, H, W, cin = x.shape
        cout = w.shape[0]
        Ho, Wo = (H // 2, W // 2) if pool else (H, W)
        out = np.zeros((B + 1, Ho, Wo, cout), np.float32)
        plan = np.zeros(6, np.int32)
        self.check(self.lib.dimb_selftest_conv3x3(self.h, _ptr(x), _ptr(w), _ptr(bias), _ptr(out), B, H, W, cin, cout, int(bool(pool)),
                                                  int(tile), float(guard), float(sentinel), _ptr(plan)), "selftest_conv3x3")
        return out[:B], out[B], tuple(int(p) for p in plan[:5]), int(plan[5])

    def conv3x3_time(self, B: int, H: int, W: int, cin: int, cout: int, pool: bool, tile: int, warm: int = 2, iters: int = 10):
        """Device milliseconds per call of one 3x3 conv layer on device-generated activations (dimb_selftest_conv3x3_time),
        precision of the context; tile as conv3x3_tiles().  Returns (ms, plan, CONV mode)."""
        ms = np.zeros(1, np.float32)
        plan = np.zeros(6, np.int32)
        self.check(self.lib.dimb_selftest_conv3x3_time(self.h, B, H, W, cin, cout, int(bool(pool)), int(tile), warm, iters, _ptr(ms),
                                                       _ptr(plan)), "selftest_conv3x3_time")
        return float(ms[0]), tuple(int(p) for p in plan[:5]), int(plan[5])

    def attention(self, variant: int, Q: np.ndarray, K, V: np.ndarray, n, heads: int = 4, stopped=None, cross: bool = False,
                  lazy: float = -1.0, pad: float = 0.0, out_pad: float = 0.0) -> np.ndarray:
        """The flash-attention kernels through their production launches (dimb_selftest_attention), precision of the context.
        variant 0 (LightGlue / SuperGlue, 4 heads x 64): Q, K, V [S][4][NP][64], n [S] live rows per side, stopped [S/2]; with
        cross the keys of side s are the q rows of side s ^ 1 (K unused).  Returns the context buffer [S][NP][256] (head h at
        columns 64 h).  variant 1 (head dim <= 128): Q [n0][heads * hd], K / V [n1][heads * hd], n = (n0, n1); returns
        [NPp][heads * hd], NPp = max(n0, n1, 1) rounded up to 128.  Rows past the live counts hold `pad` on the way in; the
        output buffer starts as `out_pad`.  lazy: rescale threshold in log2 units, in [0, 15]; negative = the context's."""
        Q = np.ascontiguousarray(Q, np.float32)
        V = np.ascontiguousarray(V, np.float32)
        K = None if K is None else np.ascontiguousarray(K, np.float32)
        nn = np.ascontiguousarray(n, np.int32)
        if variant == 0:
            S, H, NP, hd = Q.shape
            st = np.ascontiguousarray(stopped if stopped is not None else np.zeros(S // 2), np.int32)
            out = np.zeros((S, NP, H * hd), np.float32)
        else:
            H, hd, NP = int(heads), Q.shape[1] // int(heads), max(int(nn[0]), int(nn[1]), 1)
            S, st = 1, np.zeros(1, np.int32)
            out = np.zeros(((NP + 127) // 128 * 128, H * hd), np.float32)
            if K.shape[0] == 0:  # no keys: the entry still wants valid pointers
                K = V = np.zeros((1, H * hd), np.float32)
        self.check(self.lib.dimb_selftest_attention(self.h, int(variant), _ptr(Q), _ptr(K) if K is not None else None, _ptr(V), _ptr(out),
                                                    S, H, hd, NP, _ptr(nn), _ptr(st), int(bool(cross)), float(lazy), float(pad),
                                                    float(out_pad)), "selftest_attention")
        return out

    def detect(self, scores: np.ndarray, r: int, cut: int = 0, thr: float = 0.0, thr_per_image=None, border: int = 0, K: int = -1,
               cap: int | None = None, sentinel: float = -777.0) -> dict:
        """simple_nms, candidate compaction and top-k through their production launches (dimb_selftest_detect).  scores [B][H][W]
        positive; cut as nms_plan(); candidates are nms > thr (thr_per_image [B]: through
        the device-threshold argument) at least `border` pixels inside; K = -1 keeps every candidate; cap defaults to K (H * W when
        K = -1).  Every buffer starts as `sentinel` (int buffers: its bit pattern).  Returns a dict of nms [B][H][W], cand_count [B],
        cand_idx / cand_score [B][H * W], sel_idx / sel_score [B][cap], sel_count [B], '<name>_tail' [DET_TAIL] for each, and plan."""
        s = np.ascontiguousarray(scores, np.float32)
        B, H, W = s.shape
        cap = int(cap if cap is not None else (K if K > 0 else H * W))
        tp = None if thr_per_image is None else np.ascontiguousarray(thr_per_image, np.float32)
        n, ns = B * H * W, B * cap
        bufs = {"nms": (np.float32, n), "cand_count": (np.int32, B), "cand_idx": (np.int32, n), "cand_score": (np.float32, n),
                "sel_idx": (np.int32, ns), "sel_score": (np.float32, ns), "sel_count": (np.int32, B)}
        raw = {k: np.zeros(m + DET_TAIL, t) for k, (t, m) in bufs.items()}
        plan = np.zeros(4, np.int32)
        self.check(self.lib.dimb_selftest_detect(self.h, _ptr(s), B, H, W, int(r), int(cut), float(thr), None if tp is None else _ptr(tp),
                                                 int(border), int(K), cap, float(sentinel), *(_ptr(raw[k]) for k in bufs), _ptr(plan)),
                   "selftest_detect")
        shapes = {"nms": (B, H, W), "cand_idx": (B, H * W), "cand_score": (B, H * W), "sel_idx": (B, cap), "sel_score": (B, cap)}
        out = {k: raw[k][:m].reshape(shapes.get(k, (B,))) for k, (_, m) in bufs.items()}
        out.update({k + "_tail": raw[k][m:] for k, (_, m) in bufs.items()})
        out["plan"] = tuple(int(p) for p in plan)
        return out

    def select(self, scores: np.ndarray, r: int, K: int, cut: int = 0, thr: float = 0.0, thr_per_image=None, border: int = 0,
               cap: int | None = None, sort_all: bool = False, grid: bool = False, sentinel: float = -777.0, iters: int = 0) -> dict:
        """detect() with the top-k selection of any K >= 1 (dimb_selftest_select).  sort_all: ALIKED's top-k mode (sorted even when
        count <= K, then the first non-candidate pixels up to K; K <= H * W).  grid: the grid-wide path whatever K (default: the path
        production runs for K).  iters > 0: the selection alone is timed over that many more runs, out["ms"] per run.  Returns
        detect()'s dict without plan."""
        s = np.ascontiguousarray(scores, np.float32)
        B, H, W = s.shape
        cap = int(cap if cap is not None else K)
        tp = None if thr_per_image is None else np.ascontiguousarray(thr_per_image, np.float32)
        n, ns = B * H * W, B * cap
        bufs = {"nms": (np.float32, n), "cand_count": (np.int32, B), "cand_idx": (np.int32, n), "cand_score": (np.float32, n),
                "sel_idx": (np.int32, ns), "sel_score": (np.float32, ns), "sel_count": (np.int32, B)}
        raw = {k: np.zeros(m + DET_TAIL, t) for k, (t, m) in bufs.items()}
        ms = np.zeros(1, np.float32)
        self.check(self.lib.dimb_selftest_select(self.h, _ptr(s), B, H, W, int(r), int(cut), float(thr), None if tp is None else _ptr(tp),
                                                 int(border), int(K), cap, int(bool(sort_all)), int(bool(grid)), float(sentinel),
                                                 *(_ptr(raw[k]) for k in bufs), int(iters), _ptr(ms)), "selftest_select")
        shapes = {"nms": (B, H, W), "cand_idx": (B, H * W), "cand_score": (B, H * W), "sel_idx": (B, cap), "sel_score": (B, cap)}
        out = {k: raw[k][:m].reshape(shapes.get(k, (B,))) for k, (_, m) in bufs.items()}
        out.update({k + "_tail": raw[k][m:] for k, (_, m) in bufs.items()})
        out["ms"] = float(ms[0])
        return out

    def sp_softmax(self, logits: np.ndarray, B: int, h: int, w: int, sentinel: float = -777.0):
        """sp_softmax_d2s_kernel through its production launch (dimb_selftest_sp_softmax): logits [B * h * w][65] -> (scores
        [B][8h][8w], tail [DET_TAIL] of the output buffer, which starts as `sentinel`)."""
        lg = np.ascontiguousarray(logits, np.float32)
        out = np.zeros(B * h * w * 64 + DET_TAIL, np.float32)
        self.check(self.lib.dimb_selftest_sp_softmax(self.h, _ptr(lg), B, h, w, float(sentinel), _ptr(out)), "selftest_sp_softmax")
        return out[:-DET_TAIL].reshape(B, 8 * h, 8 * w), out[-DET_TAIL:]

    def sp_describe(self, sel_idx: np.ndarray, sel_score: np.ndarray, sel_count, dense: np.ndarray, h: int, w: int, fix_sampling: bool,
                    sentinel: float = -777.0) -> dict:
        """sp_describe_kernel through its production launch (dimb_selftest_sp_describe).  sel_idx / sel_score [B][cap], sel_count [B],
        dense [B][h * w][256].  Returns kpts [B][cap][2], scores [B][cap], desc [B][256][cap] and '<name>_tail' [DET_TAIL] of each
        buffer; every buffer starts as `sentinel`."""
        si = np.ascontiguousarray(sel_idx, np.int32)
        ss = np.ascontiguousarray(sel_score, np.float32)
        sc = np.ascontiguousarray(sel_count, np.int32)
        d = np.ascontiguousarray(dense, np.float32)
        B, cap = si.shape
        shapes = {"kpts": (B, cap, 2), "scores": (B, cap), "desc": (B, 256, cap)}
        raw = {k: np.zeros(int(np.prod(s)) + DET_TAIL, np.float32) for k, s in shapes.items()}
        self.check(self.lib.dimb_selftest_sp_describe(self.h, _ptr(si), _ptr(ss), _ptr(sc), _ptr(d), B, h, w, cap, int(bool(fix_sampling)),
                                                      float(sentinel), *(_ptr(raw[k]) for k in shapes)), "selftest_sp_describe")
        out = {k: raw[k][:-DET_TAIL].reshape(s) for k, s in shapes.items()}
        out.update({k + "_tail": raw[k][-DET_TAIL:] for k in shapes})
        return out

    def _run(self, fn, what, bufs, *args):
        """Calls fn(handle, *args, *pointers of bufs); bufs: name -> (dtype, valid length).  Every buffer holds DET_TAIL more
        elements.  Returns (name -> the valid part, name -> the tail)."""
        raw = {k: np.zeros(m + DET_TAIL, t) for k, (t, m) in bufs.items()}
        self.check(fn(self.h, *args, *(_ptr(raw[k]) for k in bufs)), what)
        return {k: raw[k][:m] for k, (_, m) in bufs.items()}, {k: raw[k][m:] for k, (_, m) in bufs.items()}

    @staticmethod
    def _sift_levels(levels):
        """levels: per octave an array [n_levels][B][h][w] -> (concatenated float32 levels, B, n_oct, h [n_oct], w [n_oct])."""
        levels = [np.ascontiguousarray(x, np.float32) for x in levels]
        h = np.array([x.shape[2] for x in levels], np.int32)
        w = np.array([x.shape[3] for x in levels], np.int32)
        return np.concatenate([x.ravel() for x in levels]), levels[0].shape[1], len(levels), h, w

    def sift_extrema(self, dog, L: int, contrast: float, edge: float, sigma: float, ccap: int, sentinel: float = -777.0):
        """sift.extrema through its launch helper (dimb_selftest_sift_extrema) on DoG levels: per octave [L + 2][B][h][w].  Returns
        (cand [B][ccap][6] int32 Cand records in atomic order, count [B], {'cand', 'count'} tails)."""
        lv, B, n_oct, h, w = self._sift_levels(dog)
        out, tail = self._run(self.lib.dimb_selftest_sift_extrema, "selftest_sift_extrema",
                              {"cand": (np.int32, B * ccap * 6), "count": (np.int32, B)}, _ptr(lv), B, L, n_oct, _ptr(h), _ptr(w),
                              float(contrast), float(edge), float(sigma), int(ccap), float(sentinel))
        return out["cand"].reshape(B, ccap, 6), out["count"], tail

    def sift_ori(self, gauss, L: int, sigma: float, cand: np.ndarray, cand_count, kcap: int, sentinel: float = -777.0):
        """sift.ori through its launch helper (dimb_selftest_sift_ori) on Gaussian levels (per octave [L + 3][B][h][w]) and Cand records
        cand [B][ccap][6] int32.  Returns (rec [B][6][kcap] float32, kp_count [B], {'rec', 'kp_count'} tails)."""
        lv, B, n_oct, h, w = self._sift_levels(gauss)
        cand = np.ascontiguousarray(cand, np.int32)
        cc = np.ascontiguousarray(cand_count, np.int32)
        ccap = cand.shape[1]
        out, tail = self._run(self.lib.dimb_selftest_sift_ori, "selftest_sift_ori",
                              {"rec": (np.float32, B * 6 * kcap), "kp_count": (np.int32, B)}, _ptr(lv), B, L, n_oct, _ptr(h), _ptr(w),
                              float(sigma), _ptr(cand), _ptr(cc), int(ccap), int(kcap), float(sentinel))
        return out["rec"].reshape(B, 6, kcap), out["kp_count"], tail

    def sift_select(self, rec: np.ndarray, kp_count, n_features: int, cap: int, sentinel: float = -777.0):
        """sift.select through its launch helper (dimb_selftest_sift_select) on records rec [B][6][kcap].  Returns a dict of sel
        [B][cap] (record index of each output row), kpts [B][cap][2], frames [B][cap][3], octave [B][cap], counts [B] and
        '<name>_tail' of each."""
        rec = np.ascontiguousarray(rec, np.float32)
        kc = np.ascontiguousarray(kp_count, np.int32)
        B, _, kcap = rec.shape
        shapes = {"sel": (np.int32, (B, cap)), "kpts": (np.float32, (B, cap, 2)), "frames": (np.float32, (B, cap, 3)),
                  "octave": (np.int32, (B, cap)), "counts": (np.int32, (B,))}
        out, tail = self._run(self.lib.dimb_selftest_sift_select, "selftest_sift_select",
                              {k: (t, int(np.prod(s))) for k, (t, s) in shapes.items()}, _ptr(rec), _ptr(kc), B, kcap, int(n_features),
                              int(cap), float(sentinel))
        res = {k: out[k].reshape(s) for k, (_, s) in shapes.items()}
        res.update({k + "_tail": v for k, v in tail.items()})
        return res

    def sift_desc(self, gauss, L: int, rows: np.ndarray, octave: np.ndarray, counts, cap: int, sentinel: float = -777.0):
        """sift.desc through its launch helper (dimb_selftest_sift_desc) on Gaussian levels (per octave [L + 3][B][h][w]) at output rows
        rows [B][n][4] (x, y, size, angle), octave [B][n] (output packing), counts [B].  Returns (desc [B][128][cap], tail)."""
        lv, B, n_oct, h, w = self._sift_levels(gauss)
        rows = np.ascontiguousarray(rows, np.float32)
        octave = np.ascontiguousarray(octave, np.int32)
        cnt = np.ascontiguousarray(counts, np.int32)
        n = rows.shape[1]
        out, tail = self._run(self.lib.dimb_selftest_sift_desc, "selftest_sift_desc", {"desc": (np.float32, B * 128 * cap)}, _ptr(lv), B,
                              L, n_oct, _ptr(h), _ptr(w), _ptr(rows), _ptr(octave), _ptr(cnt), int(n), int(cap), float(sentinel))
        return out["desc"].reshape(B, 128, cap), tail["desc"]

    @staticmethod
    def _f32(a):
        return None if a is None else np.ascontiguousarray(a, np.float32)

    def aliked_conv3x3(self, x, w, alpha=None, beta=None, resid=None, act=0, variant=0, sentinel: float = -777.0):
        """ALIKED's conv3 through its launch helper (dimb_selftest_aliked_conv3x3): x [cin][H][W], w [cout][cin][3][3], alpha / beta
        [cout], resid [cout][H][W].  variant 0 = the production rule, 1 / 2 / 3 = <8,1> / <16,4> / <8,4>.  Returns (out [cout][H][W],
        tail, the instantiation that ran)."""
        x, w, alpha, beta, resid = (self._f32(a) for a in (x, w, alpha, beta, resid))
        cin, H, W = x.shape
        cout = w.shape[0]
        plan = np.zeros(1, np.int32)
        out, tail = self._run(lambda h, *p: self.lib.dimb_selftest_aliked_conv3x3(h, int(variant), _ptr(x), cin, H, W, _ptr(w), *p, _ptr(plan)),
                              "selftest_aliked_conv3x3", {"out": (np.float32, cout * H * W)},
                              *(None if a is None else _ptr(a) for a in (alpha, beta, resid)), cout, int(act), float(sentinel))
        return out["out"].reshape(cout, H, W), tail["out"], int(plan[0])

    def aliked_conv1x1(self, x, w, bias=None, act=0, sentinel: float = -777.0):
        """ALIKED's conv1 (dimb_selftest_aliked_conv1x1): x [cin][P], w [cout][cin], bias [cout] -> (out [cout][P], tail)."""
        x, w, bias = self._f32(x), self._f32(w), self._f32(bias)
        cin, P = x.shape
        cout = w.shape[0]
        out, tail = self._run(self.lib.dimb_selftest_aliked_conv1x1, "selftest_aliked_conv1x1", {"out": (np.float32, cout * P)}, _ptr(x), cin,
                              P, _ptr(w), None if bias is None else _ptr(bias), cout, int(act), float(sentinel))
        return out["out"].reshape(cout, P), tail["out"]

    def aliked_avgpool(self, x, k: int, sentinel: float = -777.0):
        """al_avgpool_kernel (dimb_selftest_aliked_avgpool): x [C][H][W] -> (out [C][H // k][W // k], tail)."""
        x = self._f32(x)
        C_, H, W = x.shape
        n = C_ * (H // k) * (W // k)
        out, tail = self._run(self.lib.dimb_selftest_aliked_avgpool, "selftest_aliked_avgpool", {"out": (np.float32, n)}, _ptr(x), C_, H, W,
                              int(k), float(sentinel))
        return out["out"].reshape(C_, H // k, W // k), tail["out"]

    def aliked_pad(self, img, sentinel: float = -777.0):
        """InputPadder + al_pad_kernel (dimb_selftest_aliked_pad): img [H][W] or [H][W][3] 0..255 -> (out [3][Hp][Wp], (Hp, Wp, top,
        left), the rest of the buffer)."""
        img = self._f32(img)
        H, W = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        n = 3 * (H + 31) * (W + 31)
        raw = np.zeros(n + DET_TAIL, np.float32)
        geo = np.zeros(4, np.int32)
        self.check(self.lib.dimb_selftest_aliked_pad(self.h, _ptr(img), H, W, ch, float(sentinel), _ptr(raw), _ptr(geo)), "selftest_aliked_pad")
        Hp, Wp, top, left = (int(v) for v in geo)
        return raw[:3 * Hp * Wp].reshape(3, Hp, Wp), (Hp, Wp, top, left), raw[3 * Hp * Wp:]

    def aliked_crop(self, x, top: int, left: int, H: int, W: int, sentinel: float = -777.0):
        """al_crop_kernel (dimb_selftest_aliked_crop): x [Hp][Wp] -> (out [H][W], tail)."""
        x = self._f32(x)
        Hp, Wp = x.shape
        out, tail = self._run(self.lib.dimb_selftest_aliked_crop, "selftest_aliked_crop", {"out": (np.float32, H * W)}, _ptr(x), Hp, Wp,
                              int(top), int(left), int(H), int(W), float(sentinel))
        return out["out"].reshape(H, W), tail["out"]

    def aliked_deform(self, x, w, bn, offs=None, max_off: float = 0.0, offw=None, offb=None, resid=None, act=1, sentinel: float = -777.0):
        """ALIKED's deformable conv (dimb_selftest_aliked_deform): x [cin][H][W], w [cout][cin][3][3], bn [4][cout] (gamma, beta, mean,
        var).  Mode A: offs [18][H][W] clamped to +-max_off.  Mode B (offs None): offset_conv offw [18][cin][3][3], offb [18].  Returns
        (out [cout][H][W], tail, offsets [18][H][W] of mode B or None)."""
        x, w, bn, offs, offw, offb, resid = (self._f32(a) for a in (x, w, bn, offs, offw, offb, resid))
        cin, H, W = x.shape
        cout = w.shape[0]
        bufs = {"out": (np.float32, cout * H * W), "off": (np.float32, 18 * H * W)}
        p = lambda a: None if a is None else _ptr(a)
        out, tail = self._run(self.lib.dimb_selftest_aliked_deform, "selftest_aliked_deform", bufs, _ptr(x), cin, H, W, p(offs),
                              float(max_off), p(offw), p(offb), _ptr(w), _ptr(bn), p(resid), cout, int(act), float(sentinel))
        return out["out"].reshape(cout, H, W), tail["out"], None if offs is not None else out["off"].reshape(18, H, W)

    def aliked_fuse(self, x1, l2o, l3o, l4o, l1, s0, top: int, left: int, H: int, W: int, sentinel: float = -777.0):
        """al_fuse_kernel (dimb_selftest_aliked_fuse): x1 [16][Hp][Wp], lateral outputs l2o / l3o / l4o [32][Hp/f][Wp/f] (f = 2, 8, 32),
        conv1.weight l1 [32][16], score_head.0.weight s0 [8][128].  Returns (sh0 [8][Hp][Wp], feat [H][W][128], {'sh0', 'feat'} tails)."""
        x1, l2o, l3o, l4o, l1, s0 = (self._f32(a) for a in (x1, l2o, l3o, l4o, l1, s0))
        Hp, Wp = x1.shape[1:]
        out, tail = self._run(self.lib.dimb_selftest_aliked_fuse, "selftest_aliked_fuse",
                              {"sh0": (np.float32, 8 * Hp * Wp), "feat": (np.float32, H * W * 128)}, _ptr(x1), _ptr(l2o), _ptr(l3o),
                              _ptr(l4o), _ptr(l1), _ptr(s0), Hp, Wp, int(top), int(left), int(H), int(W), float(sentinel))
        return out["sh0"].reshape(8, Hp, Wp), out["feat"].reshape(H, W, 128), tail

    def aliked_dkd(self, score, r: int, sel_idx, count: int, cap: int, sentinel: float = -777.0):
        """al_dkd_refine_kernel (dimb_selftest_aliked_dkd) on score [H][W] at pixels sel_idx.  Returns ({'kxy' [cap][2], 'disp' [cap],
        'kscore' [cap]}, tails)."""
        score = self._f32(score)
        H, W = score.shape
        idx = np.ascontiguousarray(np.asarray(sel_idx, np.int64).astype(np.int32).reshape(-1))
        idx = idx if idx.size else np.zeros(1, np.int32)
        out, tail = self._run(self.lib.dimb_selftest_aliked_dkd, "selftest_aliked_dkd",
                              {"kxy": (np.float32, 2 * cap), "disp": (np.float32, cap), "kscore": (np.float32, cap)}, _ptr(score), H, W,
                              int(r), _ptr(idx), int(count), int(cap), float(sentinel))
        out["kxy"] = out["kxy"].reshape(cap, 2)
        return out, tail

    def aliked_sddh(self, feat, kxy, count: int, cap: int, w: dict, off=None, sentinel: float = -777.0):
        """SDDH (dimb_selftest_aliked_sddh) in the context's precision: feat [H][W][128], kxy [n][2] normalised, w the state_dict
        (desc_head.*), off [n][32] replacing the offsets stage's for the samples.  Returns ({'kpts' [cap][2], 'off' [cap][32], 'desc'
        [128][cap]}, tails)."""
        feat = self._f32(feat)
        H, W = feat.shape[:2]
        kxy = self._f32(np.asarray(kxy).reshape(-1, 2) if len(kxy) else np.zeros((1, 2)))
        off = self._f32(off)
        ws = [self._f32(w["desc_head." + k]) for k in ("offset_conv.0.weight", "offset_conv.0.bias", "offset_conv.2.weight",
                                                     "offset_conv.2.bias", "sf_conv.weight", "agg_weights")]
        out, tail = self._run(self.lib.dimb_selftest_aliked_sddh, "selftest_aliked_sddh",
                              {"kpts": (np.float32, 2 * cap), "off": (np.float32, 32 * cap), "desc": (np.float32, 128 * cap)}, _ptr(feat),
                              H, W, _ptr(kxy), int(count), int(cap), *(_ptr(a) for a in ws), None if off is None else _ptr(off),
                              float(sentinel))
        out["kpts"], out["off"], out["desc"] = out["kpts"].reshape(cap, 2), out["off"].reshape(cap, 32), out["desc"].reshape(128, cap)
        return out, tail

    def aliked_threshold(self, score, cand_count=None, thr: float = 0.0, sentinel: float = -777.0):
        """al_threshold_kernel (dimb_selftest_aliked_threshold): score [HW]; cand_count None = mean mode.  Returns (thr, tail)."""
        score = self._f32(np.asarray(score).reshape(-1))
        cc = None if cand_count is None else np.array([cand_count], np.int32)
        out, tail = self._run(self.lib.dimb_selftest_aliked_threshold, "selftest_aliked_threshold", {"thr": (np.float32, 1)}, _ptr(score),
                              score.size, None if cc is None else _ptr(cc), float(thr), float(sentinel))
        return out["thr"][0], tail["thr"]

    def nn_stats(self, f0: list, f1: list, D: int, mode: str, split: bool, host_counts: bool, sentinel: float = -777.0) -> dict:
        """The NN engine's row statistics (dimb_selftest_nn_stats): prep, then top-2 GEMM and merge of both directions, on the device
        sides f0 / f1 (lists of FeatsDev, as nn_match_batch_dev takes them).  split: three MMAs per product, else one; host_counts:
        the host-count engine of nn_match_dev (one pair, n_cap rows).  Returns n_live [2P], d1 / d2 / i1 [2P][NPp] (side 2p: the
        forward rows of pair p, side 2p + 1 its backward rows), plan [2][5] (the top-2 GEMM plan of each direction as gemm_plan gives
        it), NPp, and '<name>_tail' of every buffer."""
        P = len(f0)
        NPp = max(-(-max(f.n_cap for f in list(f0) + list(f1)) // 128) * 128, 128)
        R = 2 * P * NPp
        bufs = {"n_live": (np.int32, 2 * P), "d1": (np.float32, R), "d2": (np.float32, R), "i1": (np.int32, R), "plan": (np.int32, 10)}
        out, tail = self._run(self.lib.dimb_selftest_nn_stats, "selftest_nn_stats", bufs, P, (FeatsDev * P)(*f0), (FeatsDev * P)(*f1),
                              int(D), NN_MODES[mode], int(bool(split)), int(bool(host_counts)), NPp, float(sentinel))
        res = {k: out[k].reshape(2 * P, NPp) for k in ("d1", "d2", "i1")}
        res.update(n_live=out["n_live"], plan=out["plan"].reshape(2, 5), NPp=NPp)
        res.update({k + "_tail": v for k, v in tail.items() if k != "plan"})
        return res

    def nn_select(self, mode: str, th: float, n_live, d1: np.ndarray, d2: np.ndarray, i1: np.ndarray, cap: int,
                  sentinel: float = -777.0) -> dict:
        """nn_select_kernel (dimb_selftest_nn_select) on planted row statistics: n_live [2P], d1 / d2 / i1 [2P][NPp] as nn_stats
        returns them.  Returns idx [P][cap][2], dist [P][cap], count [P] (the full count) and '<name>_tail' of each."""
        d1, d2 = np.ascontiguousarray(d1, np.float32), np.ascontiguousarray(d2, np.float32)
        i1, nl = np.ascontiguousarray(i1, np.int32), np.ascontiguousarray(n_live, np.int32)
        S, NPp = d1.shape
        P = S // 2
        bufs = {"idx": (np.int64, P * cap * 2), "dist": (np.float32, P * cap), "count": (np.int32, P)}
        out, tail = self._run(self.lib.dimb_selftest_nn_select, "selftest_nn_select", bufs, NN_MODES[mode], float(th), P, NPp, _ptr(nl),
                              _ptr(d1), _ptr(d2), _ptr(i1), int(cap), float(sentinel))
        res = {"idx": out["idx"].reshape(P, cap, 2), "dist": out["dist"].reshape(P, cap), "count": out["count"]}
        res.update({k + "_tail": v for k, v in tail.items()})
        return res

    def lg_assign(self, sim: np.ndarray, nf, n_orig, layer, indf: np.ndarray, z: np.ndarray, th: float, cap: int,
                  sentinel: float = -777.0) -> dict:
        """The LightGlue assignment through its launch helper (dimb_selftest_lg_assign).  sim [P][NP][NP] (NP a multiple of 128),
        nf / n_orig [2P], layer [P], indf / z [2P][NP] (z = logsigmoid(matchability)).  Returns rmax / rlog / best / arg0 (rows, side
        2p), cmax / clog / arg1 (columns, side 2p + 1), best_other (the best buffer at side 2p + 1, which nothing writes), each [P][NP],
        matches [P][cap][2], mscores [P][cap], n_matches / stop_layer [P], and '<name>_tail' of every buffer."""
        sim = np.ascontiguousarray(sim, np.float32)
        P, NP, _ = sim.shape
        R = 2 * P * NP
        bufs = {"smax": (np.float32, R), "slog": (np.float32, R), "best": (np.float32, R), "arg": (np.int32, R),
                "matches": (np.int64, 2 * P * cap), "mscores": (np.float32, P * cap), "n_matches": (np.int32, P),
                "stop_layer": (np.int32, P)}
        ins = [np.ascontiguousarray(a, t) for a, t in ((nf, np.int32), (n_orig, np.int32), (layer, np.int32), (indf, np.int32),
                                                        (z, np.float32))]
        o, tail = self._run(self.lib.dimb_selftest_lg_assign, "selftest_lg_assign", bufs, P, NP, _ptr(sim), *(_ptr(a) for a in ins),
                            float(th), int(cap), float(sentinel))
        side = {k: o[k].reshape(P, 2, NP) for k in ("smax", "slog", "best", "arg")}
        out = {"rmax": side["smax"][:, 0], "rlog": side["slog"][:, 0], "best": side["best"][:, 0], "arg0": side["arg"][:, 0],
               "cmax": side["smax"][:, 1], "clog": side["slog"][:, 1], "best_other": side["best"][:, 1], "arg1": side["arg"][:, 1],
               "matches": o["matches"].reshape(P, cap, 2), "mscores": o["mscores"].reshape(P, cap), "n_matches": o["n_matches"],
               "stop_layer": o["stop_layer"]}
        out.update({k + "_tail": v for k, v in tail.items()})
        return out

    def lg_tail(self, P: int, NP: int, n_act, n_orig, stopped, counter, layer: int, thr: float, depth_conf: float, keep_thr: float,
                do_stop: bool, do_prune: bool, prune_min: int, x32=None, wt=None, bt: float = 0.0, wm=None, bm: float = 0.0, tok=None,
                mat=None, sentinel: float = -777.0) -> dict:
        """The LightGlue per-layer tail (dimb_selftest_lg_tail): from tokens x32 [2P * NP][256] with the confidence / matchability
        weights (lg_conf_kernel, then lg_decide_kernel), or, with x32 None, lg_decide_kernel alone on the given tok / mat [2P * NP].
        n_act / n_orig [2P], stopped / counter [P]: the state before.  Returns tok, mat, map [2P][NP], n_next [2P], counter and
        stopped [P] after the call, and '<name>_tail' of every buffer."""
        R = 2 * P * NP
        f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        x32, wt, wm, tok, mat = f32(x32), f32(wt), f32(wm), f32(tok), f32(mat)
        ptr = lambda a: None if a is None else _ptr(a)
        ins = [np.ascontiguousarray(a, np.int32) for a in (n_act, n_orig, stopped, counter)]
        bufs = {"tok": (np.float32, R), "mat": (np.float32, R), "counter": (np.int32, P), "stopped": (np.int32, P), "map": (np.int32, R),
                "n_next": (np.int32, 2 * P)}
        o, tail = self._run(self.lib.dimb_selftest_lg_tail, "selftest_lg_tail", bufs, int(P), int(NP), ptr(x32), ptr(wt), float(bt),
                            ptr(wm), float(bm), ptr(tok), ptr(mat), *(_ptr(a) for a in ins), int(layer), float(thr), float(depth_conf),
                            float(keep_thr), int(bool(do_stop)), int(bool(do_prune)), int(prune_min), float(sentinel))
        out = {k: o[k].reshape(2 * P, NP) if k in ("tok", "mat", "map") else o[k] for k in o}
        out.update({k + "_tail": v for k, v in tail.items()})
        return out

    def lgx_assign(self, sim: np.ndarray, z0, z1, ind0, ind1, th: float, cap: int, sentinel: float = -777.0) -> dict:
        """The shape-generic LightGlue assignment of one pair (dimb_selftest_lgx_assign): sim [m][ld] (live columns n = len(z1)), raw
        matchability logits z0 [m] / z1 [n], original indices ind0 / ind1.  Returns rlse, ls0, best0, arg0 [m], clse, ls1, best1,
        arg1 [n], matches [cap][2], mscores [cap], n_matches, and '<name>_tail' of every buffer."""
        sim = np.ascontiguousarray(sim, np.float32)
        z0, z1 = np.ascontiguousarray(z0, np.float32), np.ascontiguousarray(z1, np.float32)
        i0, i1 = np.ascontiguousarray(ind0, np.int32), np.ascontiguousarray(ind1, np.int32)
        m, n, ld = len(z0), len(z1), sim.shape[1]
        bufs = {"rlse": (np.float32, m), "clse": (np.float32, n), "ls0": (np.float32, m), "ls1": (np.float32, n),
                "best0": (np.float32, m), "arg0": (np.int32, m), "best1": (np.float32, n), "arg1": (np.int32, n),
                "matches": (np.int64, 2 * cap), "mscores": (np.float32, cap), "n_matches": (np.int32, 1)}
        o, tail = self._run(self.lib.dimb_selftest_lgx_assign, "selftest_lgx_assign", bufs, m, n, ld, _ptr(sim), _ptr(z0), _ptr(z1),
                            _ptr(i0), _ptr(i1), float(th), int(cap), float(sentinel))
        o["matches"] = o["matches"].reshape(cap, 2)
        o["n_matches"] = int(o["n_matches"][0])
        o.update({k + "_tail": v for k, v in tail.items() if k != "n_matches"})
        return o

    def sg_sinkhorn(self, scores: list, alpha: float, wave: int = 1, half_steps: int = 200, th: float = 0.2, cap: int | None = None,
                    u=None, v=None, pad: float = 1e6, sentinel: float = -777.0) -> dict:
        """SuperGlue's Sinkhorn and matching through their launch helpers (dimb_selftest_sg_sinkhorn).  scores: P float32 blocks
        [m_p][n_p]; the device layout is [P][NPt][NPt], NPt = max(m, n, 1) rounded up to 128, padding `pad`.  u / v [P][NPt + 1] or
        None (zeros): the duals before the first half step.  Returns NPt, pc [P][4], u / v [P][NPt + 1], best0 / arg0 / arg1 [P][NPt],
        matches [P][cap][2], mscores [P][cap], n_matches [P], and '<name>_tail' of every buffer."""
        P = len(scores)
        m = np.array([s.shape[0] for s in scores], np.int32)
        n = np.array([s.shape[1] for s in scores], np.int32)
        NPt = -(-max(int(m.max()), int(n.max()), 1) // 128) * 128
        cap = int(cap if cap is not None else max(int(m.max()), 1))
        flat = np.ascontiguousarray(np.concatenate([np.asarray(s, np.float32).reshape(-1) for s in scores] + [np.zeros(1, np.float32)]))
        uv = [None if a is None else np.ascontiguousarray(a, np.float32).reshape(P * (NPt + 1)) for a in (u, v)]
        bufs = {"pc": (np.float32, 4 * P), "u": (np.float32, P * (NPt + 1)), "v": (np.float32, P * (NPt + 1)),
                "best0": (np.float32, P * NPt), "arg0": (np.int32, P * NPt), "arg1": (np.int32, P * NPt),
                "matches": (np.int64, 2 * P * cap), "mscores": (np.float32, P * cap), "n_matches": (np.int32, P)}
        o, tail = self._run(self.lib.dimb_selftest_sg_sinkhorn, "selftest_sg_sinkhorn", bufs, P, _ptr(m), _ptr(n), _ptr(flat), float(alpha),
                            float(pad), None if uv[0] is None else _ptr(uv[0]), None if uv[1] is None else _ptr(uv[1]), int(wave),
                            int(half_steps), float(th), cap, float(sentinel))
        shapes = {"pc": (P, 4), "u": (P, NPt + 1), "v": (P, NPt + 1), "best0": (P, NPt), "arg0": (P, NPt), "arg1": (P, NPt),
                  "matches": (P, cap, 2), "mscores": (P, cap)}
        out = {k: o[k].reshape(shapes[k]) if k in shapes else o[k] for k in o}
        out["NPt"] = NPt
        out.update({k + "_tail": v for k, v in tail.items()})
        return out

    def __del__(self):
        try:
            self.lib.dimb_ctx_destroy(self.h)
        except Exception:
            pass


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _int_array(values):
    a = np.ascontiguousarray(np.asarray(values, np.int64).astype(np.int32).reshape(-1))
    return a, _ptr(a) if a.size else None


def tile_grid(height: int, width: int, tile_h: int, tile_w: int, overlap_h: int, overlap_w: int) -> dict:
    """The tile grid the library cuts (dimb_tile_grid, no GPU needed): n_rows, n_cols, pad_top, pad_left, stride_h, stride_w and
    the (x, y) origin of every tile in the un-padded image (tiling.compute_tiles_by_size's geometry, row-major)."""
    out = np.zeros(6, np.int32)
    rc = load_library().dimb_tile_grid(int(height), int(width), int(tile_h), int(tile_w), int(overlap_h), int(overlap_w), _ptr(out))
    if rc != OK:
        raise ValueError(f"invalid tile geometry: image {height}x{width}, tile {tile_h}x{tile_w}, overlap {overlap_h}x{overlap_w} "
                         "(need 0 <= overlap < tile and at most 2048 tiles)")
    rows, cols, pt, pl, sh, sw = (int(v) for v in out)
    origins = [(-pl + c * sw, -pt + r * sh) for r in range(rows) for c in range(cols)]
    return {"n_rows": rows, "n_cols": cols, "pad_top": pt, "pad_left": pl, "stride_h": sh, "stride_w": sw, "origins": origins}


def resize_area_tab(ssize: int, dsize: int):
    """The INTER_AREA table of one axis that dimb_resize_area_dev uses (dimb_resize_area_tab, no GPU needed): (d_idx int32, s_idx
    int32, alpha float32), one entry per (destination, source) contribution in OpenCV's order."""
    lib, cap, n = load_library(), 2 * max(int(ssize), 1), C.c_int()
    di, si, al = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.float32)
    if lib.dimb_resize_area_tab(int(ssize), int(dsize), _ptr(di), _ptr(si), _ptr(al), cap, C.byref(n)) != OK:
        raise ValueError(f"INTER_AREA downscaling needs 1 <= dsize <= ssize, got ssize {ssize}, dsize {dsize}")
    return di[:n.value].copy(), si[:n.value].copy(), al[:n.value].copy()


def resize_area_linear_tab(ssize: int, dsize: int):
    """The coefficients of one axis that dimb_resize_area_linear_dev uses when INTER_AREA enlarges (dimb_resize_area_linear_tab, no
    GPU needed): (s_idx int32 (dsize,), alpha float32 (dsize, 2), xmax)."""
    si, al, xmax = np.zeros(max(int(dsize), 1), np.int32), np.zeros((max(int(dsize), 1), 2), np.float32), C.c_int()
    if load_library().dimb_resize_area_linear_tab(int(ssize), int(dsize), _ptr(si), _ptr(al), C.byref(xmax)) != OK:
        raise ValueError(f"INTER_AREA coefficients need sizes >= 1, got ssize {ssize}, dsize {dsize}")
    return si, al, int(xmax.value)


def pyr_size(height: int, width: int, level: int):
    """(H2, W2) of an image after `level` pyramid steps (dimb_pyr_size, no GPU needed): -1 one cv2.pyrUp, 0 none, 1..3 that many
    cv2.pyrDown."""
    h2, w2 = C.c_int(), C.c_int()
    if load_library().dimb_pyr_size(int(height), int(width), int(level), C.byref(h2), C.byref(w2)) != OK:
        raise ValueError(f"pyramid steps need a level in [-1, 3] and sizes in [1, 2^20], got {height}x{width}, level {level}")
    return h2.value, w2.value


class Context:
    """One per device (dimb_ctx). precision: "exact" (fp16 hi/lo split, fp32-class) or "fast" (plain fp16)."""

    _per_device: dict = {}

    def __init__(self, device: int = 0, precision: str | None = None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.dimb_ctx_create(device, C.byref(h))
        if rc != OK:
            raise DimbError(f"dimb_ctx_create(device={device}) failed with code {rc}: a CUDA device of compute "
                            "capability 9.x (H100, sm_90a) is required; there is no CPU fallback")
        self.h = h
        self.device = device
        if precision is not None:
            self.set_precision(precision)

    @classmethod
    def get(cls, device: int = 0) -> "Context":
        if device not in cls._per_device:
            cls._per_device[device] = cls(device)
        return cls._per_device[device]

    def check(self, rc: int, what: str):
        if rc != OK:
            msg = self.lib.dimb_last_error(self.h).decode()
            raise DimbError(f"{what} failed (code {rc}): {msg}")

    def set_precision(self, precision: str):
        self.check(self.lib.dimb_ctx_set_precision(self.h, {"exact": 0, "fast": 1}[precision]), "set_precision")

    @property
    def launches(self) -> int:
        return int(self.lib.dimb_ctx_launch_count(self.h))

    def profile(self, enable: bool):
        self.check(self.lib.dimb_ctx_profile(self.h, int(bool(enable))), "dimb_ctx_profile")

    def profile_read(self) -> dict:
        """{"group": [total_ms, launches]} of the kernel groups recorded since profile(True)."""
        import json
        buf = C.create_string_buffer(1 << 16)
        self.check(self.lib.dimb_ctx_profile_read(self.h, buf, len(buf)), "dimb_ctx_profile_read")
        return json.loads(buf.value.decode())

    def nn_match(self, desc0: np.ndarray, desc1: np.ndarray, mode: str = "smnn", th: float = 0.8):
        """desc0 (D,n0), desc1 (D,n1) float32 -> (int64 (S,2), float32 (S,))."""
        d0 = np.ascontiguousarray(desc0, np.float32)
        d1 = np.ascontiguousarray(desc1, np.float32)
        D, n0 = d0.shape
        n1 = d1.shape[1]
        cap = max(n0, n1, 1)
        idx = np.zeros((cap, 2), np.int64)
        dist = np.zeros(cap, np.float32)
        n = C.c_int(0)
        self.check(self.lib.dimb_nn_match(self.h, _ptr(d0), n0, _ptr(d1), n1, D, NN_MODES[mode], float(th), _ptr(idx),
                                          _ptr(dist), C.byref(n), cap), "dimb_nn_match")
        return idx[: n.value].copy(), dist[: n.value].copy()

    def gv_fundamental(self, kpts0: np.ndarray, kpts1: np.ndarray, threshold: float = 1.0, max_iters: int = 10000, seed: int = 0):
        """Matched keypoints (n,2) each -> (F (3,3) float32 or None, inlier mask bool (n,))."""
        k0 = np.ascontiguousarray(kpts0, np.float32)
        k1 = np.ascontiguousarray(kpts1, np.float32)
        n = k0.shape[0]
        F = np.zeros(9, np.float32)
        mask = np.ones(max(n, 1), np.uint8)
        cnt = C.c_int(0)
        self.check(self.lib.dimb_gv_fundamental(self.h, _ptr(k0), _ptr(k1), n, float(threshold), int(max_iters), int(seed) & 0xffffffff, _ptr(F),
                                                _ptr(mask), C.byref(cnt)), "dimb_gv_fundamental")
        return (F.reshape(3, 3) if np.any(F) else None), mask[:n].astype(bool)

    def gv_estimate(self, kpts0: np.ndarray, kpts1: np.ndarray, threshold: float = 1.0, max_iters: int = 10000, seed: int = 0,
                    estimator: str = "ransac8", confidence: float = 0.9999):
        """Matched keypoints (n,2) each -> (F (3,3) float32 or None, inlier mask bool (n,), hypotheses run) with the named estimator
        (dimb_gv_estimate; ``confidence`` is read by lo-ransac and degensac only)."""
        k0 = np.ascontiguousarray(kpts0, np.float32)
        k1 = np.ascontiguousarray(kpts1, np.float32)
        n = k0.shape[0]
        F = np.zeros(9, np.float32)
        mask = np.ones(max(n, 1), np.uint8)
        cnt, hyp = C.c_int(0), C.c_int(0)
        conf = GvConf(float(threshold), int(max_iters), 0, 0.0, gv_estimator(estimator), float(confidence))
        self.check(self.lib.dimb_gv_estimate(self.h, _ptr(k0), _ptr(k1), n, C.byref(conf), int(seed) & 0xffffffff, _ptr(F), _ptr(mask),
                                             C.byref(cnt), C.byref(hyp)), "dimb_gv_estimate")
        return (F.reshape(3, 3) if np.any(F) else None), mask[:n].astype(bool), hyp.value

    def gv_verify_dev(self, f0: list, f1: list, d_matches, d_n_matches, cap, seeds, threshold=1.0, max_iters=10000, min_inliers=0,
                      min_inlier_ratio=0.0, d_verified=0, d_n_verified=0, d_F=0, d_mask=0, d_n_inliers=0, stream=0, estimator="ransac8",
                      confidence=0.9999):
        """Geometric verification of P match tables on the device (dimb_gv_verify_dev).  f0/f1: lists of FeatsDev (e.g.
        FeatureStoreDev.feats_dev); d_matches [P][cap][2] int64 / d_n_matches [P] int32 as LightGlueNet.match_dev writes them; seeds:
        one uint32 per pair (geometric_verification.gv_seed).  Outputs are device buffers (ints are device addresses): d_verified
        [P][cap][2] int64, d_n_verified [P] int32, d_F [P][9] float32, d_mask [P][cap] uint8, d_n_inliers [P] int32.  Asynchronous
        on `stream`.  estimator: a name in GV_ESTIMATORS; confidence is read by lo-ransac and degensac only."""
        P = len(f0)
        a0 = (FeatsDev * P)(*f0)
        a1 = (FeatsDev * P)(*f1)
        sd = (C.c_uint * P)(*[int(s) & 0xffffffff for s in seeds])
        conf = GvConf(float(threshold), int(max_iters), int(min_inliers), float(min_inlier_ratio), gv_estimator(estimator), float(confidence))
        self.check(self.lib.dimb_gv_verify_dev(self.h, P, a0, a1, d_matches, d_n_matches, cap, sd, C.byref(conf), d_verified, d_n_verified,
                                               d_F, d_mask, d_n_inliers, stream), "dimb_gv_verify_dev")

    def tile_cut_dev(self, d_images, B, H, W, channels, tile_h, tile_w, overlap_h, overlap_w, d_tiles, stream=0):
        """B float32 (H,W,channels) device images -> their tiles [B*T][tile_h][tile_w][channels] (dimb_tile_cut_dev; ints are device
        addresses); asynchronous on `stream`."""
        self.check(self.lib.dimb_tile_cut_dev(self.h, d_images, B, H, W, channels, tile_h, tile_w, overlap_h, overlap_w, d_tiles, stream),
                   "dimb_tile_cut_dev")

    def tile_match_merge_dev(self, pair_offsets, view0, view1, d_maps, map_ld, d_matches, d_n_matches, cap, d_out, d_n_out, cap2, stream=0):
        """Tile-pair match tables -> de-duplicated image-pair tables in merged rows (dimb_tile_match_merge_dev).  pair_offsets: host
        CSR [Q+1] over the tile pairs; view0 / view1: the map rows of both sides of every tile pair.  Asynchronous on `stream`."""
        off, p_off = _int_array(pair_offsets)
        v0, p0 = _int_array(view0)
        v1, p1 = _int_array(view1)
        self.check(self.lib.dimb_tile_match_merge_dev(self.h, len(off) - 1, p_off, p0, p1, d_maps, map_ld, d_matches, d_n_matches, cap, d_out,
                                                      d_n_out, cap2, stream), "dimb_tile_match_merge_dev")

    def resize_area_dev(self, d_src, B, H, W, d_dst, H2, W2, stream=0):
        """cv2.resize(INTER_AREA) of B float32 gray device images [B][H][W] -> [B][H2][W2], downscaling only (dimb_resize_area_dev);
        asynchronous on `stream`."""
        self.check(self.lib.dimb_resize_area_dev(self.h, d_src, B, H, W, d_dst, H2, W2, stream), "dimb_resize_area_dev")

    def resize_area_linear_dev(self, d_src, B, H, W, d_dst, H2, W2, stream=0):
        """cv2.resize(INTER_AREA) of B float32 gray device images [B][H][W] -> [B][H2][W2] when H2 > H or W2 > W, OpenCV's bilinear
        emulation (dimb_resize_area_linear_dev); asynchronous on `stream`."""
        self.check(self.lib.dimb_resize_area_linear_dev(self.h, d_src, B, H, W, d_dst, H2, W2, stream), "dimb_resize_area_linear_dev")

    def resize_area_rgb_dev(self, d_src, B, H, W, d_dst, H2, W2, stream=0):
        """cv2.resize(pairs_generator.gray_from_rgb(img), (W2, H2), interpolation=INTER_AREA) of B float32 RGB device images [B][H][W][3]
        -> gray [B][H2][W2], any size relation, the gray rule applied per source pixel as it is read (dimb_resize_area_rgb_dev);
        asynchronous on `stream`."""
        self.check(self.lib.dimb_resize_area_rgb_dev(self.h, d_src, B, H, W, d_dst, H2, W2, stream), "dimb_resize_area_rgb_dev")

    def pyr_dev(self, d_src, B, H, W, channels, level, d_dst, stream=0):
        """cv2.pyrDown `level` times (1..3) or cv2.pyrUp once (-1) of B float32 device images [B][H][W][channels], 1 or 3 channels,
        into d_dst [B][H2][W2][channels] (pyr_size), bitwise (dimb_pyr_dev); asynchronous on `stream`."""
        self.check(self.lib.dimb_pyr_dev(self.h, d_src, B, H, W, channels, level, d_dst, stream), "dimb_pyr_dev")

    def rot90_dev(self, d_src, B, H, W, channels, rotations, d_dst, stream=0):
        """cv2.rotate of B float32 device images [B][H][W][channels], 1 or 3 channels, by rotations[b] in (0, 90, 180, 270) degrees
        clockwise, into d_dst (image b at b * H * W * channels, (W, H) for 90 / 270), bitwise (dimb_rot90_dev); asynchronous on `stream`."""
        r, p = _int_array(rotations)
        if len(r) != B:
            raise ValueError(f"rot90_dev needs one rotation per image: {len(r)} for {B} images")
        self.check(self.lib.dimb_rot90_dev(self.h, d_src, B, H, W, channels, p, d_dst, stream), "dimb_rot90_dev")

    def kpts_extent_dev(self, B, d_kpts, kpt_ld, d_counts, d_size_out, stream=0):
        """Own-extent normalisation size (1 + max) - min per axis of B keypoint sets [B][kpt_ld][2] -> d_size_out [B][2] float32
        (dimb_kpts_extent_dev; FeatsDev.size_f32_dev takes one row); asynchronous on `stream`."""
        self.check(self.lib.dimb_kpts_extent_dev(self.h, B, d_kpts, kpt_ld, d_counts, d_size_out, stream), "dimb_kpts_extent_dev")

    def tile_preselect_dev(self, f0: list, f1: list, d_matches, d_n_matches, cap, H, W, tile_h, tile_w, overlap_h, overlap_w, scale0, scale1,
                           min_matches_per_tile, d_counts, d_flags, stream=0):
        """PRESELECTION's box count for len(f0) image pairs (dimb_tile_preselect_dev): low-resolution match tables [Q][cap][2] int64 over
        the keypoints of f0[q] / f1[q] (FeatsDev) -> d_counts [Q][T*T] int32 and d_flags [Q][T*T] uint8 (count > min_matches_per_tile).
        Asynchronous on `stream`."""
        Q = len(f0)
        a0 = (FeatsDev * Q)(*f0)
        a1 = (FeatsDev * Q)(*f1)
        self.check(self.lib.dimb_tile_preselect_dev(self.h, Q, a0, a1, d_matches, d_n_matches, cap, H, W, tile_h, tile_w, overlap_h, overlap_w,
                                                    float(scale0), float(scale1), int(min_matches_per_tile), d_counts, d_flags, stream),
                   "dimb_tile_preselect_dev")

    def tile_preselect_pairs_dev(self, f0: list, f1: list, d_matches, d_n_matches, cap, sizes, tile_h, tile_w, overlap_h, overlap_w, scales,
                                 min_matches_per_tile, d_counts, d_flags, stream=0):
        """PRESELECTION's box count for len(f0) image pairs of any sizes (dimb_tile_preselect_pairs_dev): sizes [(H0, W0, H1, W1)] and
        scales [(scale0, scale1)] per pair.  Pair q's counts (int32) and flags (uint8) are the row-major [T0][T1] block starting at
        element sum_{p<q} T0[p] * T1[p] of d_counts / d_flags.  Asynchronous on `stream`."""
        Q = len(f0)
        a0 = (FeatsDev * Q)(*f0)
        a1 = (FeatsDev * Q)(*f1)
        sz = np.ascontiguousarray(np.asarray(sizes, np.int64).reshape(-1, 4).astype(np.int32))
        sc = np.ascontiguousarray(np.asarray(scales, np.float64).reshape(-1, 2))
        if len(sz) != Q or len(sc) != Q:
            raise ValueError(f"tile_preselect_pairs_dev needs one size row and one scale row per pair: {len(sz)} / {len(sc)} for {Q} pairs")
        self.check(self.lib.dimb_tile_preselect_pairs_dev(self.h, Q, a0, a1, d_matches, d_n_matches, cap, _ptr(sz), tile_h, tile_w, overlap_h,
                                                          overlap_w, _ptr(sc), int(min_matches_per_tile), d_counts, d_flags, stream),
                   "dimb_tile_preselect_pairs_dev")

    def nn_match_dev(self, d_desc0: int, n0: int, d_desc1: int, n1: int, D: int, mode: str, th: float, d_idx: int, d_dist: int,
                     d_n: int, cap: int, f16: bool = False, ld0: int = 0, ld1: int = 0, stream: int = 0):
        """Device-pointer variant (ints are device addresses); asynchronous on `stream`."""
        self.check(self.lib.dimb_nn_match_dev(self.h, d_desc0, n0, ld0, d_desc1, n1, ld1, D, int(f16), NN_MODES[mode], float(th), d_idx,
                                              d_dist, d_n, cap, stream), "dimb_nn_match_dev")

    def nn_match_batch_dev(self, f0: list, f1: list, D: int, mode: str, th: float, d_idx: int, d_dist: int, d_n: int, cap: int,
                           stream: int = 0):
        """Brute-force NN matching of len(f0) pairs (dimb_nn_match_batch_dev): f0 / f1 are lists of FeatsDev (e.g.
        FeatureStoreDev.feats_dev) whose counts stay on the device.  Outputs are device buffers (ints are device addresses): d_idx
        [P][cap][2] int64, d_dist [P][cap] float32, d_n [P] int32 (the full count).  Asynchronous on `stream`."""
        P = len(f0)
        a0 = (FeatsDev * P)(*f0)
        a1 = (FeatsDev * P)(*f1)
        self.check(self.lib.dimb_nn_match_batch_dev(self.h, P, a0, a1, int(D), NN_MODES[mode], float(th), d_idx, d_dist, d_n, cap, stream),
                   "dimb_nn_match_batch_dev")


SP_ORDER = ["conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "conv4a", "conv4b", "convPa", "convPb",
            "convDa", "convDb"]


def pack_superpoint_weights(w: dict) -> np.ndarray:
    parts = []
    for name in SP_ORDER:
        parts += [np.asarray(w[name + ".weight"], np.float32).ravel(), np.asarray(w[name + ".bias"], np.float32).ravel()]
    return np.ascontiguousarray(np.concatenate(parts))


def lightglue_weight_names(input_dim: int, descriptor_dim: int, n_layers: int) -> list:
    names = ["posenc.Wr.weight"]
    if input_dim != descriptor_dim:
        names += ["input_proj.weight", "input_proj.bias"]
    for i in range(n_layers):
        p = f"transformers.{i}."
        for m in ("self_attn.Wqkv", "self_attn.out_proj", "self_attn.ffn.0", "self_attn.ffn.1", "self_attn.ffn.3",
                  "cross_attn.to_qk", "cross_attn.to_v", "cross_attn.to_out", "cross_attn.ffn.0", "cross_attn.ffn.1",
                  "cross_attn.ffn.3"):
            names += [p + m + ".weight", p + m + ".bias"]
    for i in range(n_layers):
        for m in ("matchability", "final_proj"):
            names += [f"log_assignment.{i}.{m}.weight", f"log_assignment.{i}.{m}.bias"]
    for i in range(n_layers - 1):
        names += [f"token_confidence.{i}.token.0.weight", f"token_confidence.{i}.token.0.bias"]
    return names


def pack_lightglue_weights(w: dict, input_dim: int, descriptor_dim: int, n_layers: int) -> np.ndarray:
    w = dict(w)
    for i in range(n_layers):  # old checkpoints: self_attn.i. / cross_attn.i. prefixes (lightglue.py:391-396)
        for blk in ("self_attn", "cross_attn"):
            for k in [k for k in w if k.startswith(f"{blk}.{i}.")]:
                w[k.replace(f"{blk}.{i}", f"transformers.{i}.{blk}", 1)] = w.pop(k)
    return np.ascontiguousarray(np.concatenate(
        [np.asarray(w[n], np.float32).ravel() for n in lightglue_weight_names(input_dim, descriptor_dim, n_layers)]))


class SuperPointNet:
    """Handle on dimb_sp: SuperPoint extraction of batches of equally sized gray images."""

    def __init__(self, ctx: Context, weights: dict, nms_radius=4, keypoint_threshold=0.005, max_keypoints=-1,
                 remove_borders=4, fix_sampling=False, max_batch=1, max_height=1024, max_width=1024):
        self.ctx = ctx
        if max_keypoints == 0 or max_keypoints < -1:
            raise ValueError('"max_keypoints" must be positive or "-1"')  # superpoint.py:152-154
        self.conf = SpConf(int(nms_radius), float(keypoint_threshold), int(max_keypoints), int(remove_borders),
                           int(bool(fix_sampling)), int(max_batch), int(max_height), int(max_width))
        blob = pack_superpoint_weights(weights)
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_sp_create(ctx.h, _ptr(blob), blob.size, C.byref(self.conf), C.byref(h)), "dimb_sp_create")
        self.h = h

    def default_cap(self, H, W):
        k = self.conf.max_keypoints
        return k if k > 0 else (H // 8 * 8) * (W // 8 * 8) // 4

    def extract(self, images: np.ndarray, cap: int | None = None):
        """images float32 (B,H,W) 0..255 -> list of dicts(keypoints (N,2), scores (N,), descriptors (256,N))."""
        images = np.ascontiguousarray(images, np.float32)
        B, H, W = images.shape
        cap = cap or self.default_cap(H, W)
        while True:
            kp = np.zeros((B, cap, 2), np.float32)
            sc = np.zeros((B, cap), np.float32)
            de = np.zeros((B, 256, cap), np.float32)
            cnt = np.zeros(B, np.int32)
            rc = self.ctx.lib.dimb_sp_extract(self.h, _ptr(images), B, H, W, _ptr(kp), _ptr(sc), _ptr(de), _ptr(cnt), cap)
            if rc == ERR_CAPACITY:
                cap = int(cnt.max())
                continue
            self.ctx.check(rc, "dimb_sp_extract")
            break
        return [{"keypoints": kp[b, : cnt[b]].copy(), "scores": sc[b, : cnt[b]].copy(),
                 "descriptors": de[b, :, : cnt[b]].copy()} for b in range(B)]

    def extract_dev(self, d_images, B, H, W, d_kpts, d_scores, d_desc, d_counts, cap, stream=0):
        """Raw device-pointer variant (ints are device addresses, e.g. torch.Tensor.data_ptr())."""
        self.ctx.check(self.ctx.lib.dimb_sp_extract_dev(self.h, d_images, B, H, W, d_kpts, d_scores, d_desc, d_counts, cap,
                                                        stream), "dimb_sp_extract_dev")

    def debug_read(self, which: int, shape) -> np.ndarray:
        out = np.zeros(shape, np.float32)
        self.ctx.check(self.ctx.lib.dimb_sp_debug_read(self.h, which, _ptr(out), out.size), "dimb_sp_debug_read")
        return out

    def __del__(self):
        try:
            self.ctx.lib.dimb_sp_destroy(self.h)
        except Exception:
            pass


def aliked_weight_names() -> list:
    """state_dict order of aliked-n16 / aliked-n16rot (thirdparty/LightGlue/lightglue/aliked.py:596-640), floats only."""
    names = []
    bn = lambda p: [p + s for s in (".weight", ".bias", ".running_mean", ".running_var")]
    names += ["block1.conv1.weight"] + bn("block1.bn1") + ["block1.conv2.weight"] + bn("block1.bn2")
    names += ["block2.conv1.weight"] + bn("block2.bn1") + ["block2.conv2.weight"] + bn("block2.bn2")
    names += ["block2.downsample.weight", "block2.downsample.bias"]
    for b in ("block3", "block4"):
        for c, n in (("conv1", "bn1"), ("conv2", "bn2")):
            names += [f"{b}.{c}.offset_conv.weight", f"{b}.{c}.offset_conv.bias", f"{b}.{c}.regular_conv.weight"] + bn(f"{b}.{n}")
        names += [f"{b}.downsample.weight", f"{b}.downsample.bias"]
    names += ["conv1.weight", "conv2.weight", "conv3.weight", "conv4.weight"]
    names += [f"score_head.{i}.weight" for i in (0, 2, 4, 6)]
    names += ["desc_head.agg_weights", "desc_head.offset_conv.0.weight", "desc_head.offset_conv.0.bias",
              "desc_head.offset_conv.2.weight", "desc_head.offset_conv.2.bias", "desc_head.sf_conv.weight"]
    return names


def pack_aliked_weights(w: dict) -> np.ndarray:
    return np.ascontiguousarray(np.concatenate([np.asarray(w[n], np.float32).ravel() for n in aliked_weight_names()]))


ALIKED_N_LIMIT = 20000  # the keypoint cut of ALIKED's threshold / mean modes when max_num_keypoints <= 0 (aliked.py:585)


class AlikedNet:
    """Handle on dimb_aliked: ALIKED-n16(rot) extraction of one image per call (the reference path is batch-1).  Detection modes as
    the LightGlue port's DKD: threshold (detection_threshold > 0), top-k (detection_threshold <= 0 < max_num_keypoints: exactly
    max_num_keypoints keypoints) and mean (both <= 0)."""

    def __init__(self, ctx: Context, weights: dict, max_num_keypoints=4000, detection_threshold=0.2, nms_radius=2,
                 max_height=1024, max_width=1024):
        self.ctx = ctx
        self.conf = AlikedConf(int(max_num_keypoints), float(detection_threshold), int(nms_radius), int(max_height), int(max_width))
        blob = pack_aliked_weights(weights)
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_aliked_create(ctx.h, _ptr(blob), blob.size, C.byref(self.conf), C.byref(h)), "dimb_aliked_create")
        self.h = h

    def extract(self, image: np.ndarray, cap: int | None = None) -> dict:
        """image float32 (H,W,3) RGB or (H,W) gray, 0..255 -> keypoints (N,2), scores (N,), descriptors (128,N)."""
        image = np.ascontiguousarray(image, np.float32)
        H, W = image.shape[:2]
        ch = 1 if image.ndim == 2 else image.shape[2]
        k = self.conf.max_num_keypoints
        cap = cap or (k if k > 0 else ALIKED_N_LIMIT)  # top-k mode returns exactly k, the other modes at most k (or n_limit)
        while True:
            kp = np.zeros((cap, 2), np.float32)
            sc = np.zeros(cap, np.float32)
            de = np.zeros((128, cap), np.float32)
            cnt = np.zeros(1, np.int32)
            rc = self.ctx.lib.dimb_aliked_extract(self.h, _ptr(image), H, W, ch, _ptr(kp), _ptr(sc), _ptr(de), _ptr(cnt), cap)
            if rc == ERR_CAPACITY:
                cap = int(cnt[0])
                continue
            self.ctx.check(rc, "dimb_aliked_extract")
            break
        n = int(cnt[0])
        return {"keypoints": kp[:n].copy(), "scores": sc[:n].copy(), "descriptors": de[:, :n].copy()}

    def extract_dev(self, d_image, H, W, channels, d_kpts, d_scores, d_desc, d_count, cap, stream=0):
        """Raw device-pointer variant (ints are device addresses, e.g. torch.Tensor.data_ptr())."""
        self.ctx.check(self.ctx.lib.dimb_aliked_extract_dev(self.h, d_image, H, W, channels, d_kpts, d_scores, d_desc, d_count, cap,
                                                            stream), "dimb_aliked_extract_dev")

    def debug_read(self, which: int, shape) -> np.ndarray:
        out = np.zeros(shape, np.float32)
        self.ctx.check(self.ctx.lib.dimb_aliked_debug_read(self.h, which, _ptr(out), out.size), "dimb_aliked_debug_read")
        return out

    def __del__(self):
        try:
            self.ctx.lib.dimb_aliked_destroy(self.h)
        except Exception:
            pass


def sift_octaves(height: int, width: int) -> list:
    """(h, w) of every octave of a SIFT pyramid, OpenCV's octave -1 (2H x 2W) first: cvRound(log2(min(2H, 2W)) - 2) + 1 octaves,
    each later one halving (floor) both sides."""
    n = int(np.rint(np.log(min(2 * height, 2 * width)) / np.log(2.0) - 2)) + 1
    sizes, h, w = [], 2 * height, 2 * width
    for o in range(n):
        if o:
            h, w = h // 2, w // 2
        sizes.append((h, w))
    return sizes


class SiftNet:
    """Handle on dimb_sift: cv2.SIFT_create(n_features, n_octave_layers, contrast_threshold, edge_threshold, sigma)
    .detectAndCompute on the device, for batches of equally sized gray images."""

    def __init__(self, ctx: Context, n_features=0, n_octave_layers=3, contrast_threshold=0.04, edge_threshold=10.0, sigma=1.6,
                 max_batch=1, max_height=1024, max_width=1024):
        self.ctx = ctx
        self.conf = SiftConf(int(n_features), int(n_octave_layers), float(contrast_threshold), float(edge_threshold), float(sigma),
                             int(max_batch), int(max_height), int(max_width))
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_sift_create(ctx.h, C.byref(self.conf), C.byref(h)), "dimb_sift_create")
        self.h = h

    def extract(self, image: np.ndarray, cap: int | None = None) -> dict:
        """image uint8 (H,W) -> keypoints (N,2), descriptors (128,N) float32 with integral 0..255 values, size / angle / response
        (N,) and octave (N,) int32 (cv2's packed KeyPoint.octave)."""
        image = np.ascontiguousarray(image)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("SiftNet.extract takes a uint8 (H, W) image")
        H, W = image.shape
        cap = cap or max(self.conf.n_features, 1) + 64
        while True:
            kp = np.zeros((cap, 2), np.float32)
            de = np.zeros((128, cap), np.float32)
            fr = np.zeros((cap, 3), np.float32)
            oc = np.zeros(cap, np.int32)
            cnt = np.zeros(1, np.int32)
            rc = self.ctx.lib.dimb_sift_extract(self.h, _ptr(image), H, W, _ptr(kp), _ptr(de), _ptr(fr), _ptr(oc), _ptr(cnt), cap)
            if rc == ERR_CAPACITY and cnt[0] > cap:
                cap = int(cnt[0])
                continue
            self.ctx.check(rc, "dimb_sift_extract")
            break
        n = int(cnt[0])
        return {"keypoints": kp[:n].copy(), "descriptors": de[:, :n].copy(), "size": fr[:n, 0].copy(), "angle": fr[:n, 1].copy(),
                "response": fr[:n, 2].copy(), "octave": oc[:n].copy()}

    def extract_dev(self, d_images, B, H, W, d_kpts, d_desc, d_counts, cap, d_frames=0, d_octave=0, stream=0):
        """Raw device-pointer variant (ints are device addresses, e.g. torch.Tensor.data_ptr())."""
        self.ctx.check(self.ctx.lib.dimb_sift_extract_dev(self.h, d_images, B, H, W, d_kpts, d_desc, d_frames or None,
                                                          d_octave or None, d_counts, cap, stream), "dimb_sift_extract_dev")

    def debug_read(self, which: int, image: int, octave: int, level: int, height: int, width: int) -> np.ndarray:
        """which 0: Gaussian level `level` of `octave`, 1: DoG level; (height, width) are the image's, the shape comes from
        sift_octaves."""
        h, w = sift_octaves(height, width)[octave]
        per = self.conf.n_octave_layers + 3 - which
        out = np.zeros((h, w), np.float32)
        self.ctx.check(self.ctx.lib.dimb_sift_debug_read(self.h, which, image, octave * per + level, _ptr(out), out.size),
                       "dimb_sift_debug_read")
        return out

    def __del__(self):
        try:
            self.ctx.lib.dimb_sift_destroy(self.h)
        except Exception:
            pass


def orb_level_sizes(height: int, width: int, nlevels: int, scale_factor: float) -> list:
    """(h, w) of every ORB pyramid level: cvRound(H / s), cvRound(W / s) in float, s = (float)pow(float(scaleFactor), level)."""
    sf = float(np.float32(scale_factor))
    out = []
    for level in range(nlevels):
        inv = np.float32(1) / np.float32(sf ** level)
        out.append((int(np.rint(np.float32(height) * inv)), int(np.rint(np.float32(width) * inv))))
    return out


class OrbNet:
    """Handle on dimb_orb: cv2.ORB_create(n_features, scale_factor, nlevels, edge_threshold, first_level, wta_k, score_type,
    patch_size, fast_threshold).detect + .compute on the device, for batches of equally sized gray images (first_level 0, wta_k 2
    and patch_size 31 only)."""

    def __init__(self, ctx: Context, n_features=500, scale_factor=1.2, nlevels=8, edge_threshold=31, first_level=0, wta_k=2,
                 score_type=0, patch_size=31, fast_threshold=20, max_batch=1, max_height=1024, max_width=1024):
        self.ctx = ctx
        self.conf = OrbConf(int(n_features), float(scale_factor), int(nlevels), int(edge_threshold), int(first_level), int(wta_k),
                            int(score_type), int(patch_size), int(fast_threshold), int(max_batch), int(max_height), int(max_width))
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_orb_create(ctx.h, C.byref(self.conf), C.byref(h)), "dimb_orb_create")
        self.h = h

    def extract(self, image: np.ndarray, cap: int | None = None) -> dict:
        """image uint8 (H,W) -> keypoints (N,2), descriptors (32,N) float32 with the byte values 0..255, size / angle / response
        (N,) and octave (N,) int32 (the level)."""
        image = np.ascontiguousarray(image)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("OrbNet.extract takes a uint8 (H, W) image")
        H, W = image.shape
        cap = cap or max(self.conf.n_features, 1) + 64
        while True:
            kp = np.zeros((cap, 2), np.float32)
            de = np.zeros((32, cap), np.float32)
            fr = np.zeros((cap, 3), np.float32)
            oc = np.zeros(cap, np.int32)
            cnt = np.zeros(1, np.int32)
            rc = self.ctx.lib.dimb_orb_extract(self.h, _ptr(image), H, W, _ptr(kp), _ptr(de), _ptr(fr), _ptr(oc), _ptr(cnt), cap)
            if rc == ERR_CAPACITY and cnt[0] > cap:
                cap = int(cnt[0])
                continue
            self.ctx.check(rc, "dimb_orb_extract")
            break
        n = int(cnt[0])
        return {"keypoints": kp[:n].copy(), "descriptors": de[:, :n].copy(), "size": fr[:n, 0].copy(), "angle": fr[:n, 1].copy(),
                "response": fr[:n, 2].copy(), "octave": oc[:n].copy()}

    def extract_dev(self, d_images, B, H, W, d_kpts, d_desc, d_counts, cap, d_frames=0, d_octave=0, stream=0):
        """Raw device-pointer variant (ints are device addresses, e.g. torch.Tensor.data_ptr())."""
        self.ctx.check(self.ctx.lib.dimb_orb_extract_dev(self.h, d_images, B, H, W, d_kpts, d_desc, d_frames or None,
                                                         d_octave or None, d_counts, cap, stream), "dimb_orb_extract_dev")

    def debug_read(self, which: int, image: int, level: int, height: int, width: int) -> np.ndarray:
        """which 0: pyramid level `level` of the last call, 1: its blurred copy; (height, width) are the image's."""
        h, w = orb_level_sizes(height, width, self.conf.nlevels, self.conf.scale_factor)[level]
        out = np.zeros((h, w), np.float32)
        self.ctx.check(self.ctx.lib.dimb_orb_debug_read(self.h, which, image, level, _ptr(out), out.size), "dimb_orb_debug_read")
        return out

    def __del__(self):
        try:
            self.ctx.lib.dimb_orb_destroy(self.h)
        except Exception:
            pass


def superglue_weight_names(n_layers: int = 18) -> list:
    bn = lambda p: [p + s for s in (".weight", ".bias", ".running_mean", ".running_var")]
    names = []
    for i in range(5):
        names += [f"kenc.encoder.{3 * i}.weight", f"kenc.encoder.{3 * i}.bias"]
        if i < 4:
            names += bn(f"kenc.encoder.{3 * i + 1}")
    for i in range(n_layers):
        p = f"gnn.layers.{i}."
        names += [p + "attn.merge.weight", p + "attn.merge.bias"]
        for j in range(3):
            names += [p + f"attn.proj.{j}.weight", p + f"attn.proj.{j}.bias"]
        names += [p + "mlp.0.weight", p + "mlp.0.bias"] + bn(p + "mlp.1") + [p + "mlp.3.weight", p + "mlp.3.bias"]
    return names + ["final_proj.weight", "final_proj.bias", "bin_score"]


class SuperGlueNet:
    """Handle on dimb_sg: SuperGlue matching of one host pair per call (match) or of up to max_pairs device pairs (match_dev)."""

    def __init__(self, ctx: Context, weights: dict, gnn_layers=("self", "cross") * 9, sinkhorn_iterations=100, match_threshold=0.2,
                 max_kpts=2048, max_pairs=1):
        self.ctx = ctx
        mask = sum(1 << i for i, n in enumerate(gnn_layers) if n == "cross")
        self.conf = SgConf(len(gnn_layers), mask, int(sinkhorn_iterations), float(match_threshold), int(max_kpts), int(max_pairs))
        blob = np.ascontiguousarray(np.concatenate([np.asarray(weights[n], np.float32).ravel() for n in superglue_weight_names(len(gnn_layers))]))
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_sg_create(ctx.h, _ptr(blob), blob.size, C.byref(self.conf), C.byref(h)), "dimb_sg_create")
        self.h = h

    def match(self, feats0: dict, feats1: dict) -> dict:
        """feats: keypoints (N,2), descriptors (256,N), scores (N,), image_size [H,W] -> matches int64 (S,2), scores (S,)."""
        fs, keep = [], []
        for f in (feats0, feats1):
            k = np.ascontiguousarray(f["keypoints"], np.float32)
            d = np.ascontiguousarray(f["descriptors"], np.float32)
            s = np.ascontiguousarray(f["scores"], np.float32)
            if d.shape != (256, k.shape[0]):
                raise ValueError(f"SuperGlue expects (256,N) descriptors, got {d.shape} for {k.shape[0]} keypoints")
            hw = np.asarray(f["image_size"]).astype(int).ravel()
            keep += [k, d, s]
            fs.append(SgFeats(k.ctypes.data, d.ctypes.data, s.ctypes.data, k.shape[0], 0, int(hw[0]), int(hw[1])))
        cap = max(1, min(fs[0].n, fs[1].n))
        m = np.zeros((cap, 2), np.int64)
        sc = np.zeros(cap, np.float32)
        n = C.c_int(0)
        self.ctx.check(self.ctx.lib.dimb_sg_match(self.h, C.byref(fs[0]), C.byref(fs[1]), _ptr(m), _ptr(sc), C.byref(n), cap), "dimb_sg_match")
        return {"matches": m[: n.value].copy(), "scores": sc[: n.value].copy()}

    def match_dev(self, f0: list, f1: list, d_matches, d_mscores, d_n_matches, cap, stream=0):
        """f0/f1: lists of SgFeatsDev (device pointers); outputs [P][cap][2] int64, [P][cap], [P] int32 device buffers (ints are
        device addresses); asynchronous on `stream`."""
        P = len(f0)
        a0 = (SgFeatsDev * P)(*f0)
        a1 = (SgFeatsDev * P)(*f1)
        self.ctx.check(self.ctx.lib.dimb_sg_match_dev(self.h, P, a0, a1, d_matches, d_mscores, d_n_matches, cap, stream),
                       "dimb_sg_match_dev")

    def __del__(self):
        try:
            self.ctx.lib.dimb_sg_destroy(self.h)
        except Exception:
            pass


class LightGlueNet:
    """Handle on dimb_lg: LightGlue matching of batches of pairs."""

    def __init__(self, ctx: Context, weights: dict, input_dim=256, descriptor_dim=256, n_layers=9, num_heads=4,
                 depth_confidence=0.95, width_confidence=0.99, filter_threshold=0.1, prune_min_kpts=1536, max_pairs=1,
                 max_kpts=2048):
        self.ctx = ctx
        self.conf = LgConf(int(input_dim), int(descriptor_dim), int(n_layers), int(num_heads), float(depth_confidence),
                           float(width_confidence), float(filter_threshold), int(prune_min_kpts), int(max_pairs),
                           int(max_kpts))
        blob = pack_lightglue_weights(weights, input_dim, descriptor_dim, n_layers)
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_lg_create(ctx.h, _ptr(blob), blob.size, C.byref(self.conf), C.byref(h)), "dimb_lg_create")
        self.h = h
        self.NP = (int(max_kpts) + 127) // 128 * 128

    def match(self, pairs):
        """pairs: list of (feats0, feats1) with keypoints (N,2), descriptors (N,D) [layout 1] or (D,N) [layout 0]
        already decided by the caller via key "_layout"; image_size optional.
        Returns list of dict(matches int64 (S,2), scores (S,), stop int)."""
        P = len(pairs)
        f0 = (Feats * P)()
        f1 = (Feats * P)()
        keep = []
        cap = 1
        for p, (a, b) in enumerate(pairs):
            for arr, f in ((f0, a), (f1, b)):
                k = np.ascontiguousarray(f["keypoints"], np.float32)
                d = np.ascontiguousarray(f["descriptors"], np.float32)
                keep += [k, d]
                e = arr[p]
                e.keypoints, e.descriptors = k.ctypes.data, d.ctypes.data
                e.n = k.shape[0]
                e.desc_layout = int(f.get("_layout", 1))
                e.desc_ld = 0
                size = f.get("image_size")
                e.has_size = int(size is not None)
                if size is not None:
                    size = np.asarray(size, np.float32).ravel()
                    e.size0, e.size1 = float(size[0]), float(size[1])
            cap = max(cap, min(a["keypoints"].shape[0], b["keypoints"].shape[0]))
        m = np.zeros((P, cap, 2), np.int64)
        s = np.zeros((P, cap), np.float32)
        nm = np.zeros(P, np.int32)
        sl = np.zeros(P, np.int32)
        self.ctx.check(self.ctx.lib.dimb_lg_match(self.h, P, f0, f1, _ptr(m), _ptr(s), _ptr(nm), _ptr(sl), cap),
                       "dimb_lg_match")
        return [{"matches": m[p, : nm[p]].copy(), "scores": s[p, : nm[p]].copy(), "stop": int(sl[p])} for p in range(P)]

    def match_dev(self, f0: list, f1: list, d_matches, d_mscores, d_n_matches, d_stop, cap, stream=0):
        """f0/f1: lists of FeatsDev (device pointers)."""
        P = len(f0)
        a0 = (FeatsDev * P)(*f0)
        a1 = (FeatsDev * P)(*f1)
        self.ctx.check(self.ctx.lib.dimb_lg_match_dev(self.h, P, a0, a1, d_matches, d_mscores, d_n_matches, d_stop, cap,
                                                      stream), "dimb_lg_match_dev")

    def debug_read(self, which: int, side: int, shape) -> np.ndarray:
        out = np.zeros(shape, np.float32)
        self.ctx.check(self.ctx.lib.dimb_lg_debug_read(self.h, which, side, _ptr(out), out.size), "dimb_lg_debug_read")
        return out

    def __del__(self):
        try:
            self.ctx.lib.dimb_lg_destroy(self.h)
        except Exception:
            pass


class FeatureStoreDev:
    """Handle on dimb_fstore: the content of features.h5 (float16 arrays + int image_size, one block per image) kept in HBM."""

    def __init__(self, ctx: Context, n_slots: int, cap: int, desc_dim: int):
        self.ctx, self.n_slots, self.desc_dim = ctx, int(n_slots), int(desc_dim)
        h = C.c_void_p()
        ctx.check(ctx.lib.dimb_fstore_create(ctx.h, n_slots, cap, desc_dim, C.byref(h)), "dimb_fstore_create")
        self.h = h
        base, sb, ns, cp = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
        ctx.check(ctx.lib.dimb_fstore_block_dev(h, C.byref(base), C.byref(sb), C.byref(ns), C.byref(cp)), "dimb_fstore_block_dev")
        self.base, self.slot_bytes, self.cap = base.value, sb.value, cp.value

    def put_dev(self, slot, d_kpts, d_scores, d_desc, desc_ld, d_count, height, width, d_tile_idx=None, stream=0):
        self.ctx.check(self.ctx.lib.dimb_fstore_put_dev(self.h, slot, d_kpts, d_scores, d_tile_idx, d_desc, desc_ld, d_count, int(height),
                                                        int(width), stream), "dimb_fstore_put_dev")

    def put(self, slot: int, feats: dict):
        """feats: FeaturesDict (keypoints (N,2), descriptors (D,N), optional scores / tile_idx, image_size [H,W])."""
        k = np.ascontiguousarray(feats["keypoints"], np.float32)
        d = np.ascontiguousarray(feats["descriptors"], np.float32)
        n = k.shape[0]
        if d.shape != (self.desc_dim, n):
            raise ValueError(f"descriptors must be ({self.desc_dim},{n}), got {d.shape}")
        s = np.ascontiguousarray(feats["scores"], np.float32) if feats.get("scores") is not None else None
        t = np.ascontiguousarray(feats["tile_idx"], np.float32) if feats.get("tile_idx") is not None else None
        hw = np.asarray(feats.get("image_size", (0, 0))).astype(int).ravel()
        self.ctx.check(self.ctx.lib.dimb_fstore_put(self.h, slot, _ptr(k), _ptr(s) if s is not None else None,
                                                    _ptr(t) if t is not None else None, _ptr(d), n, int(hw[0]), int(hw[1])), "dimb_fstore_put")

    def count(self, slot: int):
        n, size = C.c_int(), np.zeros(2, np.int32)
        self.ctx.check(self.ctx.lib.dimb_fstore_count(self.h, slot, C.byref(n), _ptr(size)), "dimb_fstore_count")
        return n.value, size

    def get(self, slot: int) -> dict:
        """The FeaturesDict get_features (io/h5.py:45-89) would return for this image."""
        n, size = self.count(slot)
        if n < 0:
            raise ValueError(f"slot {slot} of the feature store is empty")
        k, s, t = np.zeros((n, 2), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        d = np.zeros((self.desc_dim, n), np.float32)
        cnt = C.c_int()
        self.ctx.check(self.ctx.lib.dimb_fstore_get(self.h, slot, _ptr(k), _ptr(s), _ptr(t), _ptr(d), C.byref(cnt), _ptr(size), max(n, 1)),
                       "dimb_fstore_get")
        return {"keypoints": k, "descriptors": d, "scores": s, "tile_idx": t, "image_size": size.astype(np.int32)}

    def feats_dev(self, slot: int, size=None) -> FeatsDev:
        """The slot as LightGlue / NN input.  size: None (the slot header's [H,W] through size_dev), or an explicit normalisation size
        (size0, size1) carried in the struct with size_dev NULL (LighterGlue's [W,H])."""
        f = FeatsDev()
        self.ctx.check(self.ctx.lib.dimb_fstore_feats_dev(self.h, slot, C.byref(f)), "dimb_fstore_feats_dev")
        if size is not None:
            f.size_dev = None
            f.size0, f.size1 = float(size[0]), float(size[1])
        return f

    def sg_feats_dev(self, slot: int) -> SgFeatsDev:
        """The slot as SuperGlue input (float16 keypoints, descriptors and scores, image_size from the slot header)."""
        f = SgFeatsDev()
        self.ctx.check(self.ctx.lib.dimb_fstore_sg_feats_dev(self.h, slot, C.byref(f)), "dimb_fstore_sg_feats_dev")
        return f

    def tile_merge_dev(self, slots, H, W, tile_h, tile_w, overlap_h, overlap_w, d_kpts, d_scores, d_desc, d_counts, K, stream=0):
        """Tile-feature merge of len(slots) images (dimb_tile_merge_dev): the extractor outputs of their T tiles each ([B*T][K] layouts)
        -> one merged slot per image.  Asynchronous on `stream`."""
        s, p = _int_array(slots)
        self.ctx.check(self.ctx.lib.dimb_tile_merge_dev(self.h, len(s), p, H, W, tile_h, tile_w, overlap_h, overlap_w, d_kpts, d_scores, d_desc,
                                                        d_counts, K, stream), "dimb_tile_merge_dev")

    def rescale_dev(self, slots, level, H, W, stream=0):
        """Keypoints of `slots` times 2^level and header image size H x W (dimb_fstore_rescale_dev): features extracted from an image
        resized by `level` pyramid steps, back in the original image's pixels.  Asynchronous on `stream`."""
        s, p = _int_array(slots)
        self.ctx.check(self.ctx.lib.dimb_fstore_rescale_dev(self.h, len(s), p, int(level), int(H), int(W), stream), "dimb_fstore_rescale_dev")

    def unrotate_dev(self, slots, rotations, heights, widths, stream=0):
        """Keypoints of `slots`, extracted from images turned by `rotations` (degrees clockwise), back on the original heights[b] x
        widths[b] images, and those sizes in the headers (dimb_fstore_unrotate_dev).  Asynchronous on `stream`."""
        arrays = [_int_array(v) for v in (slots, rotations, heights, widths)]
        if len({len(a) for a, _ in arrays}) != 1:
            raise ValueError("unrotate_dev needs one rotation, height and width per slot")
        self.ctx.check(self.ctx.lib.dimb_fstore_unrotate_dev(self.h, len(arrays[0][0]), *[p for _, p in arrays], stream),
                       "dimb_fstore_unrotate_dev")

    def tile_views_dev(self, src_slots, n_tiles, views: "FeatureStoreDev", dst_slots, d_map, stream=0):
        """Tile views of the merged slots src_slots (dimb_tile_views_dev): view slot dst_slots[b] + t of `views`, map row of the same
        index in d_map ([views.n_slots][views.cap] int32).  Asynchronous on `stream`."""
        s, ps = _int_array(src_slots)
        d, pd = _int_array(dst_slots)
        self.ctx.check(self.ctx.lib.dimb_tile_views_dev(self.h, len(s), ps, n_tiles, views.h, pd, d_map, stream), "dimb_tile_views_dev")

    def desc_ptr(self, slot: int) -> int:
        """Device address of the slot's float16 (D, cap) descriptor block (for dimb_nn_match_dev, ld = cap)."""
        return self.feats_dev(slot).descriptors

    def __del__(self):
        try:
            self.ctx.lib.dimb_fstore_destroy(self.h)
        except Exception:
            pass


class Pipe:
    """Fused per-pair path (dimb_pipe): images -> SuperPoint x2 -> LightGlue, features stay in HBM."""

    def __init__(self, sp: SuperPointNet, lg: LightGlueNet, max_pairs: int, H: int, W: int, cap: int):
        self.ctx, self.sp, self.lg = sp.ctx, sp, lg
        self.max_pairs, self.H, self.W, self.cap = max_pairs, H, W, cap
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.dimb_pipe_create(sp.h, lg.h, max_pairs, H, W, cap, C.byref(h)), "dimb_pipe_create")
        self.h = h

    def match_image_pairs(self, images: np.ndarray, out: dict | None = None, want_kpts: bool = False) -> dict:
        """images: float32 or uint8 (2P,H,W) gray host array (pinned for async copies). Returns host arrays."""
        B = images.shape[0]
        P = B // 2
        if out is None:
            out = self.alloc_outputs(P, want_kpts)
        kp = out.get("kpts")
        fn = self.ctx.lib.dimb_pipe_match_image_pairs_u8 if images.dtype == np.uint8 else self.ctx.lib.dimb_pipe_match_image_pairs
        assert images.dtype in (np.uint8, np.float32) and images.flags.c_contiguous
        self.ctx.check(fn(
            self.h, images.ctypes.data, P, out["matches"].ctypes.data, out["mscores"].ctypes.data,
            out["n_matches"].ctypes.data, out["stop"].ctypes.data, out["n_kpts"].ctypes.data,
            kp.ctypes.data if kp is not None else None), "dimb_pipe_match_image_pairs")
        return out

    def alloc_outputs(self, P: int, want_kpts: bool = False) -> dict:
        out = {"matches": np.zeros((P, self.cap, 2), np.int64), "mscores": np.zeros((P, self.cap), np.float32),
               "n_matches": np.zeros(P, np.int32), "stop": np.zeros(P, np.int32), "n_kpts": np.zeros(2 * P, np.int32)}
        if want_kpts:
            out["kpts"] = np.zeros((2 * P, self.cap, 2), np.float32)
        return out

    def match_image_pairs_dev(self, d_images: int, P: int, stream: int = 0):
        self.ctx.check(self.ctx.lib.dimb_pipe_match_image_pairs_dev(self.h, d_images, P, stream),
                       "dimb_pipe_match_image_pairs_dev")

    def outputs_dev(self) -> dict:
        ptrs = [C.c_void_p() for _ in range(6)]
        self.ctx.check(self.ctx.lib.dimb_pipe_outputs_dev(self.h, *[C.byref(p) for p in ptrs]), "dimb_pipe_outputs_dev")
        return dict(zip(["matches", "mscores", "n_matches", "stop", "n_kpts", "kpts"], [p.value for p in ptrs]))

    def features_dev(self) -> dict:
        ptrs = [C.c_void_p() for _ in range(4)]
        self.ctx.check(self.ctx.lib.dimb_pipe_features_dev(self.h, *[C.byref(p) for p in ptrs]), "dimb_pipe_features_dev")
        return dict(zip(["kpts", "scores", "desc", "counts"], [p.value for p in ptrs]))

    def read_features(self, P: int) -> list:
        """Host copies of the last call's SuperPoint features (2P FeaturesDicts, float32, before the fp16 cast)."""
        d = self.features_dev()
        B, cap = 2 * P, self.cap
        kp, sc = np.zeros((B, cap, 2), np.float32), np.zeros((B, cap), np.float32)
        de, cnt = np.zeros((B, 256, cap), np.float32), np.zeros(B, np.int32)
        for dst, src in ((kp, d["kpts"]), (sc, d["scores"]), (de, d["desc"]), (cnt, d["counts"])):
            self.ctx.check(self.ctx.lib.dimb_read_dev(self.ctx.h, dst.ctypes.data, src, dst.nbytes), "dimb_read_dev")
        return [{"keypoints": kp[b, :cnt[b]].copy(), "scores": sc[b, :cnt[b]].copy(), "descriptors": de[b, :, :cnt[b]].copy()}
                for b in range(B)]

    def __del__(self):
        try:
            self.ctx.lib.dimb_pipe_destroy(self.h)
        except Exception:
            pass
