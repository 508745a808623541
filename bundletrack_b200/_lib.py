"""ctypes binding of the C-ABI (include/bundletrack_b200.h).  The shared library is built in-tree by
__graft_entry__.build() / `make -C bundletrack_b200/csrc`; if it is missing, or the machine has no sm_90 GPU,
every entry point fails loudly — there is no CPU or PyTorch fallback anywhere in this package."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# BT_B200_LIB selects another BUILD of the same library (kernel experiments); there is still no non-CUDA path behind it
LIB_PATH = os.environ.get("BT_B200_LIB") or os.path.join(_HERE, "lib", "libbundletrack_b200.so")

BT_OK = 0
BT_ERR_INVALID_ARG = -1
BT_ERR_CAPACITY = -2
BT_ERR_NO_DEVICE = -4
BT_MASK_AS_IS, BT_MASK_LARGEST_HULL = 0, 1      # bt_frames_preprocess_masked's mask_mode
BT_PAIR_OK, BT_PAIR_EMPTY, BT_PAIR_FAIL = 0, 1, 2
BT_FRAME_OTHER, BT_FRAME_FAIL, BT_FRAME_NO_BA = 0, 1, 2      # Frame::_status as the tracker reports it


class BtError(RuntimeError):
    """A library call failed; rc is its BT_* status (None when the error was raised on the Python side)."""
    def __init__(self, msg: str, rc: int = None):
        super().__init__(msg)
        self.rc = rc


class SolverParams(ctypes.Structure):
    _fields_ = [
        ("num_iter_outer", ctypes.c_int),
        ("num_iter_inner", ctypes.c_int),
        ("robust_delta", ctypes.c_float),
        ("image_downscale", ctypes.c_float),
        ("dense_dist_thresh", ctypes.c_float),
        ("dense_cos_normal_thresh", ctypes.c_float),
        ("depth_min", ctypes.c_float),
        ("depth_max", ctypes.c_float),
        ("w_sparse", ctypes.c_float),
        ("w_dense", ctypes.c_float),
    ]


class Window(ctypes.Structure):
    _fields_ = [
        ("n_frames", ctypes.c_int),
        ("H", ctypes.c_int),
        ("W", ctypes.c_int),
        ("n_corr", ctypes.c_int),
        ("corr", ctypes.c_void_p),
        ("depth_dev", ctypes.POINTER(ctypes.c_void_p)),
        ("normal_dev", ctypes.POINTER(ctypes.c_void_p)),
        ("fx", ctypes.c_float),
        ("fy", ctypes.c_float),
        ("cx", ctypes.c_float),
        ("cy", ctypes.c_float),
        ("dense_pairs", ctypes.c_void_p),
        ("n_dense_pairs", ctypes.c_int),
        ("compat_flip", ctypes.c_int),
        ("cache_slots", ctypes.c_void_p),
        ("corr_dev", ctypes.c_void_p),
        ("n_blocks", ctypes.c_int),
        ("block_off", ctypes.c_void_p),
        ("block_n", ctypes.c_void_p),
        ("block_i", ctypes.c_void_p),
        ("block_j", ctypes.c_void_p),
    ]


class DepthParams(ctypes.Structure):
    _fields_ = [
        ("erode_radius", ctypes.c_int),
        ("erode_diff", ctypes.c_float),
        ("erode_ratio", ctypes.c_float),
        ("bf_radius", ctypes.c_int),
        ("sigma_D", ctypes.c_float),
        ("sigma_R", ctypes.c_float),
    ]


class SolverLimits(ctypes.Structure):
    _fields_ = [
        ("max_windows", ctypes.c_int),
        ("max_frames", ctypes.c_int),
        ("max_corr", ctypes.c_int),
        ("H", ctypes.c_int),
        ("W", ctypes.c_int),
        ("image_downscale", ctypes.c_float),
    ]


class SolveStats(ctypes.Structure):
    _fields_ = [
        ("n_windows", ctypes.c_int),
        ("n_tiles_total", ctypes.c_int),
        ("n_kernel_launches", ctypes.c_int),
        ("n_src_pixels", ctypes.c_longlong),
    ]


class MatchFrame(ctypes.Structure):
    _fields_ = [
        ("kpts_dev", ctypes.c_void_p),
        ("n", ctypes.c_int),
        ("depth_dev", ctypes.c_void_p),
        ("normal_dev", ctypes.c_void_p),
        ("pose", ctypes.c_float * 16),
        ("frame_id", ctypes.c_int),
        ("window_index", ctypes.c_int),
    ]


class PruneParams(ctypes.Structure):
    _fields_ = [
        ("max_dist_no_neighbor", ctypes.c_float),
        ("cos_max_normal_no_neighbor", ctypes.c_float),
        ("max_dist_neighbor", ctypes.c_float),
        ("cos_max_normal_neighbor", ctypes.c_float),
    ]


class TrackerParams(ctypes.Structure):
    _fields_ = [
        ("H", ctypes.c_int), ("W", ctypes.c_int),
        ("fx", ctypes.c_float), ("fy", ctypes.c_float), ("cx", ctypes.c_float), ("cy", ctypes.c_float),
        ("max_feats", ctypes.c_int),
        ("max_frames_alive", ctypes.c_int),
        ("mask_mode", ctypes.c_int),
        ("depth", DepthParams), ("solver", SolverParams), ("prune", PruneParams),
        ("ransac_trials", ctypes.c_int), ("ransac_inlier_dist", ctypes.c_float),
        ("window_size", ctypes.c_int), ("max_BA_frames", ctypes.c_int), ("min_fm_edges_newframe", ctypes.c_int), ("min_feat_num", ctypes.c_int),
        ("min_rot_deg", ctypes.c_float),
        ("max_keyframes", ctypes.c_int),
    ]


class MatchExtra(ctypes.Structure):
    _fields_ = [("uv", ctypes.c_void_p), ("n", ctypes.c_int)]


class MatchVizDesc(ctypes.Structure):
    _fields_ = [
        ("colour_a", ctypes.c_void_p), ("H_a", ctypes.c_int), ("W_a", ctypes.c_int), ("roi_a", ctypes.c_int32 * 4),
        ("colour_b", ctypes.c_void_p), ("H_b", ctypes.c_int), ("W_b", ctypes.c_int), ("roi_b", ctypes.c_int32 * 4),
        ("uv", ctypes.c_void_p), ("n", ctypes.c_int), ("rng_state", ctypes.c_uint64),
    ]


class DescView(ctypes.Structure):
    _fields_ = [
        ("dev", ctypes.c_void_p),
        ("n", ctypes.c_int),
        ("dim", ctypes.c_int),
        ("pitch_bytes", ctypes.c_size_t),
    ]


# every symbol include/bundletrack_b200.h declares (tests/test_abi.py checks the .so exports all of them)
EXPORTS = [
    "bt_last_error", "bt_version", "bt_ctx_create", "bt_ctx_destroy", "bt_solver_reserve",
    "bt_solve_windows", "bt_solve_windows_begin", "bt_solve_windows_end", "bt_solve_stage", "bt_solve_run", "bt_solve_fetch", "bt_solve_get_stats",
    "bt_solve_enable_debug", "bt_solve_debug_dense", "bt_solve_debug_counts", "bt_solve_debug_system", "bt_solve_enable_timing", "bt_solve_get_timing", "bt_solve_get_host_timing", "bt_solve_enable_profile", "bt_solve_get_profile",
    "bt_matcher_reserve", "bt_desc_pool_reserve", "bt_desc_pool_store", "bt_knn_match_slots", "bt_match_pairs_pool", "bt_match_pairs_ex", "bt_match_cache_reserve", "bt_match_cache_reserve_entries", "bt_match_cache_usage", "bt_match_cache_put", "bt_match_cache_has", "bt_match_cache_status", "bt_match_cache_gather", "bt_match_cache_forget_frame", "bt_knn_match_pairs", "bt_knn_enable_timing", "bt_knn_get_timing", "bt_knn_debug_force_fallback", "bt_ransac_reserve", "bt_ransac_pairs", "bt_ransac_debug",
    "bt_pipeline_reserve", "bt_prune_mutual_pairs", "bt_match_pairs", "bt_frames_preprocess", "bt_frames_preprocess_masked", "bt_frames_preprocess_masked_u16", "bt_lfnet_request",
    "bt_frame_cache_reserve", "bt_frame_cache_store",
    "bt_rotation_geodesic", "bt_keyframe_check", "bt_select_keyframes", "bt_rigid_transform", "bt_lfnet_parse_reply", "bt_ba_gate", "bt_pose_format", "bt_pose_write_txt",
    "bt_tracks_create", "bt_tracks_destroy", "bt_tracks_update_pair", "bt_tracks_propagate", "bt_tracks_forget_frame", "bt_tracks_stats",
    "bt_tracks_dev_reserve", "bt_tracks_dev_reserve_ex", "bt_tracks_dev_update_pair", "bt_tracks_dev_propagate", "bt_tracks_dev_forget_frame", "bt_tracks_dev_stats", "bt_find_corres_pairs",
    "bt_pose_init", "bt_tracker_create", "bt_tracker_destroy", "bt_tracker_begin_frame", "bt_tracker_begin_frame_u16", "bt_tracker_end_frame", "bt_tracker_drop_frame", "bt_tracker_state", "bt_tracker_usage", "bt_tracker_last_fg",
    "bt_metrics_reserve", "bt_pose_metrics", "bt_vocap", "bt_nocs_reserve", "bt_nocs_metrics", "bt_nocs_score",
    "bt_overlay_reserve", "bt_voxel_downsample", "bt_pose_overlay",
    "bt_match_viz_shape", "bt_match_viz_reserve", "bt_match_viz",
    "bt_dev_alloc", "bt_dev_free", "bt_memcpy_h2d", "bt_memcpy_d2h", "bt_host_alloc_pinned", "bt_host_free_pinned",
    "bt_stream_sync", "bt_debug_live_resources",
]

_lib = None


def load() -> ctypes.CDLL:
    """Load the in-tree shared library; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BtError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). bundletrack_b200 has no CPU fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    lib.bt_last_error.restype = ctypes.c_char_p
    for name in EXPORTS:
        fn = getattr(lib, name)
        if name not in ("bt_last_error", "bt_ctx_destroy", "bt_rotation_geodesic", "bt_tracks_destroy", "bt_tracker_destroy"):
            fn.restype = ctypes.c_int
    lib.bt_ctx_destroy.restype = None
    lib.bt_rotation_geodesic.restype = ctypes.c_float
    lib.bt_tracks_destroy.restype = None
    lib.bt_tracker_destroy.restype = None
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != BT_OK:
        msg = load().bt_last_error().decode("utf-8", "replace")
        raise BtError(f"{what} failed with status {rc}: {msg}", rc)
