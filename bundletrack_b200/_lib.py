"""ctypes binding of the C-ABI (include/bundletrack_b200.h).  The shared library is built in-tree by
__graft_entry__.build() / `make -C bundletrack_b200/csrc`; if it is missing, or the machine has no sm_90 GPU,
every entry point fails loudly — there is no CPU or PyTorch fallback anywhere in this package."""
from __future__ import annotations

import ctypes
import os

import numpy as np

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


class TsdfParams(ctypes.Structure):
    _fields_ = [("voxel", ctypes.c_float), ("trunc", ctypes.c_float)]


class DescView(ctypes.Structure):
    _fields_ = [
        ("dev", ctypes.c_void_p),
        ("n", ctypes.c_int),
        ("dim", ctypes.c_int),
        ("pitch_bytes", ctypes.c_size_t),
    ]


class LfnetParams(ctypes.Structure):
    _fields_ = [
        ("top_k", ctypes.c_int),
        ("net_channel", ctypes.c_int), ("net_block", ctypes.c_int), ("conv_ksize", ctypes.c_int), ("net_num_scales", ctypes.c_int),
        ("net_min_scale", ctypes.c_double), ("net_max_scale", ctypes.c_double),
        ("leaky_alpha", ctypes.c_float),
        ("sm_ksize", ctypes.c_int),
        ("com_strength", ctypes.c_float), ("score_com_strength", ctypes.c_float), ("scale_com_strength", ctypes.c_float),
        ("kp_loc_size", ctypes.c_int),
        ("kp_com_strength", ctypes.c_float),
        ("nms_ksize", ctypes.c_int),
        ("nms_thresh", ctypes.c_float),
        ("crop_radius", ctypes.c_int), ("patch_size", ctypes.c_int),
        ("desc_net_channel", ctypes.c_int), ("desc_net_depth", ctypes.c_int), ("desc_conv_ksize", ctypes.c_int), ("desc_dim", ctypes.c_int),
    ]


class VosParams(ctypes.Structure):
    _fields_ = [
        ("ref_num", ctypes.c_int), ("range", ctypes.c_int),
        ("sigma1", ctypes.c_double), ("sigma2", ctypes.c_double), ("temperature", ctypes.c_double),
    ]


# Every entry point of include/bundletrack_b200.h as (restype, argtypes), in the header's order; load() applies it, so a call site passes
# plain Python values and ctypes converts each to the C type declared here (tests/test_abi.py checks the table against the header).
# int / int32_t -> c_int, float -> c_float, double -> c_double, long long -> c_longlong, size_t -> c_size_t, uint64_t -> c_uint64, a pointer
# to a struct mirrored above -> POINTER(<Structure>), any other pointer or handle -> c_void_p; bt_last_error's string -> c_char_p.
_i, _f, _d, _ll, _sz, _u64, _p, _P = (ctypes.c_int, ctypes.c_float, ctypes.c_double, ctypes.c_longlong, ctypes.c_size_t, ctypes.c_uint64,
                                     ctypes.c_void_p, ctypes.POINTER)
PROTOTYPES = {
    "bt_last_error": (ctypes.c_char_p, ()),
    "bt_version": (_i, ()),
    "bt_ctx_create": (_i, (_p, _i)),
    "bt_ctx_destroy": (None, (_p,)),
    "bt_solver_reserve": (_i, (_p, _P(SolverLimits))),
    "bt_solve_windows": (_i, (_p, _i, _P(Window), _P(SolverParams), _p, _p)),
    "bt_solve_windows_begin": (_i, (_p, _i, _P(Window), _P(SolverParams), _p, _p)),
    "bt_solve_windows_end": (_i, (_p, _p)),
    "bt_solve_stage": (_i, (_p, _i, _P(Window), _P(SolverParams), _p, _p)),
    "bt_solve_run": (_i, (_p, _p)),
    "bt_solve_fetch": (_i, (_p, _p, _p)),
    "bt_solve_get_stats": (_i, (_p, _P(SolveStats))),
    "bt_solve_enable_timing": (_i, (_p, _i)),
    "bt_solve_get_timing": (_i, (_p, _p)),
    "bt_solve_get_host_timing": (_i, (_p, _p)),
    "bt_solve_enable_profile": (_i, (_p, _i)),
    "bt_solve_get_profile": (_i, (_p, _p, _i)),
    "bt_solve_enable_debug": (_i, (_p, _i)),
    "bt_solve_debug_dense": (_i, (_p, _i, _p, _p)),
    "bt_solve_debug_counts": (_i, (_p, _i, _i, _p)),
    "bt_solve_debug_system": (_i, (_p, _i, _i, _p, _p, _p, _p)),
    "bt_matcher_reserve": (_i, (_p, _i, _i, _i)),
    "bt_knn_match_pairs": (_i, (_p, _i, _P(DescView), _P(DescView), _i, _p, _p, _p, _p, _p)),
    "bt_desc_pool_reserve": (_i, (_p, _i)),
    "bt_desc_pool_store": (_i, (_p, _i, _P(DescView), _p)),
    "bt_knn_match_slots": (_i, (_p, _i, _p, _p, _i, _p, _p, _p, _p, _p)),
    "bt_knn_enable_timing": (_i, (_p, _i)),
    "bt_knn_debug_force_fallback": (_i, (_p, _i)),
    "bt_knn_get_timing": (_i, (_p, _p, _p)),
    "bt_ransac_reserve": (_i, (_p, _i, _i, _i)),
    "bt_ransac_pairs": (_i, (_p, _i, _p, _p, _p, _i, _f, _u64, _p, _p, _p)),
    "bt_ransac_debug": (_i, (_p, _p, _i, _p, _i)),
    "bt_ransac_debug_trials": (_i, (_p, _i, _i, _p, _p, _p)),
    "bt_pipeline_reserve": (_i, (_p, _i, _i, _i, _i)),
    "bt_prune_mutual_pairs": (_i, (_p, _i, _P(MatchFrame), _P(MatchFrame), _i, _i, _f, _f, _f, _f, _p, _p, _i, _P(PruneParams), _p, _p, _p)),
    "bt_match_pairs": (_i, (_p, _i, _P(MatchFrame), _P(MatchFrame), _P(DescView), _P(DescView), _i, _i, _f, _f, _f, _f, _P(PruneParams), _i, _f, _u64, _p, _i, _p, _p, _p, _p)),
    "bt_match_pairs_pool": (_i, (_p, _i, _P(MatchFrame), _P(MatchFrame), _p, _p, _i, _i, _f, _f, _f, _f, _P(PruneParams), _i, _f, _u64, _p, _i, _p, _p, _p, _p)),
    "bt_match_pairs_ex": (_i, (_p, _i, _P(MatchFrame), _P(MatchFrame), _P(DescView), _P(DescView), _p, _p, _i, _i, _f, _f, _f, _f, _P(PruneParams), _i, _f, _u64, _P(MatchExtra), _p, _i, _p, _p, _p, _p, _p, _p)),
    "bt_match_cache_reserve": (_i, (_p, _i, _i)),
    "bt_match_cache_reserve_entries": (_i, (_p, _i, _ll)),
    "bt_match_cache_usage": (_i, (_p, _p, _p)),
    "bt_match_cache_put": (_i, (_p, _i, _p, _p, _p, _p, _p, _p, _p)),
    "bt_match_cache_has": (_i, (_p, _i, _i)),
    "bt_match_cache_status": (_i, (_p, _i, _i, _p, _p)),
    "bt_match_cache_gather": (_i, (_p, _i, _p, _p, _p, _p, _p, _i, _p, _p, _p)),
    "bt_match_cache_forget_frame": (_i, (_p, _i)),
    "bt_frames_preprocess": (_i, (_p, _i, _p, _i, _i, _f, _f, _f, _f, _P(DepthParams), _p, _p, _p, _p)),
    "bt_frames_preprocess_masked": (_i, (_p, _i, _p, _p, _i, _i, _i, _f, _f, _f, _f, _P(DepthParams), _p, _p, _p, _p, _p, _p)),
    "bt_frames_preprocess_masked_u16": (_i, (_p, _i, _p, _p, _i, _i, _i, _f, _f, _f, _f, _P(DepthParams), _p, _p, _p, _p, _p, _p)),
    "bt_lfnet_request": (_i, (_p, _i, _p, _p, _p, _i, _i, _p, _p)),
    "bt_frame_cache_reserve": (_i, (_p, _i, _i, _i, _f)),
    "bt_frame_cache_store": (_i, (_p, _i, _p, _p, _p, _i, _i, _f, _f, _f, _f, _f, _f, _p)),
    "bt_rotation_geodesic": (_f, (_p, _p)),
    "bt_keyframe_check": (_i, (_p, _i, _i, _p, _i, _i, _f)),
    "bt_select_keyframes": (_i, (_p, _p, _i, _i, _p, _p)),
    "bt_rigid_transform": (_i, (_p, _p, _i, _p)),
    "bt_ba_gate": (_i, (_i, _i)),
    "bt_pose_format": (_i, (_p, _p, _i)),
    "bt_pose_write_txt": (_i, (_p, _p)),
    "bt_lfnet_parse_reply": (_i, (_p, _sz, _p, _sz, _sz, _p, _p, _i, _p, _p)),
    "bt_tracks_create": (_i, (_p,)),
    "bt_tracks_destroy": (None, (_p,)),
    "bt_tracks_update_pair": (_i, (_p, _i, _i, _p, _p, _i)),
    "bt_tracks_propagate": (_i, (_p, _i, _i, _p, _i, _p, _i, _p)),
    "bt_tracks_forget_frame": (_i, (_p, _i)),
    "bt_tracks_stats": (_i, (_p, _p, _p)),
    "bt_tracks_dev_reserve": (_i, (_p, _i, _i, _i)),
    "bt_tracks_dev_reserve_ex": (_i, (_p, _i, _i, _i)),
    "bt_tracks_dev_update_pair": (_i, (_p, _i, _i, _p, _p, _i, _p)),
    "bt_tracks_dev_propagate": (_i, (_p, _i, _i, _p, _i, _p, _i, _p, _p)),
    "bt_tracks_dev_forget_frame": (_i, (_p, _i, _p)),
    "bt_tracks_dev_stats": (_i, (_p, _p, _p, _p)),
    "bt_find_corres_pairs": (_i, (_p, _i, _P(MatchFrame), _P(MatchFrame), _P(DescView), _P(DescView), _p, _p, _i, _i, _f, _f, _f, _f, _P(PruneParams), _i, _f, _u64, _p, _i, _p, _p, _p, _p, _p, _p)),
    "bt_pose_init": (_i, (_p, _p, _p, _p, _p, _p, _p, _p)),
    "bt_tracker_create": (_i, (_p, _i, _P(TrackerParams))),
    "bt_tracker_destroy": (None, (_p,)),
    "bt_tracker_begin_frame": (_i, (_p, _i, _p, _p, _p, _p, _p, _p, _p, _p)),
    "bt_tracker_begin_frame_u16": (_i, (_p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p)),
    "bt_tracker_end_frame": (_i, (_p, _p, _i, _P(DescView), _p, _p, _p)),
    "bt_tracker_drop_frame": (_i, (_p, _p)),
    "bt_tracker_state": (_i, (_p, _p, _p, _p, _i, _p)),
    "bt_tracker_usage": (_i, (_p, _p, _p, _p, _p)),
    "bt_tracker_last_fg": (_i, (_p, _p)),
    "bt_tracker_frame_depth": (_i, (_p, _i, _p)),
    "bt_metrics_reserve": (_i, (_p, _i, _i)),
    "bt_pose_metrics": (_i, (_p, _p, _i, _p, _p, _i, _p, _p, _p)),
    "bt_vocap": (_i, (_p, _i, _d, _p)),
    "bt_nocs_reserve": (_i, (_p, _i)),
    "bt_nocs_metrics": (_i, (_p, _p, _p, _p, _p, _i, _p, _p, _p, _p)),
    "bt_nocs_score": (_i, (_p, _p, _p, _p, _p, _i, _p, _p)),
    "bt_surface_reserve": (_i, (_p, _i, _i)),
    "bt_mesh_sample": (_i, (_p, _p, _i, _p, _i, _i, _u64, _p, _p)),
    "bt_surface_distances": (_i, (_p, _p, _i, _p, _i, _p, _p, _p)),
    "bt_surface_score": (_i, (_p, _i, _p, _i, _p, _i, _p)),
    "bt_mask_reserve": (_i, (_p, _i, _i, _i)),
    "bt_mask_metrics": (_i, (_p, _p, _p, _i, _i, _i, _d, _p, _p, _p, _p)),
    "bt_mask_score": (_i, (_p, _p, _i, _p)),
    "bt_voxel_downsample": (_i, (_p, _i, _p, _p, _f, _p, _p, _p)),
    "bt_overlay_reserve": (_i, (_p, _i, _i)),
    "bt_pose_overlay": (_i, (_p, _i, _p, _i, _p, _f, _f, _f, _f, _p, _p, _i, _i, _p, _p, _p)),
    "bt_match_viz_shape": (_i, (_p, _p, _p, _p)),
    "bt_match_viz_reserve": (_i, (_p, _i, _i)),
    "bt_match_viz": (_i, (_p, _i, _P(MatchVizDesc), _p, _p)),
    "bt_recon_reserve": (_i, (_p, _i, _i, _i, _ll, _i, _i)),
    "bt_tsdf_fuse": (_i, (_p, _i, _p, _p, _f, _f, _f, _f, _i, _i, _p, _p)),
    "bt_tsdf_mesh": (_i, (_p, _p, _p, _p, _p, _p)),
    "bt_tsdf_grid": (_i, (_p, _p, _p, _p, _p, _p)),
    "bt_lfnet_weights_size": (_i, (_p, _p)),
    "bt_lfnet_reserve": (_i, (_p, _p, _i)),
    "bt_lfnet_load_weights": (_i, (_p, _p, _sz)),
    "bt_lfnet_detect": (_i, (_p, _i, _p, _p, _p, _p, _p)),
    "bt_lfnet_enable_timing": (_i, (_p, _i)),
    "bt_lfnet_get_timing": (_i, (_p, _p)),
    "bt_lfnet_debug_maps": (_i, (_p, _i, _p, _p, _p, _p, _p)),
    "bt_lfnet_file_info": (_i, (_p, _p, _p)),
    "bt_lfnet_load_file": (_i, (_p, _p, _i, _p)),
    "bt_vos_schedule": (_i, (_i, _i, _i, _p, _p)),
    "bt_vos_weights_size": (_i, (_p, _p)),
    "bt_vos_reserve": (_i, (_p, _p, _i, _i)),
    "bt_vos_load_weights": (_i, (_p, _p, _sz)),
    "bt_vos_begin": (_i, (_p, _p, _p, _p, _p)),
    "bt_vos_next": (_i, (_p, _p, _p, _p)),
    "bt_vos_enable_timing": (_i, (_p, _i)),
    "bt_vos_get_timing": (_i, (_p, _p)),
    "bt_vos_debug": (_i, (_p, _i, _p, _p, _p, _p, _p)),
    "bt_dev_alloc": (_i, (_p, _sz)),
    "bt_dev_free": (_i, (_p,)),
    "bt_memcpy_h2d": (_i, (_p, _p, _sz, _p)),
    "bt_memcpy_d2h": (_i, (_p, _p, _sz, _p)),
    "bt_host_alloc_pinned": (_i, (_p, _sz)),
    "bt_host_free_pinned": (_i, (_p,)),
    "bt_stream_sync": (_i, (_p,)),
    "bt_debug_live_resources": (_i, (_p, _p, _p)),
    "bt_debug_fail_alloc": (_i, (_i,)),
}
EXPORTS = list(PROTOTYPES)

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
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != BT_OK:
        msg = load().bt_last_error().decode("utf-8", "replace")
        raise BtError(f"{what} failed with status {rc}: {msg}", rc)


class Handle:
    """A library object made by the entry point `create` (which writes it to its first argument) and freed once by `destroy`.  Pass it
    straight to any lib.bt_* call: its _as_parameter_ is one c_void_p, which close() frees and sets to NULL in place.  Every holder of the
    Handle then passes NULL, which the library refuses with BT_ERR_INVALID_ARG, instead of the freed address.  The object is freed when the
    last holder lets the Handle go, or by close()."""

    def __init__(self, create: str, destroy: str, *args):
        self._as_parameter_ = ctypes.c_void_p()
        lib = load()
        self._destroy = getattr(lib, destroy)
        check(getattr(lib, create)(ctypes.byref(self._as_parameter_), *args), create)

    def close(self) -> None:
        if self._as_parameter_:
            self._destroy(self._as_parameter_)
            self._as_parameter_.value = None

    def __del__(self):
        self.close()


class Context(Handle):
    """A bt_ctx on CUDA device `device`: the scratch every facade of the package works in."""

    def __init__(self, device: int = 0):
        super().__init__("bt_ctx_create", "bt_ctx_destroy", device)


class Facade:
    """Base of the objects that work on a context.  ctx=None makes a Context this object owns, and close() destroys it; a given Context is
    shared, and close() only lets it go.  .ctx, .stream and .lib are valid arguments for raw lib.bt_* calls."""

    def __init__(self, ctx=None, device: int = 0, stream: int = 0):
        self.lib = load()
        self.stream = ctypes.c_void_p(stream)
        self._own = ctx is None
        self.ctx = Context(device) if ctx is None else ctx

    def close(self) -> None:
        if self._own and self.ctx is not None:
            self.ctx.close()
        self.ctx = None


# ---- marshalling: what every facade hands the library -------------------------------------------------------------------------------
def ptr(x):
    """The address argument of x: a tensor's data_ptr(), a numpy array as a c_void_p that keeps the array alive; anything else (None, an
    int address, a Handle) as it is.  A tensor's address does not keep the tensor alive: hold it in a local across the call, and for an
    asynchronous call until the stream has read it."""
    if isinstance(x, np.ndarray):
        return x.ctypes.data_as(ctypes.c_void_p)
    return x.data_ptr() if hasattr(x, "data_ptr") else x


def ptrs(xs) -> "ctypes.Array":
    """A host array of the addresses of xs (tensors, ints or None), for the library's `T* const*` arguments."""
    return (ctypes.c_void_p * len(xs))(*[ptr(x) for x in xs])


def i32s(xs) -> "ctypes.Array":
    return (ctypes.c_int32 * len(xs))(*[int(v) for v in xs])


def intrinsics(K) -> tuple:
    """(fx, fy, cx, cy) of a 3 x 3 camera matrix or of a 4-vector that already holds them."""
    K = np.asarray(K, np.float64)
    return tuple(float(v) for v in ((K[0, 0], K[1, 1], K[0, 2], K[1, 2]) if K.ndim == 2 else K))


def prepared(fn, *args) -> tuple:
    """fn's arguments with every Python number converted to its declared type once, for a call made many times with the same
    arguments: ctypes passes an instance of the declared type without converting it again."""
    return tuple(t(a) if isinstance(a, (int, float)) else a for t, a in zip(fn.argtypes, args))


def desc_view(t) -> DescView:
    """The bt_desc_view of a [n, dim] float32 CUDA tensor whose rows may be pitched (stride(1) == 1)."""
    return DescView(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0) * 4 if t.shape[0] > 1 else t.shape[1] * 4)
