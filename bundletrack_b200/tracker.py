"""`Bundler::processNewFrame` (the reference's src/Bundler.cpp:56-183) as one object: give it frames, get poses.  A thin ctypes mirror of
bt_tracker_* (include/bundletrack_b200.h); the step itself - ids, the frame deque, keyframes, matching, the initial pose, the BA gate and the
solve - runs in the library.  The step is split where the reference asks the LF-Net server for features: `begin_frame` returns the request
image, the caller does the round trip (its reply goes through policy.lfnet_parse_reply) and hands keypoints and descriptors to `end_frame`,
or calls `drop_frame` when detection failed."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .config import depth_params, load_yml, mask_mode, prune_params, solver_params


def tracker_params(yml, H: int, W: int, K, max_feats: int, max_frames_alive: int, mode: int = None, max_keyframes: int = 0) -> "_lib.TrackerParams":
    """bt_tracker_params from the config keys the reference reads (bundle.window_size / max_BA_frames / min_fm_edges_newframe,
    keyframe.min_feat_num / min_rot, ransac.max_iter / inlier_dist and those config.py maps).  mode: _lib.BT_MASK_* (default: config.mask_mode).
    max_keyframes > 0 holds that many keyframes apart from max_frames_alive (the header's bt_tracker_params)."""
    y = load_yml(yml)
    fx, fy, cx, cy = _lib.intrinsics(K)
    b, kf, rs = y["bundle"], y["keyframe"], y["ransac"]
    p = _lib.TrackerParams()
    p.H, p.W, p.fx, p.fy, p.cx, p.cy = int(H), int(W), fx, fy, cx, cy
    p.max_feats, p.max_frames_alive, p.max_keyframes = int(max_feats), int(max_frames_alive), int(max_keyframes)
    p.mask_mode = mask_mode(yml) if mode is None else int(mode)
    p.depth, p.solver, p.prune = depth_params(y), solver_params(y), prune_params(y)
    p.ransac_trials, p.ransac_inlier_dist = int(rs["max_iter"]), float(rs["inlier_dist"])
    p.window_size, p.max_BA_frames, p.min_fm_edges_newframe = int(b["window_size"]), int(b["max_BA_frames"]), int(b["min_fm_edges_newframe"])
    p.min_feat_num, p.min_rot_deg = int(kf["min_feat_num"]), float(kf["min_rot"])
    return p


class Tracker:
    """Tracker(yml, H, W, K, max_feats, max_frames_alive, max_keyframes=0): everything is reserved here (bt_tracker_create states the
    memory).  For a whole sequence give it a keyframe pool: max_frames_alive = window_size + 4 or so and max_keyframes = the most keyframes the
    sequence can admit.  Device arguments are torch CUDA tensors (or raw device addresses); the library works on `stream` (default: the legacy
    default stream)."""

    def __init__(self, yml, H: int, W: int, K, max_feats: int, max_frames_alive: int, device: int = 0, stream: int = 0, mode: int = None,
                 max_keyframes: int = 0):
        self.lib = _lib.load()
        self.params = tracker_params(yml, H, W, K, max_feats, max_frames_alive, mode, max_keyframes)
        self.stream = ctypes.c_void_p(stream)
        self.t = _lib.Handle("bt_tracker_create", "bt_tracker_destroy", device, self.params)

    def close(self):
        self.t.close()

    def begin_frame(self, depth_raw, mask, colour, request_out, loader_id: int = 0, first_pose=None):
        """depth_raw float32 [H,W], mask uint8 [H,W], colour uint8 [H,W,3] BGR, request_out uint8 [400,400,3]: device.  loader_id / first_pose
        (4x4 cam->model) are used only when the tracker holds no frame.  Returns (status, roi (umin, umax, vmin, vmax))."""
        roi = np.zeros(4, np.int32)
        st = ctypes.c_int(-1)
        fp = None if first_pose is None else np.ascontiguousarray(first_pose, np.float32).reshape(16)
        _lib.check(self.lib.bt_tracker_begin_frame(self.t, loader_id, _lib.ptr(fp), *(_lib.ptr(x) for x in (depth_raw, mask, colour, request_out, roi)),
                                                   ctypes.byref(st), self.stream), "bt_tracker_begin_frame")
        return st.value, roi

    def begin_frame_mm(self, depth_mm, mask, colour, request_out, loader_id: int = 0, first_pose=None):
        """`begin_frame` on the depth PNG's samples: depth_mm is device uint16 [H,W] millimetres (the library converts them as
        Utils::readDepthImage does).  Returns (status, roi, frame_id, pose [4,4] float32 cam->model): the new frame's id and initial pose,
        for every status (a frame that fails the ROI gate is recorded with this pose)."""
        roi = np.zeros(4, np.int32)
        st, fid = ctypes.c_int(-1), ctypes.c_int(-1)
        pose = np.zeros((4, 4), np.float32)
        fp = None if first_pose is None else np.ascontiguousarray(first_pose, np.float32).reshape(16)
        _lib.check(self.lib.bt_tracker_begin_frame_u16(self.t, loader_id, _lib.ptr(fp), *(_lib.ptr(x) for x in (depth_mm, mask, colour, request_out, roi)),
                                                       ctypes.byref(fid), _lib.ptr(pose), ctypes.byref(st), self.stream), "bt_tracker_begin_frame_u16")
        return st.value, roi, fid.value, pose

    def end_frame(self, kpts, desc):
        """kpts: numpy [n,2] float32 image pixels; desc: device float32 [n,256].  Returns (pose [4,4] float32 cam->model, status)."""
        k = np.ascontiguousarray(kpts, np.float32).reshape(-1, 2)
        pose = np.zeros((4, 4), np.float32)
        st = ctypes.c_int(-1)
        _lib.check(self.lib.bt_tracker_end_frame(self.t, _lib.ptr(k), len(k), _lib.desc_view(desc), _lib.ptr(pose), ctypes.byref(st), self.stream),
                   "bt_tracker_end_frame")
        return pose, st.value

    def drop_frame(self):
        """Feature detection failed: the pending frame is FAIL and forgotten.  Returns its pose."""
        pose = np.zeros((4, 4), np.float32)
        _lib.check(self.lib.bt_tracker_drop_frame(self.t, _lib.ptr(pose)), "bt_tracker_drop_frame")
        return pose

    def state(self):
        """Every frame alive, oldest first: (ids int32 [n], poses float32 [n,4,4], is_keyframe bool [n])."""
        n = ctypes.c_int(0)
        cap = self.params.max_frames_alive + self.params.max_keyframes
        ids = np.zeros(cap, np.int32)
        poses = np.zeros((cap, 4, 4), np.float32)
        kf = np.zeros(cap, np.int32)
        _lib.check(self.lib.bt_tracker_state(self.t, _lib.ptr(ids), _lib.ptr(poses), _lib.ptr(kf), cap, ctypes.byref(n)), "bt_tracker_state")
        return ids[:n.value].copy(), poses[:n.value].copy(), kf[:n.value].astype(bool)

    def last_fg(self) -> int:
        """Device address of Frame::_fg_mask (uint8 [H,W]) of the frame the last begin_frame segmented, ROI failures and dropped frames
        included; valid until the next begin_frame on the tracker's stream."""
        p = ctypes.c_void_p()
        _lib.check(self.lib.bt_tracker_last_fg(self.t, ctypes.byref(p)), "bt_tracker_last_fg")
        return int(p.value)

    def usage(self):
        """(map points alive, pairs in the match cache, entries of their blocks); synchronises the tracker's stream."""
        pts, pairs, ents = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_longlong(0)
        _lib.check(self.lib.bt_tracker_usage(self.t, ctypes.byref(pts), ctypes.byref(pairs), ctypes.byref(ents), self.stream), "bt_tracker_usage")
        return pts.value, pairs.value, ents.value
