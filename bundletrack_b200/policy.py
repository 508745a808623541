"""Host-side mirror of the policy functions around the hot path (`Bundler::checkAndAddKeyframe`, `Bundler::selectKeyFramesForBA`,
`Utils::solveRigidTransformBetweenPoints`; /root/reference/src/Bundler.cpp:185-274, Utils.cpp:42-47,180-214) on top of the C-ABI.
These entry points are plain host code in the library: they work without a GPU."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib


def rotation_geodesic(pose_a, pose_b) -> float:
    a, b = np.ascontiguousarray(pose_a, np.float32), np.ascontiguousarray(pose_b, np.float32)
    return float(_lib.load().bt_rotation_geodesic(_lib.ptr(a), _lib.ptr(b)))


def keyframe_check(pose_new, frame_id: int, n_keypts: int, keyframe_poses, min_feat_num: int = 0, min_rot_deg: float = 10.0) -> bool:
    kp = np.ascontiguousarray(keyframe_poses, np.float32).reshape(-1, 4, 4)
    pn = np.ascontiguousarray(pose_new, np.float32)
    return bool(_lib.load().bt_keyframe_check(_lib.ptr(pn), frame_id, n_keypts, _lib.ptr(kp), len(kp), min_feat_num, min_rot_deg))


def select_keyframes(pose_new, keyframe_poses, max_BA_frames: int = 15) -> np.ndarray:
    kp = np.ascontiguousarray(keyframe_poses, np.float32).reshape(-1, 4, 4)
    pn = np.ascontiguousarray(pose_new, np.float32)
    out = np.zeros(max(len(kp), 1), np.int32)
    n = ctypes.c_int(0)
    _lib.check(_lib.load().bt_select_keyframes(_lib.ptr(pn), _lib.ptr(kp), len(kp), max_BA_frames, _lib.ptr(out), ctypes.byref(n)), "bt_select_keyframes")
    return out[:n.value].copy()


def rigid_transform(pts1, pts2) -> np.ndarray:
    a, b = np.ascontiguousarray(pts1, np.float32).reshape(-1, 3), np.ascontiguousarray(pts2, np.float32).reshape(-1, 3)
    out = np.zeros((4, 4), np.float32)
    _lib.check(_lib.load().bt_rigid_transform(_lib.ptr(a), _lib.ptr(b), len(a), _lib.ptr(out)), "bt_rigid_transform")
    return out


def lfnet_parse_reply(parts, roi):
    """parts: the three byte strings of the LF-Net server's reply; roi = (umin, umax, vmin, vmax).  Returns (kpts [n,2] float32 in image
    pixels, desc [n,dim] float32 view of part 2)."""
    info, kp, desc = (bytes(p) for p in parts)
    kpts, n, dim = _parse_reply(info, kp, len(desc), roi)
    return kpts, np.frombuffer(desc, np.float32).reshape(n, dim)


def lfnet_reply_keypoints(n: int, dim: int, kpts_400, roi) -> np.ndarray:
    """The keypoints of a reply with n rows of dim-dimensional descriptors whose keypoint part is kpts_400 (n x (x, y) float32 in the
    400 x 400 network input), in image pixels: lfnet_parse_reply's transform for a source whose descriptors never leave the device."""
    kp = np.ascontiguousarray(kpts_400, np.float32).reshape(-1)
    return _parse_reply(np.array([n, dim], np.int32).tobytes(), kp.tobytes(), 4 * n * dim, roi)[0]


def _parse_reply(info: bytes, kp: bytes, desc_bytes: int, roi):
    n_guess = max(len(kp) // 8, 1)
    out = np.zeros((n_guess, 2), np.float32)
    n, dim = ctypes.c_int(0), ctypes.c_int(0)
    _lib.check(_lib.load().bt_lfnet_parse_reply(info, len(info), kp, len(kp), desc_bytes, _lib.i32s(roi), _lib.ptr(out), n_guess, ctypes.byref(n),
                                                ctypes.byref(dim)), "bt_lfnet_parse_reply")
    return out[:n.value], n.value, dim.value


class Tracks:
    """Map-point bookkeeping (`SiftManager::updateFramePairMapPoints` / `findCorresByMapPoints`, FeatureManager.cpp:448-520)."""

    def __init__(self):
        self.lib = _lib.load()
        self.h = _lib.Handle("bt_tracks_create", "bt_tracks_destroy")

    def close(self):
        self.h.close()

    def update_pair(self, frame_a: int, frame_b: int, uv, is_inlier=None):
        uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 4)
        inl = None if is_inlier is None else np.ascontiguousarray(is_inlier, np.uint8)
        _lib.check(self.lib.bt_tracks_update_pair(self.h, frame_a, frame_b, _lib.ptr(uv), _lib.ptr(inl), len(uv)), "bt_tracks_update_pair")

    def propagate(self, frame_a: int, frame_b: int, existing_uv, capacity: int = 65536) -> np.ndarray:
        ex = np.ascontiguousarray(existing_uv, np.float32).reshape(-1, 4)
        out = np.zeros((capacity, 4), np.float32)
        n = ctypes.c_int(0)
        _lib.check(self.lib.bt_tracks_propagate(self.h, frame_a, frame_b, _lib.ptr(ex), len(ex), _lib.ptr(out), capacity, ctypes.byref(n)),
                   "bt_tracks_propagate")
        return out[:n.value].copy()

    def forget_frame(self, frame: int):
        _lib.check(self.lib.bt_tracks_forget_frame(self.h, frame), "bt_tracks_forget_frame")

    def stats(self):
        a, b = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(self.lib.bt_tracks_stats(self.h, ctypes.byref(a), ctypes.byref(b)), "bt_tracks_stats")
        return a.value, b.value


def ba_gate(n_edges_newframe: int, min_fm_edges_newframe: int = 10) -> bool:
    """Bundler::optimizeGPU's gate (/root/reference/src/Bundler.cpp:343-347): False = Frame::NO_BA, the optimizer is not called."""
    return bool(_lib.load().bt_ba_gate(n_edges_newframe, min_fm_edges_newframe))


def pose_text(cur_in_model) -> str:
    """Bundler::saveNewframeResult's pose record (Bundler.cpp:362-378): ob_in_cam = inverse(cur_in_model), printed like Eigen prints it."""
    p = np.ascontiguousarray(cur_in_model, np.float32)
    buf = ctypes.create_string_buffer(1024)
    _lib.check(_lib.load().bt_pose_format(_lib.ptr(p), buf, 1024), "bt_pose_format")
    return buf.value.decode()


def save_pose_txt(path: str, cur_in_model) -> None:
    p = np.ascontiguousarray(cur_in_model, np.float32)
    _lib.check(_lib.load().bt_pose_write_txt(path.encode(), _lib.ptr(p)), "bt_pose_write_txt")
