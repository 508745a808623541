"""Pose accuracy as BundleTrack is judged: ADD and ADD-S per frame (the reference's scripts/Utils.py add / adi) on the device, and their
VOCap AUC (scripts/eval_ycbineoat.py) on the host.  A thin ctypes mirror of bt_pose_metrics / bt_vocap (include/bundletrack_b200.h).
Poses are ob_in_cam (model -> camera), the matrices poses/<id>.txt holds; `ob_in_cam` turns the tracker's cam -> model poses into them."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib


def ob_in_cam(cam_in_model) -> np.ndarray:
    """The tracker's cam -> model poses (bt_tracker_end_frame's pose_out, [4,4] or [F,4,4]) as float64 ob_in_cam = inverse(cam_in_model),
    the matrix Bundler::saveNewframeResult records."""
    return np.linalg.inv(np.asarray(cam_in_model, np.float64))


def vocap(err, max_err: float = 0.1) -> float:
    """Area under the accuracy-threshold curve of the errors up to max_err, divided by max_err (the paper's tables print it x 100)."""
    e = np.ascontiguousarray(np.asarray(err, np.float64).reshape(-1))
    out = ctypes.c_double(0.0)
    _lib.check(_lib.load().bt_vocap(e.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(e.size), ctypes.c_double(max_err), ctypes.byref(out)), "bt_vocap")
    return out.value


def _poses(p, what: str) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(p, np.float64))
    if a.shape[-2:] != (4, 4):
        raise ValueError(f"{what}: expected [F,4,4] poses, got {a.shape}")
    return a.reshape(-1, 4, 4)


class PoseMetrics:
    """ADD / ADD-S of many frames in one device call.  Scratch for max_pts model points and max_frames frames per call is reserved here."""

    def __init__(self, max_pts: int, max_frames: int, device: int = 0, stream: int = 0, ctx=None):
        self.lib = _lib.load()
        self.stream = ctypes.c_void_p(stream)
        self.device = device
        self._own = ctx is None
        self.ctx = ctypes.c_void_p() if ctx is None else ctx
        if self._own:
            _lib.check(self.lib.bt_ctx_create(ctypes.byref(self.ctx), ctypes.c_int(device)), "bt_ctx_create")
        _lib.check(self.lib.bt_metrics_reserve(self.ctx, ctypes.c_int(max_pts), ctypes.c_int(max_frames)), "bt_metrics_reserve")

    def close(self):
        if self._own and self.ctx:
            self.lib.bt_ctx_destroy(self.ctx)
            self.ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __call__(self, model_pts, pred, gt):
        """model_pts: [N,3] float64 (numpy, or a CUDA tensor kept on the device between calls); pred, gt: [F,4,4] ob_in_cam.
        Returns (add, adds): float64 numpy [F], metres."""
        import torch
        dev = torch.device("cuda", self.device)
        pts = model_pts if isinstance(model_pts, torch.Tensor) else torch.from_numpy(np.asarray(model_pts, np.float64))
        pts = pts.to(device=dev, dtype=torch.float64).reshape(-1, 3).contiguous()
        P, G = _poses(pred, "pred"), _poses(gt, "gt")
        if len(P) != len(G):
            raise ValueError(f"{len(P)} predicted poses but {len(G)} ground-truth poses")
        F = len(P)
        add = torch.empty(F, dtype=torch.float64, device=dev)
        adds = torch.empty(F, dtype=torch.float64, device=dev)
        _lib.check(self.lib.bt_pose_metrics(self.ctx, ctypes.c_void_p(pts.data_ptr()), ctypes.c_int(pts.shape[0]), P.ctypes.data_as(ctypes.c_void_p),
                                            G.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(F), ctypes.c_void_p(add.data_ptr()),
                                            ctypes.c_void_p(adds.data_ptr()), self.stream), "bt_pose_metrics")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        return add.cpu().numpy(), adds.cpu().numpy()


def pose_metrics(model_pts, pred, gt, device: int = 0):
    """One-shot ADD / ADD-S (float64 numpy [F], metres) of ob_in_cam poses pred against gt over the model points [N,3]."""
    n = int(np.prod(np.shape(model_pts))) // 3
    f = len(_poses(pred, "pred"))
    m = PoseMetrics(max(n, 1), max(f, 1), device=device)
    try:
        return m(model_pts, pred, gt)
    finally:
        m.close()
