"""Pose accuracy as BundleTrack is judged: ADD and ADD-S per frame (the reference's scripts/Utils.py add / adi) on the device, and their
VOCap AUC (scripts/eval_ycbineoat.py) on the host.  A thin ctypes mirror of bt_pose_metrics / bt_vocap (include/bundletrack_b200.h).
Also the NOCS-REAL275 scores, an object model's accuracy against a reference mesh (SurfaceScore), and the DAVIS J and F scores of
object masks against ground-truth masks (MaskScore).
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
    _lib.check(_lib.load().bt_vocap(_lib.ptr(e), e.size, max_err, ctypes.byref(out)), "bt_vocap")
    return out.value


def _poses(p, what: str) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(p, np.float64))
    if a.shape[-2:] != (4, 4):
        raise ValueError(f"{what}: expected [F,4,4] poses, got {a.shape}")
    return a.reshape(-1, 4, 4)


class PoseMetrics(_lib.Facade):
    """ADD / ADD-S of many frames in one device call.  Scratch for max_pts model points and max_frames frames per call is reserved here."""

    def __init__(self, max_pts: int, max_frames: int, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device = device
        _lib.check(self.lib.bt_metrics_reserve(self.ctx, max_pts, max_frames), "bt_metrics_reserve")

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
        _lib.check(self.lib.bt_pose_metrics(self.ctx, _lib.ptr(pts), pts.shape[0], _lib.ptr(P), _lib.ptr(G), F, _lib.ptr(add), _lib.ptr(adds), self.stream),
                   "bt_pose_metrics")
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


# NOCS-REAL275 (the reference's 6-PACK benchmark, scripts/benchmark.py).  Class ids are benchmark.py's synset indices; the y-axis rule
# applies to bottle, bowl and can only (the benchmark passes handle_visibility = 1 for every mug).
NOCS_CLASSES = ("bottle", "bowl", "camera", "can", "laptop", "mug")
NOCS_SYMMETRIC = (1, 2, 4)


def _i32(a, n: int, what: str) -> np.ndarray:
    v = np.ascontiguousarray(np.asarray(a).reshape(-1).astype(np.int32))
    if v.size != n:
        raise ValueError(f"{what}: expected {n} values, got {v.size}")
    return v


def _f64(a, n: int, what: str) -> np.ndarray:
    v = np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1))
    if v.size != n:
        raise ValueError(f"{what}: expected {n} values, got {v.size}")
    return v


class NocsMetrics(_lib.Facade):
    """theta (degrees), shift (mm) and IoU of many NOCS records in one device call (bt_nocs_metrics); room for max_records per call."""

    def __init__(self, max_records: int, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device = device
        _lib.check(self.lib.bt_nocs_reserve(self.ctx, max_records), "bt_nocs_reserve")

    def __call__(self, pred, gt, corners, symmetric):
        """pred, gt: [N,4,4] with translations in mm, as the benchmark compares them; corners: [N,8,3] (or [8,3] for all); symmetric: [N]
        flags.  Returns (theta_deg, shift, iou): float64 numpy [N]."""
        import torch
        dev = torch.device("cuda", self.device)
        P, G = _poses(pred, "pred"), _poses(gt, "gt")
        if len(P) != len(G):
            raise ValueError(f"{len(P)} predicted poses but {len(G)} ground-truth poses")
        N = len(P)
        C = np.asarray(corners, np.float64)
        if C.shape == (8, 3):
            C = np.broadcast_to(C, (N, 8, 3))
        C = _f64(C, 24 * N, "corners")
        S = _i32(symmetric, N, "symmetric")
        out = torch.empty((3, N), dtype=torch.float64, device=dev)
        _lib.check(self.lib.bt_nocs_metrics(self.ctx, _lib.ptr(P), _lib.ptr(G), _lib.ptr(C), _lib.ptr(S), N, *(_lib.ptr(o) for o in out), self.stream),
                   "bt_nocs_metrics")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        o = out.cpu().numpy()
        return o[0].copy(), o[1].copy(), o[2].copy()


def nocs_metrics(pred, gt, corners, symmetric, device: int = 0):
    """One-shot bt_nocs_metrics: (theta_deg, shift, iou), float64 numpy [N]."""
    n = len(_poses(pred, "pred"))
    m = NocsMetrics(max(n, 1), device=device)
    try:
        return m(pred, gt, corners, symmetric)
    finally:
        m.close()


def nocs_score(cls, scored, theta_deg, shift, iou):
    """benchmark.py's aggregation (bt_nocs_score, host code).  Returns (per_class [6,4], overall [4]); columns: 5 deg 5 cm fraction, IoU25
    fraction, mean theta (degrees), mean shift (mm).  The benchmark prints fractions x 100 and the shift / 10 (cm)."""
    c = np.ascontiguousarray(np.asarray(cls).reshape(-1).astype(np.int32))
    n = c.size
    s = _i32(scored, n, "scored")
    t, d, u = _f64(theta_deg, n, "theta_deg"), _f64(shift, n, "shift"), _f64(iou, n, "iou")
    per = np.zeros((6, 4), np.float64)
    ov = np.zeros(4, np.float64)
    p = _lib.ptr
    _lib.check(_lib.load().bt_nocs_score(p(c), p(s), p(t), p(d), p(u), n, p(per), p(ov)), "bt_nocs_score")
    return per, ov


# Object model accuracy (DESIGN.md §3.15): both meshes sampled uniformly by area on the device, exact nearest distances both ways, and
# the scores on the host.  The meshes are compared in the frame they are given in: nothing aligns them, so a tracking error shows.
SCORE_KEYS = ("accuracy", "completeness", "chamfer", "median_model_to_ref", "p95_model_to_ref", "median_ref_to_model", "p95_ref_to_model")


def surface_score(d_ab, d_ba, taus=(0.002, 0.005, 0.01)) -> dict:
    """bt_surface_score (host code) of the model -> reference distances d_ab and the reference -> model distances d_ba (metres): accuracy
    (mean d_ab), completeness (mean d_ba), chamfer, the median and p95 of each direction, and per tau precision, recall and F-score."""
    a = np.ascontiguousarray(np.asarray(d_ab, np.float64).reshape(-1))
    b = np.ascontiguousarray(np.asarray(d_ba, np.float64).reshape(-1))
    t = np.ascontiguousarray(np.asarray(taus, np.float64).reshape(-1))
    out = np.zeros(len(SCORE_KEYS) + 3 * t.size, np.float64)
    _lib.check(_lib.load().bt_surface_score(_lib.ptr(a), a.size, _lib.ptr(b), b.size, _lib.ptr(t), t.size, _lib.ptr(out)), "bt_surface_score")
    res = dict(zip(SCORE_KEYS, out[:len(SCORE_KEYS)].tolist()))
    per = out[len(SCORE_KEYS):].reshape(-1, 3)
    res.update(taus=t.tolist(), precision=per[:, 0].tolist(), recall=per[:, 1].tolist(), fscore=per[:, 2].tolist())
    return res


class SurfaceScore(_lib.Facade):
    """A mesh scored against a reference mesh on the device.  Room for meshes of up to max_faces faces and max_samples samples per side
    is reserved here."""

    def __init__(self, max_faces: int, max_samples: int, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device = device
        _lib.check(self.lib.bt_surface_reserve(self.ctx, max_faces, max_samples), "bt_surface_reserve")

    def _dev(self, x, dtype, what: str):
        import torch
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        t = t.to(device=torch.device("cuda", self.device), dtype=dtype).contiguous()
        if t.dim() != 2 or t.shape[1] != 3:
            raise ValueError(f"{what}: expected [n, 3], got {list(t.shape)}")
        return t

    def sample(self, verts, faces, n_samples: int, seed: int = 0):
        """n_samples points uniform by area on the mesh (verts [V,3], faces [F,3] vertex indices; numpy or CUDA tensors): a float64 CUDA
        tensor [n_samples, 3], bit-reproducible for a seed."""
        import torch
        v = self._dev(verts, torch.float64, "verts")
        f = self._dev(faces, torch.int32, "faces")
        out = torch.empty((int(n_samples), 3), dtype=torch.float64, device=v.device)
        _lib.check(self.lib.bt_mesh_sample(self.ctx, _lib.ptr(v), v.shape[0], _lib.ptr(f), f.shape[0], int(n_samples), int(seed), _lib.ptr(out),
                                           self.stream), "bt_mesh_sample")
        return out

    def distances(self, a, b):
        """(d_ab, d_ba): float64 numpy, d_ab[i] = min_j |a_i - b_j| and d_ba[j] = min_i |b_j - a_i|, exact, for point sets a [n,3] and b [m,3]."""
        import torch
        A, B = self._dev(a, torch.float64, "a"), self._dev(b, torch.float64, "b")
        d_ab = torch.empty(A.shape[0], dtype=torch.float64, device=A.device)
        d_ba = torch.empty(B.shape[0], dtype=torch.float64, device=A.device)
        _lib.check(self.lib.bt_surface_distances(self.ctx, _lib.ptr(A), A.shape[0], _lib.ptr(B), B.shape[0], _lib.ptr(d_ab), _lib.ptr(d_ba), self.stream),
                   "bt_surface_distances")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        return d_ab.cpu().numpy(), d_ba.cpu().numpy()

    def score(self, model_verts, model_faces, ref_verts, ref_faces, n_samples: int = 100_000, taus=(0.002, 0.005, 0.01), seed: int = 0) -> dict:
        """Both meshes sampled with n_samples points and the same seed, then surface_score of the distances both ways, plus n_samples."""
        a = self.sample(model_verts, model_faces, n_samples, seed)
        b = self.sample(ref_verts, ref_faces, n_samples, seed)
        res = surface_score(*self.distances(a, b), taus)
        res["n_samples"] = int(n_samples)
        return res


# Mask accuracy (DESIGN.md §3.16): the DAVIS region similarity J and boundary accuracy F per frame on the device, and their per-sequence
# statistics on the host, in the DAVIS toolkit's CSV order.
MASK_SCORE_KEYS = ("J&F-Mean", "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay")
MASK_COUNT_KEYS = ("inter", "union", "n_pred", "n_gt", "m_pred", "m_gt")


def mask_score(j, f) -> dict:
    """bt_mask_score (host code) of one sequence's per-frame J and F: the mean, the recall (the fraction of frames above 0.5) and the decay
    of each, and J&F, the mean of the two means, under MASK_SCORE_KEYS."""
    a = np.ascontiguousarray(np.asarray(j, np.float64).reshape(-1))
    b = np.ascontiguousarray(np.asarray(f, np.float64).reshape(-1))
    if a.size != b.size:
        raise ValueError(f"mask_score: {a.size} J values and {b.size} F values")
    out = np.zeros(len(MASK_SCORE_KEYS), np.float64)
    _lib.check(_lib.load().bt_mask_score(_lib.ptr(a), _lib.ptr(b), a.size, _lib.ptr(out)), "bt_mask_score")
    return dict(zip(MASK_SCORE_KEYS, out.tolist()))


class MaskScore(_lib.Facade):
    """J and F of predicted masks against ground-truth masks on the device.  Room for calls of up to max_frames frames of h x w is reserved
    here; longer inputs are scored max_frames at a time."""

    def __init__(self, max_frames: int, h: int, w: int, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device, self.max_frames = device, int(max_frames)
        _lib.check(self.lib.bt_mask_reserve(self.ctx, int(max_frames), int(h), int(w)), "bt_mask_reserve")

    @staticmethod
    def _frames(x, what: str):
        import torch
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        if t.dtype == torch.bool:
            t = t.view(torch.uint8)
        if t.dtype != torch.uint8 or t.dim() != 3:
            raise ValueError(f"{what}: expected uint8 or bool [F, H, W], got {t.dtype} {list(t.shape)}")
        return t

    def __call__(self, pred, gt, bound_th: float = 0.008, counts: bool = False):
        """(j, f), float64 numpy [F], of pred against gt (numpy or CUDA, uint8 or bool [F, H, W], foreground = non-zero); with counts=True
        also the int64 [F, 6] counts |P & G|, |P | G|, n_P, n_G, m_P, m_G (MASK_COUNT_KEYS)."""
        import torch
        P, G = self._frames(pred, "pred"), self._frames(gt, "gt")
        if P.shape != G.shape:
            raise ValueError(f"pred {list(P.shape)} and gt {list(G.shape)} differ")
        n, h, w = P.shape
        dev = torch.device("cuda", self.device)
        j = torch.empty(n, dtype=torch.float64, device=dev)
        f = torch.empty(n, dtype=torch.float64, device=dev)
        c = torch.empty((n, 6), dtype=torch.int64, device=dev) if counts else None
        held = []                                  # each call's inputs, alive until the stream has read them
        for s in range(0, n, self.max_frames):
            e = min(n, s + self.max_frames)
            p, g = P[s:e].to(dev).contiguous(), G[s:e].to(dev).contiguous()
            held += [p, g]
            _lib.check(self.lib.bt_mask_metrics(self.ctx, _lib.ptr(p), _lib.ptr(g), e - s, h, w, float(bound_th), _lib.ptr(j[s:]), _lib.ptr(f[s:]),
                                                _lib.ptr(c[s:]) if counts else None, self.stream), "bt_mask_metrics")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        out = (j.cpu().numpy(), f.cpu().numpy())
        return out + (c.cpu().numpy(),) if counts else out

    def objects(self, pred, gt, n_objects: int, void_value: int = 255, bound_th: float = 0.008, counts: bool = False):
        """(j, f), float64 numpy [F, n_objects], of label maps (uint8 [F, H, W] object ids, numpy or CUDA): object k of frame i at [i, k - 1],
        scored on P = (pred == k) and G = (gt == k) with the pixels where gt == void_value removed from both (void_value -1: none), DAVIS
        2017's db_eval_iou / f_measure with void_pixels (bt_mask_metrics_objects).  counts=True also gives the int64 [F, n_objects, 6] counts.
        Each (frame, object) pair takes one of the max_frames reserved rows, so calls hold max_frames // n_objects frames."""
        import torch
        P, G = self._frames(pred, "pred"), self._frames(gt, "gt")
        if P.shape != G.shape:
            raise ValueError(f"pred {list(P.shape)} and gt {list(G.shape)} differ")
        n, h, w = P.shape
        k = int(n_objects)
        step = self.max_frames // k
        if step < 1:
            raise ValueError(f"{k} objects need {k} reserved rows per frame; max_frames is {self.max_frames}")
        dev = torch.device("cuda", self.device)
        j = torch.empty((n, k), dtype=torch.float64, device=dev)
        f = torch.empty((n, k), dtype=torch.float64, device=dev)
        c = torch.empty((n, k, 6), dtype=torch.int64, device=dev) if counts else None
        held = []
        for s in range(0, n, step):
            e = min(n, s + step)
            p, g = P[s:e].to(dev).contiguous(), G[s:e].to(dev).contiguous()
            held += [p, g]
            _lib.check(self.lib.bt_mask_metrics_objects(self.ctx, _lib.ptr(p), _lib.ptr(g), e - s, h, w, k, int(void_value), float(bound_th),
                                                        _lib.ptr(j[s:]), _lib.ptr(f[s:]), _lib.ptr(c[s:]) if counts else None, self.stream),
                       "bt_mask_metrics_objects")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        out = (j.cpu().numpy(), f.cpu().numpy())
        return out + (c.cpu().numpy(),) if counts else out
