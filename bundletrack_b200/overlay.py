"""Tracking overlays: the reference's LOG frames (Bundler::saveNewframeResult with `LOG: 1`, src/Bundler.cpp:379-411) drawn on the device.  A
thin ctypes mirror of bt_overlay_reserve / bt_voxel_downsample / bt_pose_overlay (include/bundletrack_b200.h):

- load_obj_points: the model's points as pcl::io::loadOBJFile reads them (the `v` lines, in file order);
- Overlay: the model voxel-gridded once at 1.5 cm (DataLoader.cpp:92, 316), then per frame the model under the tracked pose, voxel-gridded at
  1 cm, projected and stamped onto the frame's colour dimmed outside the object mask (Utils::drawProjectPoints, Utils.cpp:216-226), plus the
  masked colour_raw image;
- write_log_frame: the frame id label (cv::putText) and the three files the reference writes, through OpenCV as the reference does."""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _lib

MODEL_LEAF = 0.015          # DataLoader.cpp:92, 316
TILE = 2048                 # points per tile of the device grid (overlay.cu kTile): clouds of TILE +- 1 points cross a tile boundary


def load_obj_points(path: str) -> np.ndarray:
    """float32 [n,3]: x, y, z of every `v` line of the OBJ file in file order.  Values after the third on a `v` line (vertex colours) are
    ignored; `vn`, `vt`, `f`, comments and every other line add no points."""
    pts = []
    with open(path) as f:
        for k, line in enumerate(f, 1):
            t = line.split()
            if not t or t[0] != "v":
                continue
            if len(t) < 4:
                raise ValueError(f"{path}:{k}: a vertex line needs x, y and z")
            pts.append((float(t[1]), float(t[2]), float(t[3])))
    if not pts:
        raise ValueError(f"{path}: no vertex")
    return np.asarray(pts, np.float64).astype(np.float32)


class VoxelGrid(_lib.Facade):
    """bt_voxel_downsample: PCL's VoxelGrid of many float32 [n,3] device clouds in one asynchronous call.  Scratch for max_frames clouds of
    max_pts points is reserved here (or on `ctx`, shared with an Overlay)."""

    def __init__(self, max_pts: int, max_frames: int = 1, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device = device
        self.reserve(max_pts, max_frames)

    def reserve(self, max_pts: int, max_frames: int) -> None:
        _lib.check(self.lib.bt_overlay_reserve(self.ctx, max_pts, max_frames), "bt_overlay_reserve")

    def enqueue(self, clouds, leaf: float, outs, n_out) -> None:
        """clouds / outs: float32 [n_c,3] CUDA tensors (outs with room for n_c rows); n_out: int32 CUDA tensor [len(clouds)].  Asynchronous."""
        _lib.check(self.lib.bt_voxel_downsample(self.ctx, len(clouds), _lib.ptrs(clouds), _lib.i32s([c.shape[0] for c in clouds]), leaf, _lib.ptrs(outs),
                                                _lib.ptr(n_out), self.stream), "bt_voxel_downsample")

    def __call__(self, clouds, leaf: float):
        """Each cloud (numpy or CUDA, [n,3]) voxel-gridded at leaf: a list of float32 numpy [m,3]; synchronises the stream."""
        import torch
        dev = torch.device("cuda", self.device)
        cl = [(c if isinstance(c, torch.Tensor) else torch.from_numpy(np.asarray(c, np.float32))).to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
              for c in clouds]
        outs = [torch.empty_like(c) for c in cl]
        n_out = torch.empty(len(cl), dtype=torch.int32, device=dev)
        torch.cuda.current_stream(dev).synchronize()        # the uploads are done before the library's stream reads them
        self.enqueue(cl, leaf, outs, n_out)
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        counts = n_out.cpu().numpy()
        return [o[:int(k)].cpu().numpy() for o, k in zip(outs, counts)]


class Overlay:
    """The LOG frame of a tracked object.  model_pts: the OBJ's points (load_obj_points), voxel-gridded here once at MODEL_LEAF on the device;
    K: 3 x 3 or (fx, fy, cx, cy); frames of H x W; up to max_frames frames per render call.  leaf=None draws model_pts as given.  Device
    work runs on `stream`."""

    def __init__(self, model_pts, K, H: int, W: int, max_frames: int = 1, device: int = 0, stream: int = 0, ctx=None, leaf: float = MODEL_LEAF):
        import torch
        raw = np.ascontiguousarray(np.asarray(model_pts, np.float32).reshape(-1, 3))
        if len(raw) == 0:
            raise ValueError("the model has no point")
        self.K = _lib.intrinsics(K)
        self.H, self.W, self.max_frames, self.device = int(H), int(W), int(max_frames), device
        self.grid = VoxelGrid(len(raw), 1, device=device, stream=stream, ctx=ctx)
        self.lib, self.ctx, self.stream = self.grid.lib, self.grid.ctx, self.grid.stream
        self.model = raw if leaf is None else self.grid([raw], leaf)[0]
        self.grid.reserve(max(len(self.model), 1), self.max_frames)
        dev = torch.device("cuda", device)
        self.model_dev = torch.from_numpy(self.model).to(dev)
        torch.cuda.current_stream(dev).synchronize()

    def close(self):
        self.grid.close()

    def render(self, cur_in_model, colour, fg, viz_out, raw_out=None) -> None:
        """Draw len(colour) frames in one asynchronous call on the stream.  cur_in_model: [F,4,4] (or [4,4]) the tracker's cam -> model poses;
        colour: device uint8 [H,W,3] BGR per frame (the original colour); fg: device uint8 [H,W] per frame (Frame::_fg_mask, or a device
        address); viz_out / raw_out: device uint8 [H,W,3] per frame (raw_out may be None)."""
        P = np.ascontiguousarray(np.asarray(cur_in_model, np.float32).reshape(-1, 16))
        F = len(colour)
        if len(P) != F or len(fg) != F or len(viz_out) != F or (raw_out is not None and len(raw_out) != F):
            raise ValueError(f"{len(P)} poses, {F} colour images, {len(fg)} masks, {len(viz_out)} viz outputs: they must agree")
        if self.model.shape[0] == 0:
            raise ValueError("the voxel-gridded model is empty (no finite point)")
        _lib.check(self.lib.bt_pose_overlay(self.ctx, F, _lib.ptr(self.model_dev), len(self.model), _lib.ptr(P), *self.K, _lib.ptrs(colour), _lib.ptrs(fg),
                                            self.H, self.W, _lib.ptrs(viz_out), None if raw_out is None else _lib.ptrs(raw_out), self.stream), "bt_pose_overlay")

    def render_host(self, cur_in_model, colour, fg):
        """render() on host or device images; returns (viz, raw) as uint8 numpy [F,H,W,3] and synchronises the stream."""
        import torch
        dev = torch.device("cuda", self.device)
        to = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).to(dev)
        col = [to(c) for c in colour]
        m = [to(f) for f in fg]
        viz = [torch.empty((self.H, self.W, 3), dtype=torch.uint8, device=dev) for _ in col]
        raw = [torch.empty_like(v) for v in viz]
        torch.cuda.current_stream(dev).synchronize()
        self.render(cur_in_model, col, m, viz, raw)
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        return np.stack([v.cpu().numpy() for v in viz]), np.stack([r.cpu().numpy() for r in raw])


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise RuntimeError("writing LOG frames needs OpenCV's Python module (cv2): the reference draws the label and encodes the JPEG and PNG "
                           "files with OpenCV, and no other encoder gives the same bytes") from e
    return cv2


def label(viz: np.ndarray, id_str: str) -> np.ndarray:
    """A copy of viz with the frame id drawn as the reference draws it: cv::putText(id, {5, 30}, FONT_HERSHEY_PLAIN, 2, {255, 0, 0}, 1, 8)."""
    cv2 = _cv2()
    img = np.ascontiguousarray(viz, np.uint8).copy()
    cv2.putText(img, id_str, (5, 30), cv2.FONT_HERSHEY_PLAIN, 2, (255, 0, 0), 1, 8, False)
    return img


def write_log_frame(debug_dir: str, id_str: str, viz: np.ndarray, raw: np.ndarray) -> None:
    """The label on viz, then <debug_dir>/<id>/color_viz.jpg and <debug_dir>/color_viz/<id>_color_viz.jpg (JPEG quality 80) and
    <debug_dir>/color_raw/<id>_color_raw.png (the masked colour).  Directories are created, color_viz/ included (the reference never creates
    it, so its write there fails on a fresh debug_dir)."""
    cv2 = _cv2()
    img = label(viz, id_str)
    jobs = ((os.path.join(debug_dir, id_str, "color_viz.jpg"), img, [cv2.IMWRITE_JPEG_QUALITY, 80]),
            (os.path.join(debug_dir, "color_viz", f"{id_str}_color_viz.jpg"), img, [cv2.IMWRITE_JPEG_QUALITY, 80]),
            (os.path.join(debug_dir, "color_raw", f"{id_str}_color_raw.png"), np.ascontiguousarray(raw, np.uint8), []))
    for path, a, params in jobs:
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if not cv2.imwrite(path, a, params):
            raise OSError(f"cv2.imwrite could not write {path}")


# ---- match images: the reference's LOG correspondence drawings (SiftManager::vizCorresBetween, src/FeatureManager.cpp:760-796)

RNG_DEFAULT = 0xFFFFFFFF            # cv::theRNG()'s state when a process starts
JPEG_MAX_SIDE = 65500               # libjpeg's limit: cv2.imwrite returns False past it


def rng_after(state: int, n_matches: int) -> int:
    """cv::RNG's state after the colours of an image of n_matches matches (three draws per match)."""
    for _ in range(3 * int(n_matches)):
        state = ((state & 0xFFFFFFFF) * 4164903690 + (state >> 32)) & 0xFFFFFFFFFFFFFFFF
    return state


def match_image_shape(roi_a, roi_b):
    """(rows, cols) of the match image of two ROIs (umin, umax, vmin, vmax)."""
    rows, cols = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().bt_match_viz_shape(_lib.i32s(roi_a), _lib.i32s(roi_b), ctypes.byref(rows), ctypes.byref(cols)), "bt_match_viz_shape")
    return rows.value, cols.value


def match_image_path(debug_dir: str, new_id: str, id_a: str, id_b: str, stage: str) -> str:
    """<debug_dir>/<new frame id>/<A id>_match_<B id>_<stage>.jpg, the reference's name for a match image."""
    return os.path.join(debug_dir, new_id, f"{id_a}_match_{id_b}_{stage}.jpg")


class MatchViz(_lib.Facade):
    """bt_match_viz: match images drawn on the device, many per asynchronous call.  Scratch for max_images images and max_matches matches
    per call is reserved here (or on `ctx`)."""

    def __init__(self, max_images: int = 1, max_matches: int = 4096, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.device = device
        _lib.check(self.lib.bt_match_viz_reserve(self.ctx, max_images, max_matches), "bt_match_viz_reserve")

    def draw(self, images, outs) -> None:
        """images: (colour_a, roi_a, colour_b, roi_b, uv, rng_state) per image; colours are device uint8 [H,W,3], uv a device float32 [n,4]
        (uA, vA, uB, vB) or None; outs: device uint8 [rows, cols, 3] per image (match_image_shape).  Asynchronous on the stream."""
        n = len(images)
        if len(outs) != n:
            raise ValueError(f"{n} images and {len(outs)} outputs")
        descs = (_lib.MatchVizDesc * n)()
        for k, (d, (ca, ra, cb, rb, uv, st), o) in enumerate(zip(descs, images, outs)):
            self._check(k, ca, ra, cb, rb, uv, o)
            d.colour_a, d.H_a, d.W_a = ca.data_ptr(), ca.shape[0], ca.shape[1]
            d.colour_b, d.H_b, d.W_b = cb.data_ptr(), cb.shape[0], cb.shape[1]
            d.roi_a[:] = [int(v) for v in ra]
            d.roi_b[:] = [int(v) for v in rb]
            d.uv, d.n = (None, 0) if uv is None or uv.shape[0] == 0 else (uv.data_ptr(), uv.shape[0])
            d.rng_state = int(st)
        _lib.check(self.lib.bt_match_viz(self.ctx, n, descs, _lib.ptrs(outs), self.stream), "bt_match_viz")

    def _check(self, k, ca, ra, cb, rb, uv, out) -> None:
        """The library reads these through raw device pointers: each must be a contiguous CUDA tensor on this device, of the dtype and
        shape the call expects."""
        import torch

        def dev_tensor(x, what, dtype):
            if not isinstance(x, torch.Tensor) or not x.is_cuda or x.device.index != self.device:
                raise ValueError(f"image {k}: {what} must be a CUDA tensor on device {self.device}")
            if x.dtype != dtype or not x.is_contiguous():
                raise ValueError(f"image {k}: {what} must be a contiguous {dtype} tensor, not {x.dtype}{'' if x.is_contiguous() else ' (strided)'}")

        for c, what in ((ca, "colour_a"), (cb, "colour_b")):
            dev_tensor(c, what, torch.uint8)
            if c.dim() != 3 or c.shape[2] != 3:
                raise ValueError(f"image {k}: {what} must be [H, W, 3], not {list(c.shape)}")
        if uv is not None:
            dev_tensor(uv, "uv", torch.float32)
            if uv.dim() != 2 or uv.shape[1] != 4:
                raise ValueError(f"image {k}: uv must be [n, 4] (uA, vA, uB, vB), not {list(uv.shape)}")
        dev_tensor(out, "out", torch.uint8)
        want = (*match_image_shape(ra, rb), 3)
        if tuple(out.shape) != want:
            raise ValueError(f"image {k}: out must be {list(want)}, not {list(out.shape)}")

    def draw_host(self, images):
        """draw() on host or device inputs; returns uint8 numpy images and synchronises the stream."""
        import torch
        dev = torch.device("cuda", self.device)
        to = lambda a, dt: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dt))).to(dev).contiguous()
        ims = []
        for ca, ra, cb, rb, uv, st in images:
            u = None if uv is None or len(uv) == 0 else to(np.asarray(uv, np.float32).reshape(-1, 4), np.float32)
            ims.append((to(ca, np.uint8), ra, to(cb, np.uint8), rb, u, st))
        outs = [torch.empty((*match_image_shape(ra, rb), 3), dtype=torch.uint8, device=dev) for _, ra, _, rb, _, _ in ims]
        torch.cuda.current_stream(dev).synchronize()
        self.draw(ims, outs)
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        return [o.cpu().numpy() for o in outs]


def write_match_image(path: str, img: np.ndarray) -> bool:
    """imwrite(path, img, JPEG quality 80) as vizCorresBetween does.  An image wider or taller than JPEG allows is not written, as
    cv::imwrite writes nothing for it: returns False (the caller reports it) instead of failing the run."""
    cv2 = _cv2()
    if max(img.shape[:2]) > JPEG_MAX_SIDE:
        return False
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if not cv2.imwrite(path, np.ascontiguousarray(img, np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 80]):
        raise OSError(f"cv2.imwrite could not write {path}")
    return True
