"""Deterministic synthetic RGB-D tracking windows for the pose-graph hot path.

Shapes follow the reference's boundary types (SURVEY.md §8a/§8d):
  * depth   float32 [N, H, W]      metres, 0 = invalid (Frame::invalidatePixelsByMask leaves zeros,
                                   /root/reference/src/Frame.cpp:138-145)
  * normal  float32 [N, H, W, 4]   unit normal in the camera frame facing the camera, w = 0, zeros when invalid
                                   (/root/reference/src/cuda/CUDAImageUtil.cu:342-413 writes make_float4(n, 0))
  * poses   float32 [N, 4, 4]      row-major cam->model ("_pose_in_model", /root/reference/src/Frame.h:58)
  * corr    EntryJ[C]              {u32 imgIdx_i, u32 imgIdx_j, f32 pos_i[3], f32 pos_j[3]}, i < j
                                   (/root/reference/src/cuda/SIFTImageManager.h:44-59, built as in
                                   /root/reference/src/Bundler.cpp:298-324)
  * K       (fx, fy, cx, cy)       NOCS intrinsics (/root/reference/src/DataLoader.cpp:75-77)

The object is an ellipsoid rendered analytically (ray/quadric intersection), so depth and normals are exact
before the 1 mm depth noise is added.  Everything is numpy; nothing here touches the GPU or the oracle.
"""
from __future__ import annotations

import dataclasses
from typing import Optional

import numpy as np

NOCS_K = (591.0125, 590.16775, 322.525, 244.11084)

ENTRYJ_DTYPE = np.dtype(
    [("imgIdx_i", "<u4"), ("imgIdx_j", "<u4"), ("pos_i", "<f4", (3,)), ("pos_j", "<f4", (3,))]
)
assert ENTRYJ_DTYPE.itemsize == 32


def so3_exp(w: np.ndarray) -> np.ndarray:
    w = np.asarray(w, dtype=np.float64)
    th = np.linalg.norm(w)
    Kx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + Kx
    return np.eye(3) + np.sin(th) / th * Kx + (1 - np.cos(th)) / th ** 2 * (Kx @ Kx)


def se3(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def rot_geodesic(Ra: np.ndarray, Rb: np.ndarray) -> float:
    """Geodesic angle between two rotations; atan2 of the skew part keeps precision near 0 (arccos(trace) loses
    half the digits there, which matters at the 1e-4 rad gate with float32 inputs)."""
    D = np.asarray(Ra, np.float64).T @ np.asarray(Rb, np.float64)
    s = 0.5 * np.sqrt((D[2, 1] - D[1, 2]) ** 2 + (D[0, 2] - D[2, 0]) ** 2 + (D[1, 0] - D[0, 1]) ** 2)
    c = (np.trace(D) - 1.0) * 0.5
    return float(np.arctan2(s, c))


@dataclasses.dataclass
class Window:
    depth: np.ndarray        # [N,H,W] f32
    normal: np.ndarray       # [N,H,W,4] f32
    poses_init: np.ndarray   # [N,4,4] f32 row-major cam->model
    poses_gt: np.ndarray     # [N,4,4] f64
    corr: np.ndarray         # EntryJ[C]
    K: tuple                 # fx, fy, cx, cy
    radii: np.ndarray        # ellipsoid radii (model frame = camera-0 frame)
    ob_in_cam: np.ndarray    # [N,4,4] f64 object->camera

    @property
    def n_frames(self) -> int:
        return self.depth.shape[0]

    @property
    def H(self) -> int:
        return self.depth.shape[1]

    @property
    def W(self) -> int:
        return self.depth.shape[2]


def render_ellipsoid(radii, ob_in_cam, K, H, W, rng: Optional[np.random.Generator], depth_noise=0.001):
    """Depth + normal map of an ellipsoid with the given object->camera pose."""
    fx, fy, cx, cy = K
    u = (np.arange(W, dtype=np.float64) - cx) / fx
    v = (np.arange(H, dtype=np.float64) - cy) / fy
    dx, dy = np.meshgrid(u, v)
    d = np.stack([dx, dy, np.ones_like(dx)], -1)               # ray dirs, z = 1  => t = depth
    R = ob_in_cam[:3, :3]
    c = ob_in_cam[:3, 3]
    Q = R @ np.diag(1.0 / np.asarray(radii, dtype=np.float64) ** 2) @ R.T
    Qd = d @ Q.T
    A = np.einsum("hwk,hwk->hw", d, Qd)
    Qc = Q @ c
    B = -2.0 * (d @ Qc)
    Cc = float(c @ Qc) - 1.0
    disc = B * B - 4 * A * Cc
    hit = disc > 0
    t = np.where(hit, (-B - np.sqrt(np.where(hit, disc, 0.0))) / (2 * A), 0.0)
    hit &= t > 0.1
    P = d * t[..., None]
    n = (P - c) @ Q.T
    nn = np.linalg.norm(n, axis=-1, keepdims=True)
    n = np.where(nn > 0, n / np.where(nn > 0, nn, 1.0), 0.0)
    depth = np.where(hit, t, 0.0)
    if rng is not None and depth_noise > 0:
        depth = np.where(hit, depth + rng.normal(0.0, depth_noise, depth.shape), 0.0)
    normal = np.zeros((H, W, 4), dtype=np.float32)
    normal[..., :3] = np.where(hit[..., None], n, 0.0)
    return depth.astype(np.float32), normal


def _sample_pose(rng, z_range=(0.5, 1.0)):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    R = so3_exp(axis * rng.uniform(0, np.pi))
    z = rng.uniform(*z_range)
    c = np.array([rng.uniform(-0.08, 0.08) * z, rng.uniform(-0.06, 0.06) * z, z])
    return R, c


def make_window(
    seed: int,
    n_frames: int = 10,
    n_corr: int = 2000,
    H: int = 480,
    W: int = 640,
    K=NOCS_K,
    outlier_frac: float = 0.10,
    point_noise: float = 0.001,
    depth_noise: float = 0.001,
    rot_noise_deg: float = 1.0,
    trans_noise: float = 0.003,
    rel_rot_deg=(5.0, 40.0),
    occlusion: bool = False,
    render: bool = True,
) -> Window:
    """One tracking window (SURVEY.md §8d "Synthetic inputs").  Frame 0 is the gauge: its pose is exact."""
    rng = np.random.default_rng(np.uint64(0xB7) + np.uint64(seed))
    radii = rng.uniform(0.04, 0.12, size=3)
    R0, c0 = _sample_pose(rng)
    ob_in_cam = np.zeros((n_frames, 4, 4))
    ob_in_cam[0] = se3(R0, c0)
    for k in range(1, n_frames):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        ang = np.deg2rad(rng.uniform(*rel_rot_deg))
        Rk = so3_exp(axis * ang) @ ob_in_cam[k - 1][:3, :3]
        _, ck = _sample_pose(rng)
        ob_in_cam[k] = se3(Rk, ck)
    # model frame := camera-0 frame  =>  cam_k -> model = ob_in_cam_0 * inv(ob_in_cam_k)
    poses_gt = np.stack([ob_in_cam[0] @ np.linalg.inv(ob_in_cam[k]) for k in range(n_frames)])
    poses_init = poses_gt.copy()
    for k in range(1, n_frames):
        xi_r = rng.normal(0, np.deg2rad(rot_noise_deg), 3)
        xi_t = rng.normal(0, trans_noise, 3)
        poses_init[k] = poses_gt[k] @ se3(so3_exp(xi_r), xi_t)

    depth = np.zeros((n_frames, H, W), np.float32)
    normal = np.zeros((n_frames, H, W, 4), np.float32)
    if render:
        for k in range(n_frames):
            depth[k], normal[k] = render_ellipsoid(radii, ob_in_cam[k], K, H, W, rng, depth_noise)
            if occlusion:  # YCBInEOAT-style occluder: zero a random half-plane through the silhouette
                ys, xs = np.nonzero(depth[k] > 0)
                if len(xs):
                    px, py = xs.mean(), ys.mean()
                    th = rng.uniform(0, 2 * np.pi)
                    off = rng.uniform(0.2, 0.6) * max(np.ptp(xs), np.ptp(ys), 1)
                    yy, xx = np.mgrid[0:H, 0:W]
                    cut = (xx - px) * np.cos(th) + (yy - py) * np.sin(th) > off
                    depth[k][cut] = 0
                    normal[k][cut] = 0

    corr = make_correspondences(rng, radii, ob_in_cam, n_corr, K, H, W, outlier_frac, point_noise)
    return Window(depth, normal, poses_init.astype(np.float32), poses_gt, corr, tuple(K), radii, ob_in_cam)


def make_correspondences(rng, radii, ob_in_cam, n_corr, K, H, W, outlier_frac, point_noise):
    """3D-3D matches on the co-visible ellipsoid surface, spread over all i<j pairs, grouped pair by pair in the
    order Bundler::optimizeGPU emits them (/root/reference/src/Bundler.cpp:298-324)."""
    n_frames = ob_in_cam.shape[0]
    pairs = [(i, j) for i in range(n_frames) for j in range(i + 1, n_frames)]
    per = [n_corr // len(pairs) + (1 if p < n_corr % len(pairs) else 0) for p in range(len(pairs))]
    fx, fy, cx, cy = K
    out = np.zeros(n_corr, ENTRYJ_DTYPE)
    o = 0
    D = np.asarray(radii)
    for (i, j), m in zip(pairs, per):
        got = 0
        while got < m:
            # uniform directions scaled onto the ellipsoid (object frame)
            s = rng.normal(size=(4 * (m - got) + 16, 3))
            s /= np.linalg.norm(s, axis=1, keepdims=True)
            p_ob = s * D
            n_ob = s / D
            ok = np.ones(len(s), bool)
            pts = []
            for f in (i, j):
                R, c = ob_in_cam[f][:3, :3], ob_in_cam[f][:3, 3]
                pc = p_ob @ R.T + c
                nc = n_ob @ R.T
                ok &= np.einsum("nk,nk->n", nc, -pc) > 0.05 * np.linalg.norm(nc, axis=1) * np.linalg.norm(pc, axis=1)
                uu = pc[:, 0] * fx / pc[:, 2] + cx
                vv = pc[:, 1] * fy / pc[:, 2] + cy
                ok &= (uu >= 0) & (uu <= W - 1) & (vv >= 0) & (vv <= H - 1)
                pts.append(pc)
            idx = np.nonzero(ok)[0][: m - got]
            if len(idx) == 0:
                # pair not co-visible from these views: fall back to any surface point (still a valid 3D-3D pair)
                idx = np.arange(min(m - got, len(s)))
            k = len(idx)
            pi = pts[0][idx] + rng.normal(0, point_noise, (k, 3))
            pj = pts[1][idx] + rng.normal(0, point_noise, (k, 3))
            is_out = rng.uniform(size=k) < outlier_frac
            dirs = rng.normal(size=(k, 3))
            dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
            pj = pj + dirs * (is_out * rng.uniform(0.01, 0.05, k))[:, None]
            out["imgIdx_i"][o:o + k] = i
            out["imgIdx_j"][o:o + k] = j
            out["pos_i"][o:o + k] = pi
            out["pos_j"][o:o + k] = pj
            o += k
            got += k
    return out


def pose_errors(poses_a: np.ndarray, poses_b: np.ndarray):
    """(max geodesic rotation error [rad], max translation error [m]) between two [N,4,4] pose stacks."""
    a = np.asarray(poses_a, np.float64)
    b = np.asarray(poses_b, np.float64)
    rmax = max(rot_geodesic(a[k, :3, :3], b[k, :3, :3]) for k in range(a.shape[0]))
    tmax = float(np.abs(a[:, :3, 3] - b[:, :3, 3]).max()) if a.size else 0.0
    tn = float(np.linalg.norm(a[:, :3, 3] - b[:, :3, 3], axis=1).max())
    return rmax, max(tmax, tn)


def make_descriptors(seed: int, n_a: int, n_b: int, dim: int = 256, match_frac: float = 0.3, noise: float = 0.1):
    """Unit-norm descriptors with planted matches (SURVEY.md §8d: i.i.d. unit Gaussians, `match_frac` of B planted
    as the matching A code + N(0, noise^2) per component, renormalised)."""
    rng = np.random.default_rng(np.uint64(0xD5) + np.uint64(seed))
    a = rng.normal(size=(n_a, dim))
    b = rng.normal(size=(n_b, dim))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    m = int(min(n_a, n_b) * match_frac)
    ia = rng.permutation(n_a)[:m]
    ib = rng.permutation(n_b)[:m]
    b[ib] = a[ia] + rng.normal(0, noise, (m, dim))
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    return a.astype(np.float32), b.astype(np.float32), ia, ib


def make_feature_frames(win: Window, n_feats: int = 500, seed: int = 0, n_surface: int = 4000, kp_noise: float = 0.3, desc_noise: float = 0.05,
                        distractor_frac: float = 0.2, dim: int = 256):
    """Keypoints + unit-norm descriptors for every frame of a rendered window (the matcher side of SURVEY.md §8d):
    `n_surface` points on the ellipsoid carry a random code each; a frame sees those facing it, keypoint = projection +
    sub-pixel noise, descriptor = code + noise (renormalised); `distractor_frac` of the features are unmatched.
    Returns list of dicts {kpts [n,2] f32 (x,y), desc [n,dim] f32, ids [n] (surface id or -1)}."""
    rng = np.random.default_rng(np.uint64(0xFEA7) + np.uint64(seed))
    sdir = rng.normal(size=(n_surface, 3))
    sdir /= np.linalg.norm(sdir, axis=1, keepdims=True)
    p_ob, n_ob = sdir * win.radii, sdir / win.radii
    codes = rng.normal(size=(n_surface, dim))
    codes /= np.linalg.norm(codes, axis=1, keepdims=True)
    fx, fy, cx, cy = win.K
    frames = []
    for f in range(win.n_frames):
        R, c = win.ob_in_cam[f][:3, :3], win.ob_in_cam[f][:3, 3]
        pc, nc = p_ob @ R.T + c, n_ob @ R.T
        vis = np.einsum("nk,nk->n", nc, -pc) > 0.15 * np.linalg.norm(nc, axis=1) * np.linalg.norm(pc, axis=1)
        u, v = pc[:, 0] * fx / pc[:, 2] + cx, pc[:, 1] * fy / pc[:, 2] + cy
        vis &= (u >= 1) & (u <= win.W - 2) & (v >= 1) & (v <= win.H - 2)
        ui, vi = np.clip(np.rint(u).astype(int), 0, win.W - 1), np.clip(np.rint(v).astype(int), 0, win.H - 1)
        vis &= win.depth[f][vi, ui] > 0.1
        idx = np.nonzero(vis)[0]
        n_match = min(len(idx), int(n_feats * (1 - distractor_frac)))
        idx = rng.permutation(idx)[:n_match]
        kp = np.stack([u[idx], v[idx]], 1) + rng.normal(0, kp_noise, (n_match, 2))
        de = codes[idx] + rng.normal(0, desc_noise, (n_match, dim)) / np.sqrt(dim) * 4.0
        ys, xs = np.nonzero(win.depth[f] > 0.1)
        n_dis = n_feats - n_match
        if len(xs) and n_dis > 0:
            sel = rng.integers(0, len(xs), n_dis)
            kp = np.concatenate([kp, np.stack([xs[sel], ys[sel]], 1) + rng.uniform(-0.4, 0.4, (n_dis, 2))])
            de = np.concatenate([de, rng.normal(size=(n_dis, dim))])
            ids = np.concatenate([idx, -np.ones(n_dis, int)])
        else:
            ids = idx
        de /= np.linalg.norm(de, axis=1, keepdims=True)
        perm = rng.permutation(len(kp))
        frames.append({"kpts": kp[perm].astype(np.float32), "desc": de[perm].astype(np.float32), "ids": ids[perm]})
    return frames


def make_raw_depth(seed: int, H: int = 480, W: int = 640, K=None, noise: float = 0.0003, hole_frac: float = 0.02, flying_frac: float = 0.01):
    """A raw sensor-like depth image for the frame front end (SURVEY.md §8f rank 1): a rendered ellipsoid (the window
    generator's frame 0) + N(0, noise) on valid pixels + random holes + isolated "flying" pixels displaced by 2-6 cm that
    the erosion must remove.  Returns (raw [H,W] float32, K)."""
    K = tuple(v * W / 640.0 for v in NOCS_K) if K is None else K
    w = make_window(seed, n_frames=2, n_corr=10, H=H, W=W, K=K)
    rng = np.random.default_rng(np.uint64(0xDE97) + np.uint64(seed))
    d = w.depth[0].astype(np.float32).copy()
    valid = d > 0
    raw = d + valid * rng.normal(0, noise, d.shape).astype(np.float32)
    fly = valid & (rng.random(d.shape) < flying_frac)
    raw = raw + fly * rng.uniform(0.02, 0.06, d.shape).astype(np.float32) * rng.choice([-1.0, 1.0], d.shape).astype(np.float32)
    raw[rng.random(d.shape) < hole_frac] = 0.0
    return raw.astype(np.float32), K


def make_object_mask(seed: int, H: int = 480, W: int = 640, n_distractors: int = 3, speckle_frac: float = 0.002, n_holes: int = 4,
                     value: int = 255) -> np.ndarray:
    """An object mask as the reference reads it from a mask PNG (uint8 H x W, non-zero = object): a rotated elliptic main blob, smaller
    disc-shaped distractor blobs, isolated speckle pixels and a few holes punched into the main blob.  Pure numpy (no OpenCV), so the
    segmentation tests and benchmarks can make their inputs anywhere.  value: the foreground byte (any non-zero value)."""
    rng = np.random.default_rng(np.uint64(0x5E6) + np.uint64(seed))
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    m = np.zeros((H, W), bool)
    cx, cy = rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H
    a, b = rng.uniform(0.12, 0.3) * W, rng.uniform(0.12, 0.3) * H
    th = rng.uniform(0, np.pi)
    u, v = (x - cx) * np.cos(th) + (y - cy) * np.sin(th), -(x - cx) * np.sin(th) + (y - cy) * np.cos(th)
    m |= (u / max(a, 0.5)) ** 2 + (v / max(b, 0.5)) ** 2 <= 1.0
    for _ in range(n_holes):
        hx, hy = cx + rng.uniform(-0.5, 0.5) * a, cy + rng.uniform(-0.5, 0.5) * b
        m &= (x - hx) ** 2 + (y - hy) ** 2 > rng.uniform(1.0, 0.15 * min(a, b) + 1.5) ** 2
    for _ in range(n_distractors):
        r = rng.uniform(0.02, 0.06) * min(H, W) + 0.5
        m |= (x - rng.uniform(0, W)) ** 2 + (y - rng.uniform(0, H)) ** 2 <= r * r
    m |= rng.random((H, W)) < speckle_frac
    return (m * np.uint8(value)).astype(np.uint8)


def ragged_ellipse_masks(n_frames: int, H: int = 480, W: int = 640, seed: int = 0):
    """(pred, gt): uint8 [n_frames, H, W] 0 / 255 masks of an ellipse that moves across the frame and turns, its outline made ragged by a few
    harmonics of the polar angle.  The prediction is the same ellipse displaced by up to about 2 % of the frame, with harmonics of its own
    that change from frame to frame, as a segmenter's error would.  For the mask scores' tests and benchmark."""
    rng = np.random.default_rng(np.uint64(0xDA715) + np.uint64(seed))
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    k = np.arange(3, 9, dtype=np.float32)
    amp_g, ph_g = rng.uniform(0.01, 0.04, 6).astype(np.float32), rng.uniform(0, 2 * np.pi, 6).astype(np.float32)
    out = np.zeros((2, n_frames, H, W), np.uint8)
    for f in range(n_frames):
        t = f / max(n_frames - 1, 1)
        cx, cy = (0.3 + 0.4 * t) * W, (0.4 + 0.2 * np.sin(2 * np.pi * t)) * H
        ax, ay, th = 0.18 * W, 0.22 * H, np.float32(np.pi * t)
        d = 0.02 * rng.uniform(-1, 1, 2) * (W, H)
        amp_p, ph_p = rng.uniform(0.01, 0.04, 6).astype(np.float32), rng.uniform(0, 2 * np.pi, 6).astype(np.float32)
        for m, (ox, oy, amp, ph) in enumerate(((d[0], d[1], amp_p, ph_p), (0.0, 0.0, amp_g, ph_g))):
            u, v = x - np.float32(cx + ox), y - np.float32(cy + oy)
            u, v = u * np.cos(th) + v * np.sin(th), v * np.cos(th) - u * np.sin(th)
            ang = np.arctan2(v / ay, u / ax)
            rag = 1 + (amp[:, None, None] * np.cos(k[:, None, None] * ang + ph[:, None, None])).sum(0)
            out[m, f] = ((u / ax) ** 2 + (v / ay) ** 2 <= rag * rag) * np.uint8(255)
    return out[0], out[1]


def make_ransac_case(seed: int, n: int, inlier_frac: float = 0.7, noise: float = 0.0005):
    """Model-frame point pairs as SiftManager::runRansacMultiPairGPU uploads them (/root/reference/src/FeatureManager.cpp:676-706):
    B = T A + noise for the inliers, the rest displaced by centimetres.  Returns (A [n,4], B [n,4] float32 with w = 1, inlier mask)."""
    rng = np.random.default_rng(seed)
    A = rng.uniform(-0.1, 0.1, (n, 3)) + [0, 0, 0.7]
    R = so3_exp(rng.normal(0, 0.3, 3)); t = rng.normal(0, 0.05, 3)
    B = A @ R.T + t + rng.normal(0, noise, (n, 3))
    out = rng.uniform(size=n) > inlier_frac
    B[out] += rng.normal(0, 1, (int(out.sum()), 3)) * 0.02 + 0.03
    A4 = np.concatenate([A, np.ones((n, 1))], 1).astype(np.float32)
    B4 = np.concatenate([B, np.ones((n, 1))], 1).astype(np.float32)
    return A4, B4, ~out


@dataclasses.dataclass
class Sequence:
    """A tracked object over time, as the tracker's caller sees it: per frame the raw depth, the mask PNG's bytes, the colour image and
    what the LF-Net server would reply (keypoints, descriptors; None where feature detection fails)."""
    depth_raw: np.ndarray    # [N,H,W] f32, metres, 0 = hole
    mask: np.ndarray         # [N,H,W] u8, 255 = object (the silhouette plus a distractor blob)
    colour: np.ndarray       # [N,H,W,3] u8 BGR
    feats: list              # per frame {kpts [n,2] f32, desc [n,dim] f32, ids [n]} or None
    poses_gt: np.ndarray     # [N,4,4] f64 cam->model, model = camera frame 0
    K: tuple
    roi_fail: tuple          # frames whose mask is empty (the tracker's ROI gate fails)
    neighbour_fail: tuple    # frames whose features cannot match the previous frame
    detect_fail: tuple       # frames without features (detection failed)
    radii: Optional[np.ndarray] = None        # the ellipsoid's radii (object frame), metres
    ob_in_cam0: Optional[np.ndarray] = None   # [4,4] f64 object -> camera 0: a point x of the object frame is ob_in_cam0 x in the model frame

    @property
    def n_frames(self) -> int:
        return self.depth_raw.shape[0]


def _dilate(m: np.ndarray, r: int) -> np.ndarray:
    p = np.pad(m, r)
    out = np.zeros_like(m)
    for dy in range(2 * r + 1):
        for dx in range(2 * r + 1):
            out |= p[dy:dy + m.shape[0], dx:dx + m.shape[1]]
    return out


def make_sequence(seed: int, n_frames: int, H: int = 480, W: int = 640, K=None, n_feats: int = 500, rot_deg=(2.0, 6.0), hole_frac: float = 0.02,
                  roi_fail=(), neighbour_fail=(), detect_fail=()) -> Sequence:
    """A smooth trajectory of one rendered ellipsoid (render_ellipsoid) with features from make_feature_frames: per frame a rotation of
    rot_deg degrees about an axis that drifts slowly, and a few millimetres of translation.  Raw depth has 1 mm noise and `hole_frac` holes;
    the mask is the silhouette plus a disc-shaped distractor blob away from it (largest-hull mode drops it, as-is mode keeps it); the colour
    image is a gradient with the object shaded by its normals.  Events at the listed frames: an empty mask (roi_fail), random descriptors at
    background pixels that have no depth (neighbour_fail: the neighbour pair finds no match), no features at all (detect_fail: feats is None)."""
    K = tuple(v * W / 640.0 for v in NOCS_K) if K is None else tuple(K)
    rng = np.random.default_rng(np.uint64(0x5EC) + np.uint64(seed))
    radii = rng.uniform(0.05, 0.1, size=3)
    R, _ = _sample_pose(rng)
    c = np.array([rng.uniform(-0.02, 0.02), rng.uniform(-0.02, 0.02), rng.uniform(0.6, 0.75)])
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ob_in_cam = np.zeros((n_frames, 4, 4))
    ob_in_cam[0] = se3(R, c)
    for k in range(1, n_frames):
        axis = axis + rng.normal(0, 0.3, 3)
        axis /= np.linalg.norm(axis)
        R = so3_exp(axis * np.deg2rad(rng.uniform(*rot_deg))) @ R
        c = c + rng.normal(0, 0.003, 3)
        c[2] = np.clip(c[2], 0.55, 0.8)
        c[:2] = np.clip(c[:2], -0.04, 0.04)
        ob_in_cam[k] = se3(R, c)
    poses_gt = np.stack([ob_in_cam[0] @ np.linalg.inv(ob_in_cam[k]) for k in range(n_frames)])
    depth = np.zeros((n_frames, H, W), np.float32)
    normal = np.zeros((n_frames, H, W, 4), np.float32)
    for k in range(n_frames):
        depth[k], normal[k] = render_ellipsoid(radii, ob_in_cam[k], K, H, W, rng)
    win = Window(depth, normal, poses_gt.astype(np.float32), poses_gt, np.zeros(0, ENTRYJ_DTYPE), K, radii, ob_in_cam)
    feats = make_feature_frames(win, n_feats=n_feats, seed=seed, n_surface=max(4000, 4 * n_feats))
    yy, xx = np.mgrid[0:H, 0:W]
    raw = depth.copy()
    mask = np.zeros((n_frames, H, W), np.uint8)
    colour = np.zeros((n_frames, H, W, 3), np.uint8)
    r_blob = 0.05 * min(H, W)
    for k in range(n_frames):
        sil = depth[k] > 0
        raw[k][rng.random((H, W)) < hole_frac] = 0.0
        ys, xs = np.nonzero(sil)
        # the distractor sits in the image corner farthest from the silhouette's centre
        bx = r_blob + 1 if xs.mean() > W / 2 else W - r_blob - 2
        by = r_blob + 1 if ys.mean() > H / 2 else H - r_blob - 2
        blob = (xx - bx) ** 2 + (yy - by) ** 2 <= r_blob ** 2
        mask[k] = (sil | blob).astype(np.uint8) * 255
        shade = (60 + 150 * np.abs(normal[k][..., :3])).astype(np.uint8)
        bg = np.stack([xx * 255 // W, yy * 255 // H, np.full((H, W), 128)], -1).astype(np.uint8)
        colour[k] = np.where(sil[..., None], shade, bg)
        if k in neighbour_fail:
            n = len(feats[k]["kpts"])
            far = np.nonzero(~_dilate(sil, 4))
            sel = rng.integers(0, len(far[0]), n)
            d = rng.normal(size=(n, feats[k]["desc"].shape[1]))
            feats[k] = {"kpts": np.stack([far[1][sel], far[0][sel]], 1).astype(np.float32),
                        "desc": (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32), "ids": -np.ones(n, int)}
        if k in roi_fail:
            mask[k] = 0
        if k in detect_fail:
            feats[k] = None
    return Sequence(raw, mask, colour, feats, poses_gt, K, tuple(roi_fail), tuple(neighbour_fail), tuple(detect_fail), radii, ob_in_cam[0].copy())


def write_png(path: str, img: np.ndarray) -> None:
    """A PNG of img with the standard library's zlib: uint8 [H,W] (grey), uint8 [H,W,3] BGR (stored as RGB, as cv2.imwrite does) or uint16
    [H,W] (16-bit grey, big-endian samples).  Filter type 0 on every row; no ancillary chunks."""
    import struct
    import zlib
    a = np.asarray(img)
    if a.dtype == np.uint8 and a.ndim == 2:
        depth, ctype, rows = 8, 0, a
    elif a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3:
        depth, ctype, rows = 8, 2, a[..., ::-1].reshape(a.shape[0], -1)
    elif a.dtype == np.uint16 and a.ndim == 2:
        depth, ctype, rows = 16, 0, a.astype(">u2").view(np.uint8).reshape(a.shape[0], -1)
    else:
        raise ValueError(f"write_png: unsupported array {a.dtype} {a.shape}")
    raw = np.concatenate([np.zeros((rows.shape[0], 1), np.uint8), np.ascontiguousarray(rows)], 1).tobytes()

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", a.shape[1], a.shape[0], depth, ctype, 0, 0, 0))
                + chunk(b"IDAT", zlib.compress(raw, 1)) + chunk(b"IEND", b""))


def depth_mm(depth_m: np.ndarray) -> np.ndarray:
    """Depth in metres as a 16-bit depth PNG holds it: millimetres rounded from the float64 product, clipped to [0, 65535]."""
    return np.clip(np.round(np.asarray(depth_m, np.float64) * 1000), 0, 65535).astype(np.uint16)


def write_ycbineoat_video(seq: Sequence, video_dir: str) -> None:
    """seq as a YCBInEOAT video directory (sequence.YcbineoatVideo reads it): rgb/, depth/ (16-bit millimetres), masks/, cam_K.txt and
    annotated_poses/ (ob_in_cam per frame), frames named %07d.png."""
    import os
    for sub in ("rgb", "depth", "masks", "annotated_poses"):
        os.makedirs(os.path.join(video_dir, sub), exist_ok=True)
    for k in range(seq.n_frames):
        # millimetres from the float32 product, not depth_mm: the two round a few pixels of a sequence 1 mm apart, and the GPU tests'
        # input videos are written this way
        for sub, img in (("rgb", seq.colour[k]), ("depth", np.round(seq.depth_raw[k] * 1000).astype(np.uint16)), ("masks", seq.mask[k])):
            write_png(os.path.join(video_dir, sub, f"{k:07d}.png"), img)
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))
        with open(os.path.join(video_dir, "annotated_poses", f"{k:07d}.txt"), "w") as f:
            f.write("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in G))
    K = np.array([[seq.K[0], 0, seq.K[2]], [0, seq.K[1], seq.K[3]], [0, 0, 1]])
    with open(os.path.join(video_dir, "cam_K.txt"), "w") as f:
        f.write("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in K))


def write_nocs_scene(seq: Sequence, root: str, scene: int = 1, model: str = "camera_bench_norm", masks_dir: Optional[str] = None,
                     obj_points: Optional[np.ndarray] = None) -> tuple:
    """seq as NOCS-REAL275 scene `scene` of object `model` under root/nocs (sequence.NocsScene reads it): colour and depth PNGs (depth_mm),
    the first frame's ob_in_cam as the ground truth 0000.txt, the class-3 data list, and with obj_points [n, 3] the object's OBJ model.  The
    mask PNGs go to masks_dir (default root/masks).  Returns (nocs_dir, masks_dir)."""
    import os
    nocs, masks = os.path.join(root, "nocs"), masks_dir or os.path.join(root, "masks")
    data = f"{nocs}/real_test/scene_{scene}"
    gt = f"{nocs}/gts/real_test_text/scene_{scene}/model_{model}"
    lst = f"{nocs}/NOCS-REAL275-additional/data_list/real_val/3/{model}"
    for d in (data, masks, gt, lst):
        os.makedirs(d)
    for k in range(seq.n_frames):
        write_png(f"{data}/{k:04d}_color.png", seq.colour[k])
        write_png(f"{data}/{k:04d}_depth.png", depth_mm(seq.depth_raw[k]))
        write_png(f"{masks}/{k:04d}.png", seq.mask[k])
    np.savetxt(f"{gt}/0000.txt", np.linalg.inv(seq.poses_gt[0]))
    with open(f"{lst}/list.txt", "w") as f:
        f.write("".join(f"real_val/scene_{scene}/{k:04d}\n" for k in range(seq.n_frames)))
    if obj_points is not None:
        os.makedirs(f"{nocs}/obj_models/real_test")
        with open(f"{nocs}/obj_models/real_test/{model}.obj", "w") as f:
            f.write("".join(f"v {x:.9g} {y:.9g} {z:.9g}\n" for x, y, z in np.asarray(obj_points, np.float64)))
    return nocs, masks


def recorded_features(seq: Sequence):
    """run_sequence's feature callable that replays seq: frame id_str's keypoints and descriptors, sequence.DetectionFailed for a frame
    without features."""
    from .sequence import DetectionFailed

    def features(id_str, request, roi):
        f = seq.feats[int(id_str)]
        if f is None:
            raise DetectionFailed(id_str)
        return f["kpts"], f["desc"]
    return features


def make_ellipsoid_model(seed: int, n: int, radii=(0.05, 0.04, 0.03)) -> np.ndarray:
    """float32 [n,3]: n points on the surface of an ellipsoid with the given semi-axes (metres), the stand-in for an OBJ model's vertices."""
    rng = np.random.default_rng(seed)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (u * np.asarray(radii, np.float64)).astype(np.float32)
