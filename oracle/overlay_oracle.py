"""numpy float32 restatement of the tracking overlay (the reference's LOG frames, Bundler::saveNewframeResult, src/Bundler.cpp:379-411), in the
operation order the device pins (DESIGN.md §3.10):

- load_obj_vertices: pcl::io::loadOBJFile's points, the `v x y z` lines in file order;
- voxel_grid: PCL 1.9 VoxelGrid::applyFilter (downsample_all_data_, min_points_per_voxel_ = 0), with the points of a voxel summed in input
  order (PCL's std::sort leaves that order open);
- transform / inverse4: ob_in_cam = the float cofactor inverse of cur_in_model, each coordinate ((m0 x + m1 y) + m2 z) + m3;
- project: u = roundf(x fx / z + cx), v likewise, kept inside the image;
- render: the colour dimmed where fg == 0 ((uint8)(c * 0.2) in double), the 5-pixel stamp of cv::circle(r = 1, filled) in BGR (0, 255, 255)
  at every projected centroid, and the masked colour_raw image."""
from __future__ import annotations

import numpy as np

F32 = np.float32
STAMP = ((0, 0), (-1, 0), (1, 0), (0, -1), (0, 1))          # (du, dv) of cv::circle(r = 1, filled, LINE_8)
COLOUR = (0, 255, 255)                                       # BGR


def load_obj_vertices(path: str) -> np.ndarray:
    """float32 [n,3]: the first three values of every `v` line, in file order."""
    pts = []
    with open(path) as f:
        for line in f:
            t = line.split()
            if t and t[0] == "v":
                pts.append([float(x) for x in t[1:4]])
    return np.asarray(pts, np.float64).astype(F32).reshape(-1, 3)


def _grid(p: np.ndarray, leaf: float):
    """(mode, finite mask, idx per finite point): mode "empty", "copy" (the overflow rule) or "grid"."""
    inv = F32(1) / F32(leaf)
    fin = np.isfinite(p).all(1)
    q = p[fin]
    if len(q) == 0:
        return "empty", fin, None
    mn, mx = q.min(0), q.max(0)
    cells = 1
    for a in range(3):
        span = (mx[a] - mn[a]) * inv
        cells *= int(min(float(span), 9.2e18)) + 1
    if cells > 2 ** 31 - 1:
        return "copy", fin, None
    min_b = np.floor(mn * inv).astype(np.int64)
    div = np.floor(mx * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(q * inv) - min_b.astype(F32)).astype(np.int64)
    idx = (ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * ((div[0] * div[1]) & 0xFFFFFFFF)) & 0xFFFFFFFF
    return "grid", fin, idx


def voxel_grid(points, leaf: float) -> np.ndarray:
    """float32 [m,3]: one centroid per occupied voxel in ascending voxel index; the input unchanged under the overflow rule."""
    p = np.ascontiguousarray(points, F32).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        mode, fin, idx = _grid(p, leaf)
    if mode == "empty":
        return np.zeros((0, 3), F32)
    if mode == "copy":
        return p.copy()
    q = p[fin]
    order = np.argsort(idx, kind="stable")
    s_idx, s_pts = idx[order], q[order]
    heads = np.flatnonzero(np.r_[True, s_idx[1:] != s_idx[:-1]])
    counts = np.diff(np.r_[heads, len(s_idx)])
    sums = np.zeros((len(heads), 3), F32)
    for k in range(int(counts.max())):          # the k-th point of every voxel, so each voxel's sum runs in its points' input order
        live = counts > k
        sums[live] = sums[live] + s_pts[heads[live] + k]
    return sums / counts.astype(F32)[:, None]


def inverse4(m) -> np.ndarray:
    """The float cofactor inverse of a row-major 4 x 4 (policy.cu inverse4), operation for operation in float32."""
    m = [F32(v) for v in np.asarray(m, F32).reshape(16)]
    t = [F32(0)] * 16
    t[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10]
    t[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10]
    t[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9]
    t[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9]
    t[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10]
    t[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10]
    t[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9]
    t[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9]
    t[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6]
    t[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6]
    t[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5]
    t[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5]
    t[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6]
    t[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6]
    t[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5]
    t[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5]
    det = m[0] * t[0] + m[1] * t[4] + m[2] * t[8] + m[3] * t[12]
    if not det != 0:
        raise ValueError("singular pose")
    inv = F32(1) / det
    return np.array([v * inv for v in t], F32).reshape(4, 4)


def transform(points, P) -> np.ndarray:
    """((m0 x + m1 y) + m2 z) + m3 per coordinate, float32, every operation rounded."""
    p = np.asarray(points, F32).reshape(-1, 3)
    P = np.asarray(P, F32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] for r in range(3)], 1).astype(F32)


def _roundf(v: np.ndarray) -> np.ndarray:
    """C roundf: halves away from zero, exactly (v + 0.5 would round in float)."""
    t = np.trunc(v)
    return t + np.where(np.abs(v - t) >= F32(0.5), np.sign(v), F32(0)).astype(F32)


def project(cent, K, H: int, W: int) -> np.ndarray:
    """int [k,2] (u, v) of the centroids that land inside H x W, in centroid order.  NaN, infinite and out-of-int values are outside."""
    c = np.asarray(cent, F32).reshape(-1, 3)
    fx, fy, cx, cy = (F32(v) for v in K)
    with np.errstate(all="ignore"):
        u = _roundf((c[:, 0] * fx) / c[:, 2] + cx)
        v = _roundf((c[:, 1] * fy) / c[:, 2] + cy)
        ok = (u >= 0) & (u < W) & (v >= 0) & (v < H)
    return np.stack([u[ok], v[ok]], 1).astype(np.int64)


def dim(colour, fg) -> np.ndarray:
    """Bundler.cpp:385-396: each channel (uchar)(c * 0.2) in double where fg == 0."""
    out = np.array(colour, np.uint8, copy=True)
    out[fg == 0] = (out[fg == 0].astype(np.float64) * 0.2).astype(np.uint8)
    return out


def stamp(img: np.ndarray, uv) -> np.ndarray:
    """cv::circle(img, (u, v), 1, (0, 255, 255), -1) at every centre: the pixel and its four neighbours, clipped."""
    H, W = img.shape[:2]
    for du, dv in STAMP:
        u, v = uv[:, 0] + du, uv[:, 1] + dv
        ok = (u >= 0) & (u < W) & (v >= 0) & (v < H)
        img[v[ok], u[ok]] = COLOUR
    return img


def centroids(model, cur_in_model) -> np.ndarray:
    """The model under ob_in_cam = inverse4(cur_in_model), voxel-gridded at 0.01."""
    return voxel_grid(transform(model, inverse4(cur_in_model)), 0.01)


def render(colour, fg, model, cur_in_model, K):
    """(viz, raw): the LOG frame without its label, and colour_raw (the colour zeroed where fg == 0)."""
    colour = np.asarray(colour, np.uint8)
    H, W = colour.shape[:2]
    viz = stamp(dim(colour, fg), project(centroids(model, cur_in_model), K, H, W))
    raw = np.where((np.asarray(fg) != 0)[..., None], colour, 0).astype(np.uint8)
    return viz, raw
