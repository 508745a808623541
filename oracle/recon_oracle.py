"""numpy float32 restatement of the object-model path (bundletrack_b200/csrc/recon.cu), in the operation order the device pins, so the device's
bounds, grid (sum, count) and mesh can be compared with it bit for bit (DESIGN.md §3.14):

- bounds: every valid pixel (finite d > 0) back-projected, X = ((u - cx) d) / fx, Y = ((v - cy) d) / fy, Z = d, moved into the model frame
  ((R0 X + R1 Y) + R2 Z) + t per coordinate; min / max per axis;
- grid: m = ceil(trunc / voxel) + 1, origin = lo - m voxel, n = ceil((hi - lo) / voxel) + 1 + 2 m, sample i at origin + i voxel;
- integrate: per frame in order, c = R^T (p - t) as ((R0r q0 + R1r q1) + R2r q2), u = floor(((x fx) / z + cx) + 0.5), the TSDF update;
- mesh: marching tetrahedra over the six Kuhn tets of every cube, vertices in (sample, direction) order, faces in (cube, tet, triangle) order.

Test infrastructure only: bundletrack_b200/ never imports it."""
from __future__ import annotations

import numpy as np

F32 = np.float32
# a vertex direction as a corner-offset bitmask (bit 0: +x, bit 1: +y, bit 2: +z), in the order {x, y, z, xy, xz, yz, xyz}, and back
DIR_CODE = (1, 2, 4, 3, 5, 6, 7)
DIR_OF_CODE = {c: k for k, c in enumerate(DIR_CODE)}
# the six tets of a cube (axis permutations xyz, xzy, yxz, yzx, zxy, zyx), corners as offset codes in a positively oriented order
TETS = ((0, 1, 3, 7), (0, 5, 1, 7), (0, 3, 2, 7), (0, 2, 6, 7), (0, 4, 5, 7), (0, 6, 4, 7))
# even permutations of a tet's corners starting with the corner alone on its side, and with the two inside corners (by their mask)
ODD = ((0, 1, 2, 3), (1, 0, 3, 2), (2, 3, 0, 1), (3, 2, 1, 0))
PAIR = {3: (0, 1, 2, 3), 5: (0, 2, 3, 1), 6: (1, 2, 0, 3), 9: (0, 3, 1, 2), 10: (1, 3, 2, 0), 12: (2, 3, 0, 1)}


def _poses(cam_in_model):
    P = np.asarray(cam_in_model, F32).reshape(-1, 4, 4)
    return P[:, :3, :3], P[:, :3, 3]


def bounds(depths, cam_in_model, K):
    """(lo [3], hi [3]) float32 of the valid pixels in the model frame, or None when no frame has one."""
    fx, fy, cx, cy = (F32(v) for v in K)
    R, t = _poses(cam_in_model)
    lo, hi = np.full(3, np.inf, F32), np.full(3, -np.inf, F32)
    for f, d in enumerate(depths):
        d = np.asarray(d, F32)
        vv, uu = np.nonzero((d > 0) & np.isfinite(d))
        if len(uu) == 0:
            continue
        z = d[vv, uu]
        c = (((uu.astype(F32) - cx) * z) / fx, ((vv.astype(F32) - cy) * z) / fy, z)
        for a in range(3):
            p = ((R[f, a, 0] * c[0] + R[f, a, 1] * c[1]) + R[f, a, 2] * c[2]) + t[f, a]
            lo[a], hi[a] = min(lo[a], p.min()), max(hi[a], p.max())
    return None if not np.isfinite(lo[0]) else (lo, hi)


def grid(lo, hi, voxel, trunc):
    """(dims (nx, ny, nz), origin float32 [3]) of the grid around the bounds."""
    voxel, trunc = F32(voxel), F32(trunc)
    m = int(np.ceil(trunc / voxel)) + 1
    n = tuple(int(np.ceil((F32(hi[a]) - F32(lo[a])) / voxel)) + 1 + 2 * m for a in range(3))
    origin = np.array([F32(lo[a]) - F32(m) * voxel for a in range(3)], F32)
    return n, origin


def coords(n, origin, voxel):
    """The sample positions per axis: origin_a + i voxel."""
    return [origin[a] + np.arange(n[a], dtype=F32) * F32(voxel) for a in range(3)]


def integrate(depths, cam_in_model, K, n, origin, voxel, trunc):
    """(sum float32, count int32), both [nz, ny, nx]."""
    fx, fy, cx, cy = (F32(v) for v in K)
    trunc = F32(trunc)
    R, t = _poses(cam_in_model)
    xs, ys, zs = coords(n, origin, voxel)
    Z, Y, X = np.meshgrid(zs, ys, xs, indexing="ij")
    p = (X.ravel(), Y.ravel(), Z.ravel())
    s = np.zeros(p[0].shape, F32)
    cnt = np.zeros(p[0].shape, np.int32)
    for f, d in enumerate(depths):
        d = np.asarray(d, F32)
        H, W = d.shape
        q = [p[a] - t[f, a] for a in range(3)]
        c = [(R[f, 0, r] * q[0] + R[f, 1, r] * q[1]) + R[f, 2, r] * q[2] for r in range(3)]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            fu = np.floor(((c[0] * fx) / c[2] + cx) + F32(0.5))
            fv = np.floor(((c[1] * fy) / c[2] + cy) + F32(0.5))
        ok = (c[2] > 0) & (fu >= 0) & (fu < W) & (fv >= 0) & (fv < H)
        idx = np.nonzero(ok)[0]
        dd = d[fv[idx].astype(np.int64), fu[idx].astype(np.int64)]
        keep = dd > 0
        idx, dd = idx[keep], dd[keep]
        sdf = dd - c[2][idx]
        keep = ~(sdf < -trunc)
        idx, sdf = idx[keep], sdf[keep]
        s[idx] = s[idx] + np.minimum(F32(1), sdf / trunc)
        cnt[idx] += 1
    return s.reshape(n[2], n[1], n[0]), cnt.reshape(n[2], n[1], n[0])


def fuse(depths, cam_in_model, K, voxel, trunc):
    """The whole fuse: dict of lo, hi, dims, origin, sum, count (None when no frame has a valid pixel)."""
    b = bounds(depths, cam_in_model, K)
    if b is None:
        return None
    n, origin = grid(*b, voxel, trunc)
    s, c = integrate(depths, cam_in_model, K, n, origin, voxel, trunc)
    return {"lo": b[0], "hi": b[1], "dims": n, "origin": origin, "sum": s, "count": c}


def tet_triangles(t: int, inside: int):
    """The triangles of tet t for the inside mask of its four corners (bit k: corner k has f < 0): each a tuple of three edges (code_a,
    code_b), wound so that the normal points to the outside corners."""
    code = TETS[t]
    k = bin(inside).count("1")
    if k in (0, 4):
        return []
    if k != 2:
        a = ((inside if k == 1 else ~inside & 15) & -(inside if k == 1 else ~inside & 15)).bit_length() - 1
        A, B, C, D = (code[i] for i in ODD[a])
        return [((A, B), (A, C), (A, D))] if k == 1 else [((A, B), (A, D), (A, C))]
    A, B, C, D = (code[i] for i in PAIR[inside])
    return [((A, C), (A, D), (B, D)), ((A, C), (B, D), (B, C))]


def field(s, c):
    """sum / count in float32, NaN where count = 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(c > 0, s / np.maximum(c, 1).astype(F32), F32(np.nan)).astype(F32)


def mesh(g, voxel):
    """(verts float32 [n,3], faces int32 [m,3]) of the grid dict g from fuse, in the device's order."""
    nx, ny, nz = g["dims"]
    f = field(g["sum"], g["count"]).ravel()
    off = lambda code: (code & 1) + ((code >> 1) & 1) * nx + ((code >> 2) & 1) * nx * ny
    zz, yy, xx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    cube = (xx + nx * (yy + ny * zz)).ravel().astype(np.int64)      # ascending
    fc = np.stack([f[cube + off(c)] for c in range(8)], 1)
    # per (cube, tet, triangle slot): the three edges as (owner sample, direction), and whether the slot holds a triangle
    owner = np.zeros((len(cube), 6, 2, 3), np.int64)
    dirs = np.zeros((len(cube), 6, 2, 3), np.int64)
    present = np.zeros((len(cube), 6, 2), bool)
    for t, code in enumerate(TETS):
        v4 = fc[:, list(code)]
        observed = ~np.isnan(v4).any(1)
        inside = ((v4 < 0) * (1 << np.arange(4))).sum(1)
        for mask in range(1, 15):
            sel = np.nonzero(observed & (inside == mask))[0]
            for k, tri in enumerate(tet_triangles(t, mask)):
                present[sel, t, k] = True
                for e, (a, b) in enumerate(tri):
                    lo, hi = (a, b) if a & b == a else (b, a)
                    owner[sel, t, k, e] = cube[sel] + off(lo)
                    dirs[sel, t, k, e] = DIR_OF_CODE[lo ^ hi]
    key = (owner * 7 + dirs)[present]                                     # [m, 3], (cube, tet, triangle) order
    vkeys = np.unique(key)
    faces = np.searchsorted(vkeys, key).astype(np.int32).reshape(-1, 3)
    vo, vd = vkeys // 7, vkeys % 7
    code = np.array(DIR_CODE)[vd]
    n = (nx, ny, nz)
    idx = (vo % nx, (vo // nx) % ny, vo // (nx * ny))
    other = vo + (code & 1) + ((code >> 1) & 1) * nx + ((code >> 2) & 1) * nx * ny
    fa, fb = f[vo], f[other]
    tt = fa / (fa - fb)
    xs = coords(n, g["origin"], voxel)
    xs1 = [g["origin"][a] + np.arange(1, n[a] + 1, dtype=F32) * F32(voxel) for a in range(3)]   # sample i + 1
    verts = np.empty((len(vkeys), 3), F32)
    for a in range(3):
        pa = xs[a][idx[a]]
        pb = np.where((code >> a) & 1, xs1[a][idx[a]], pa)
        verts[:, a] = pa + tt * (pb - pa)
    return verts, faces


# ---- mesh checks -----------------------------------------------------------------------------------------------------------------------

def edge_check(faces) -> bool:
    """True when every edge is used by exactly two faces, walked in opposite directions (closed and consistently wound)."""
    f = np.asarray(faces, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = d[:, 0] * (int(f.max()) + 1) + d[:, 1]
    rev = d[:, 1] * (int(f.max()) + 1) + d[:, 0]
    if len(np.unique(key)) != len(key):
        return False
    return bool(np.isin(rev, key).all())


def euler(verts, faces) -> int:
    f = np.asarray(faces, np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    n_e = len(np.unique(e[:, 0] * (len(verts) + 1) + e[:, 1]))
    return len(np.unique(f)) - n_e + len(f)


def signed_volume(verts, faces) -> float:
    v = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


# ---- synthetic views -------------------------------------------------------------------------------------------------------------------

def views_around(dist: float, centre=(0.0, 0.0, 0.0)):
    """ob_in_cam [26,4,4] float64: cameras at `dist` from centre along the 26 directions of {-1,0,1}^3 \\ 0, each looking at the centre
    (the object frame is the model frame)."""
    out = []
    for d in np.array([(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1) if (x, y, z) != (0, 0, 0)], np.float64):
        d /= np.linalg.norm(d)
        c = np.asarray(centre, np.float64) + dist * d
        z = -d
        up = np.array([0.0, 0.0, 1.0]) if abs(z[2]) < 0.9 else np.array([0.0, 1.0, 0.0])
        x = np.cross(up, z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])                        # rows: the camera axes in the object frame
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, -R @ c
        out.append(T)
    return np.stack(out)


def ellipsoid_distance(p, radii):
    """Distance of points p [n,3] to the ellipsoid sum (x_a / r_a)^2 = 1 in float64: the closest point is x_a = p_a r_a^2 / (s + r_a^2) for
    the root s of sum (p_a r_a / (s + r_a^2))^2 = 1, found by Newton (convex and decreasing on s > -min r^2)."""
    p = np.abs(np.asarray(p, np.float64))
    r2 = np.asarray(radii, np.float64) ** 2
    s = np.zeros(len(p))
    for _ in range(200):
        den = s[:, None] + r2
        F = (p ** 2 * r2 / den ** 2).sum(1) - 1.0
        dF = (-2 * p ** 2 * r2 / den ** 3).sum(1)
        s = np.maximum(s - F / dF, 0.5 * (s - r2.min()))
    x = p * r2 / (s[:, None] + r2)
    return np.linalg.norm(p - x, axis=1)
