"""numpy restatement of the object model's accuracy (bundletrack_b200/csrc/metrics.cu, DESIGN.md §3.15): surface samples in the kernels'
integer and float64 order, so the device's samples can be compared with them bit for bit, and nearest distances from a k-d tree with a
float64 recheck:

- per face w = |(B - A) x (C - A)|, every product and sum rounded on its own, sums left to right;
- q = floor(w / max w * 2^32) as an integer, the CDF its exact 64-bit cumulative sum;
- sample k: h_i = splitmix64 output i from state seed (i = 3k, 3k + 1, 3k + 2), position ((k 2^32 + (h_3k >> 32)) total) // (N 2^32), the
  first face whose CDF exceeds it, s = sqrt(u1) with u = (h >> 11) 2^-53, and the point ((1 - s) A + s (1 - u2) B) + s u2 C;
- distances: the k-d tree's nearest candidates, each rechecked as sqrt((dx dx + dy dy) + dz dz).

Test infrastructure only: bundletrack_b200/ never imports it."""
from __future__ import annotations

import numpy as np

U64 = np.uint64


def splitmix64(seed: int, i) -> np.ndarray:
    """splitmix64 output i (0-based) of the generator started at state `seed`, for a uint64 array of i."""
    i = np.asarray(i, U64)
    with np.errstate(over="ignore"):
        z = U64(seed) + (i + U64(1)) * U64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def face_weights(verts, faces) -> np.ndarray:
    """w = |(B - A) x (C - A)| per face, float64 (twice the area).  Raises ValueError for an index outside the vertices or a non-finite w."""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    bad = np.nonzero(((f < 0) | (f >= len(v))).any(1))[0]
    if len(bad):
        raise ValueError(f"face {bad[0]} has a vertex index outside [0, {len(v)})")
    A, B, C = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    u, w = B - A, C - A
    cx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    cy = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    cz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    area2 = np.sqrt((cx * cx + cy * cy) + cz * cz)
    bad = np.nonzero(~np.isfinite(area2) | ~np.isfinite(v[f].sum((1, 2))))[0]
    if len(bad):
        raise ValueError(f"face {bad[0]} has a non-finite vertex")
    return area2


def face_cdf(verts, faces) -> np.ndarray:
    """The inclusive uint64 CDF of the integer weights floor(w / max w * 2^32)."""
    w = face_weights(verts, faces)
    wmax = w.max()
    q = np.zeros(len(w), U64) if wmax == 0 else np.floor((w / wmax) * 4294967296.0).astype(U64)
    return np.cumsum(q, dtype=U64)


def sample(verts, faces, n: int, seed: int = 0, return_faces: bool = False):
    """[n, 3] float64 samples, as bt_mesh_sample writes them (and the face of each when return_faces)."""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    cdf = face_cdf(v, f)
    total = int(cdf[-1])
    if total == 0:
        raise ValueError("the mesh has no area")
    k = np.arange(n, dtype=U64)
    h0, h1, h2 = splitmix64(seed, U64(3) * k), splitmix64(seed, U64(3) * k + U64(1)), splitmix64(seed, U64(3) * k + U64(2))
    x = (k << U64(32)) + (h0 >> U64(32))
    pos = np.array([int(a) * total // (n << 32) for a in x.tolist()], U64)
    face = np.searchsorted(cdf, pos, side="right")
    u1 = (h1 >> U64(11)).astype(np.float64) * 2.0 ** -53
    u2 = (h2 >> U64(11)).astype(np.float64) * 2.0 ** -53
    s = np.sqrt(u1)
    b0, b1, b2 = 1.0 - s, s * (1.0 - u2), s * u2
    A, B, C = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    p = (b0[:, None] * A + b1[:, None] * B) + b2[:, None] * C
    return (p, face) if return_faces else p


def recheck(a, b, idx) -> np.ndarray:
    """|a_i - b_idx[i]| as the kernel's rerank forms it, for idx [n] or [n, k] (then the smallest over k)."""
    d = a[:, None, :] - b[np.asarray(idx).reshape(len(a), -1)]
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).min(1)


def nearest(a, b, k: int = 4) -> np.ndarray:
    """min_j |a_i - b_j| in float64: the k-d tree's k nearest candidates, each rechecked in the kernel's order."""
    from scipy.spatial import cKDTree
    a = np.asarray(a, np.float64).reshape(-1, 3)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    _, idx = cKDTree(b).query(a, k=min(k, len(b)))
    return recheck(a, b, idx)


def quantile(x, p: float) -> float:
    """x[lo] + (pos - lo) (x[lo + 1] - x[lo]) at pos = p (n - 1) of the sorted values."""
    x = np.sort(np.asarray(x, np.float64))
    pos = p * (len(x) - 1)
    lo = int(pos)
    if lo + 1 >= len(x):
        return float(x[-1])
    return float(x[lo] + (pos - lo) * (x[lo + 1] - x[lo]))


def score(d_ab, d_ba, taus) -> dict:
    """bt_surface_score restated: means in index order, quantiles, and per tau precision, recall and F."""
    d_ab, d_ba = np.asarray(d_ab, np.float64), np.asarray(d_ba, np.float64)
    acc, comp = float(np.cumsum(d_ab)[-1] / len(d_ab)), float(np.cumsum(d_ba)[-1] / len(d_ba))
    out = {"accuracy": acc, "completeness": comp, "chamfer": (acc + comp) / 2.0,
           "median_model_to_ref": quantile(d_ab, 0.5), "p95_model_to_ref": quantile(d_ab, 0.95),
           "median_ref_to_model": quantile(d_ba, 0.5), "p95_ref_to_model": quantile(d_ba, 0.95),
           "taus": [float(t) for t in taus], "precision": [], "recall": [], "fscore": []}
    for t in taus:
        P = int((d_ab < t).sum()) / len(d_ab)
        R = int((d_ba < t).sum()) / len(d_ba)
        out["precision"].append(P)
        out["recall"].append(R)
        out["fscore"].append(2.0 * P * R / (P + R) if P + R > 0.0 else 0.0)
    return out


def uv_sphere(radius: float, n_lat: int, n_lon: int, centre=(0.0, 0.0, 0.0), radii=None):
    """A closed triangulated sphere (or, with radii, an axis-aligned ellipsoid): poles plus n_lat - 1 rings of n_lon vertices."""
    r = np.full(3, radius) if radii is None else np.asarray(radii, np.float64)
    th = np.pi * np.arange(1, n_lat) / n_lat
    ph = 2 * np.pi * np.arange(n_lon) / n_lon
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph), np.sin(th)[:, None] * np.sin(ph), np.repeat(np.cos(th)[:, None], n_lon, 1)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], ring, [[0, 0, -1]]]) * r + np.asarray(centre, np.float64)
    top, bot = 0, len(v) - 1
    idx = lambda i, j: 1 + i * n_lon + (j % n_lon)
    f = [(top, idx(0, j), idx(0, j + 1)) for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1))]
    f += [(bot, idx(n_lat - 2, j + 1), idx(n_lat - 2, j)) for j in range(n_lon)]
    return v, np.asarray(f, np.int32)
