"""oracle/matcher_oracle.py — TEST INFRASTRUCTURE ONLY.

CPU restatement of the matcher half of the hot path (SURVEY.md §8a a15-a18):
  * knn()            what the two cv::cuda::DescriptorMatcher::knnMatch(…, k=5) calls in SiftManager::findCorresbyNN
                     (/root/reference/src/FeatureManager.cpp:271-273) return: for every query row the k train rows of
                     smallest L2 distance, ascending, DMatch.distance = sqrt(sum (a-b)^2).  The arithmetic lives in
                     OpenCV's cudafeatures2d brute-force matcher, which is NOT under /root/reference and whose version the
                     reference never pins (CMakeLists.txt:23 `find_package(OpenCV REQUIRED)`); there are no reference
                     tests at that boundary => parity unpinned by the reference.  We define it as EXACT brute force:
                     distances accumulated in float64 from the float32 inputs, ties -> lower train index, and cross-check
                     against OpenCV's CPU BFMatcher (the reference's own NO_OPENCV_CUDA path, FeatureManager.cpp:266-269).
  * prune_matches()  SiftManager::pruneMatches (FeatureManager.cpp:290-336)
  * collect_mutual() SiftManager::collectMutualMatches (:338-368) — a UNION, duplicates kept (SURVEY.md D1)
"""
from __future__ import annotations

import numpy as np


def _d2_direct(qrow: np.ndarray, t: np.ndarray) -> np.ndarray:
    """float64 sum of (q - t)^2 over the last axis: the distance both knn() and knn_direct() order by, computed alike."""
    diff = qrow[None, :] - t
    return (diff * diff).sum(1)


def _top_k(c: np.ndarray, dd: np.ndarray, kk: int, idx_row: np.ndarray, dist_row: np.ndarray):
    order = np.lexsort((c, dd))[:kk]
    idx_row[:kk] = c[order]
    dist_row[:kk] = np.sqrt(dd[order]).astype(np.float32)


def knn(query: np.ndarray, train: np.ndarray, k: int = 5, block: int = 512):
    """Exact kNN.  Returns (idx [nq,k] int32, dist [nq,k] float32); rows with fewer than k candidates pad with -1/inf.

    The float64 expansion |q|^2 + |t|^2 - 2 q.t only preselects: it cancels when descriptors share a large offset (|q|, |t| >> |q - t|).
    Whatever the summation order, its error is below (dim + 2) 2^-53 (|q| + |t|)^2 (norms and dot product each to dim 2^-53 of their
    magnitude, plus the two additions); `margin` is four times that for the row's largest train norm.  The k rows of smallest expanded d2
    have exact d2 <= kth + margin, so every row whose exact d2 is at most that has expanded d2 <= kth + 2 margin: those rows are
    recomputed by direct differences and ordered by (d2, index), as knn_direct() orders all of them."""
    q = np.asarray(query, np.float32)
    t = np.asarray(train, np.float32).astype(np.float64)
    nq, nt = q.shape[0], t.shape[0]
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), np.inf, np.float32)
    if nq == 0 or nt == 0:
        return idx, dist
    tn = (t * t).sum(1)
    tmax = np.sqrt(tn.max())
    kk = min(k, nt)
    for s in range(0, nq, block):
        qb = q[s:s + block].astype(np.float64)
        qn = (qb * qb).sum(1)
        d2 = qn[:, None] + tn[None, :] - 2.0 * (qb @ t.T)
        kth = np.partition(d2, kk - 1, axis=1)[:, kk - 1]
        margin = 4.0 * 2.0 ** -53 * (q.shape[1] + 2) * (np.sqrt(qn) + tmax) ** 2
        keep = d2 <= (kth + 2.0 * margin)[:, None]
        for r in range(qb.shape[0]):
            c = np.nonzero(keep[r])[0]
            _top_k(c, _d2_direct(qb[r], t[c]), kk, idx[s + r], dist[s + r])
    return idx, dist


def knn_direct(query: np.ndarray, train: np.ndarray, k: int = 5):
    """Plain brute force: direct-difference float64 d2 to every train row, top k by (d2, index).  Slow; the check on knn()."""
    q = np.asarray(query, np.float32).astype(np.float64)
    t = np.asarray(train, np.float32).astype(np.float64)
    nq, nt = q.shape[0], t.shape[0]
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), np.inf, np.float32)
    all_rows = np.arange(nt)
    for r in range(nq if nt else 0):
        _top_k(all_rows, _d2_direct(q[r], t), min(k, nt), idx[r], dist[r])
    return idx, dist


def knn_cv2(query, train, k=5):
    """OpenCV CPU brute force (the reference's NO_OPENCV_CUDA=1 path) — used as a cross-check and as the timed CPU baseline."""
    import cv2
    m = cv2.BFMatcher(cv2.NORM_L2).knnMatch(np.ascontiguousarray(query, np.float32), np.ascontiguousarray(train, np.float32), k=k)
    idx = np.full((len(m), k), -1, np.int32)
    dist = np.full((len(m), k), np.inf, np.float32)
    for r, row in enumerate(m):
        for c, dm in enumerate(row):
            idx[r, c] = dm.trainIdx
            dist[r, c] = dm.distance
    return idx, dist


# ---------------------------------------------------------------------------------------------------------------------
def ransac_pair(A, B, u3, dist_thresh):
    """Restatement of ransacMultiPairGPU for ONE pair (/root/reference/src/cuda/cuda_ransac.cu:1145-1217,1293-1302).
    A, B: [n,3] model-frame points; u3: [n_trials,3] the uniforms curand_uniform() yields after curand_init(0, trial, 0)
    (XORWOW; taken from tests/golden/curand_xorwow_seed0.npy, generated with the same curand call).
    Rigid fit = least-squares rotation (Kabsch, float64 SVD) — the reference uses an approximate fp32 SVD of the same
    3x3 matrix.  Winner = max inlier count, ties -> lowest trial id (the reference's arg-max is racy, SURVEY.md Q8).
    Returns (inlier ids ascending, best trial id, per-trial counts)."""
    A = np.asarray(A, np.float64)[:, :3]
    B = np.asarray(B, np.float64)[:, :3]
    n = A.shape[0]
    T = u3.shape[0]
    counts = np.zeros(T, np.int64)
    poses = [None] * T
    if n >= 3:
        # round half away from zero like CUDA roundf
        ids = np.floor(np.asarray(u3, np.float32) * np.float32(n - 1) + np.float32(0.5)).astype(np.int64)
        for t in range(T):
            i0, i1, i2 = ids[t]
            if i0 == i1 or i1 == i2 or i0 == i2:
                continue
            s, d = A[[i0, i1, i2]], B[[i0, i1, i2]]
            sm, dm = s.mean(0), d.mean(0)
            S = (s - sm).T @ (d - dm)                      # S[a][b] = sum src_a dst_b
            U, _, Vt = np.linalg.svd(S)
            R = Vt.T @ U.T
            if np.linalg.det(R) < 0:
                Vt[2] *= -1
                R = Vt.T @ U.T
            tt = dm - R @ sm
            poses[t] = (R, tt)
            dist = np.linalg.norm(B - (A @ R.T + tt), axis=1)
            counts[t] = int((dist <= dist_thresh).sum())
    best = int(np.argmax(counts)) if counts.max() > 0 else -1      # argmax returns the first (lowest) index on ties
    if best < 0:
        return np.zeros(0, np.int32), -1, counts
    R, tt = poses[best]
    dist = np.linalg.norm(B - (A @ R.T + tt), axis=1)
    return np.nonzero(dist <= dist_thresh)[0].astype(np.int32), best, counts


def ransac_sample_ids(u3, n):
    """The ids every trial samples from n points: roundf(u * (float)(n - 1)), the product in float32 and rounded half away from zero
    (k_ransac_model).  [n_trials, 3] int64; all zero when n < 1."""
    p = np.asarray(u3, np.float32) * np.float32(max(n - 1, 0))
    return np.floor(p.astype(np.float64) + 0.5).astype(np.int64)


def ransac_expected_good(A, B, ids, n):
    """good as k_ransac_model sets it for finite fits: n >= 3, three distinct ids, all six sample points finite."""
    A = np.asarray(A, np.float32)[:, :3]
    B = np.asarray(B, np.float32)[:, :3]
    if n < 3:
        return np.zeros(len(ids), bool)
    distinct = (ids[:, 0] != ids[:, 1]) & (ids[:, 1] != ids[:, 2]) & (ids[:, 0] != ids[:, 2])
    finite = np.isfinite(A[ids]).all((1, 2)) & np.isfinite(B[ids]).all((1, 2))
    return distinct & finite


def kabsch64(s, d):
    """Float64 least-squares rigid fit of d ~ R s + t (det R = +1) and its residual sum of squares."""
    s = np.asarray(s, np.float64)
    d = np.asarray(d, np.float64)
    sm, dm = s.mean(0), d.mean(0)
    U, _, Vt = np.linalg.svd((s - sm).T @ (d - dm))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T)) or 1.0])
    R = Vt.T @ D @ U.T
    t = dm - R @ sm
    return R, t, float(((d - (s @ R.T + t)) ** 2).sum())


# ------------------------------------------------------------------------------ exact float32 arithmetic (round to nearest even)
def f32_round(x):
    """The float32 nearest to the rational x (ties to even; overflow to +-inf; subnormals kept), as a Python float."""
    from fractions import Fraction
    if x == 0:
        return 0.0
    x = Fraction(x)
    sign, a = (-1.0, -x) if x < 0 else (1.0, x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = max(e, -126) - 23                       # the unit in the last place at a's binade
    m = a / Fraction(2) ** q
    r = m.numerator // m.denominator
    rem = m - r
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and r % 2 == 1):
        r += 1
    v = float(Fraction(r) * Fraction(2) ** q)
    if v > float(np.finfo(np.float32).max):
        return sign * float("inf")
    return sign * v


def f32_fma(a, b, c):
    from fractions import Fraction
    if not all(np.isfinite([a, b, c])):
        return float(np.float32(np.float64(a) * np.float64(b) + np.float64(c)))
    return f32_round(Fraction(a) * Fraction(b) + Fraction(c))


def f32_mul(a, b):
    return f32_fma(a, b, 0.0) if np.isfinite([a, b]).all() else float(np.float32(a) * np.float32(b))


def f32_add(a, b):
    from fractions import Fraction
    if not np.isfinite([a, b]).all():
        return float(np.float32(a) + np.float32(b))
    return f32_round(Fraction(a) + Fraction(b))


RANSAC_ORDERS = ("kernel", "plain", "plain_squares", "plain_model")


def ransac_d2_exact(P, a, b, order="kernel"):
    """One point's squared distance under the float32 pose P [3, 4] exactly as float32 code computes it.
    order="kernel": k_ransac_eval's documented order, m = fma(P2, az, fma(P0, ax, P1 * ay)) + P3, d = b - m, d2 = fma(dz, dz, fma(dx, dx,
    dy * dy)) (k_ransac_inliers is the same expression as nvcc contracts it).  Without contraction every product and sum rounds on its
    own: m = ((P0 ax + P1 ay) + P2 az) + P3 and d2 = (dx^2 + dy^2) + dz^2.  order="plain" takes both uncontracted, "plain_squares" only
    d2 and "plain_model" only m."""
    P = [[float(v) for v in row] for row in np.asarray(P, np.float32)]
    a = [float(v) for v in np.asarray(a, np.float32)[:3]]
    b = [float(v) for v in np.asarray(b, np.float32)[:3]]
    fused_m = order in ("kernel", "plain_squares")
    fused_sq = order in ("kernel", "plain_model")
    d = []
    for r in range(3):
        if fused_m:
            m = f32_add(f32_fma(P[r][2], a[2], f32_fma(P[r][0], a[0], f32_mul(P[r][1], a[1]))), P[r][3])
        else:
            m = f32_add(f32_add(f32_add(f32_mul(P[r][0], a[0]), f32_mul(P[r][1], a[1])), f32_mul(P[r][2], a[2])), P[r][3])
        d.append(f32_add(b[r], -m))
    if fused_sq:
        return f32_fma(d[2], d[2], f32_fma(d[0], d[0], f32_mul(d[1], d[1])))
    return f32_add(f32_add(f32_mul(d[0], d[0]), f32_mul(d[1], d[1])), f32_mul(d[2], d[2]))


def sqrt_le_max(th):
    """bt_common.cuh's sqrt_le_max: the largest float32 d with sqrtf(d) <= th (sqrtf correctly rounded), -1 when none, +inf for +inf."""
    th = np.float32(th)
    if not th > 0:
        return np.float32(0.0) if th == 0 else np.float32(-1.0)
    if np.isinf(th):
        return np.float32(np.inf)
    with np.errstate(over="ignore"):
        d = np.float32(th * th)
    while d > 0 and np.sqrt(d) > th:
        d = np.nextafter(d, np.float32(-np.inf))
    while np.sqrt(np.nextafter(d, np.float32(np.inf))) <= th:
        d = np.nextafter(d, np.float32(np.inf))
    return d


IN, OUT, MARGINAL = 1, 0, 2
_U = 2.0 ** -24


def ransac_classify(poses, A, B, thresh):
    """Every point under each float32 pose (poses [T, 3, 4] or one [3, 4]): IN / OUT by the kernel's decision d2 <= sqrt_le_max(thresh),
    MARGINAL when that decision depends on how the float32 expression is contracted (an order of RANSAC_ORDERS decides otherwise than
    the kernel's).  Returns (decision [T, n] bool, the kernel's, and status [T, n] IN / OUT / MARGINAL), without the T axis for one pose.

    A float64 evaluation from the float32 inputs decides every point outside a band around d2_max that bounds the float32 error: each
    coordinate of m = P a + t rounds at most 4 times and d = b - m once more, so |d_float32 - d| <= E = 8 u (sum_i |P_ri a_i| + |t_r| + |b_r|),
    and d2 moves by at most 2 |d| E + E^2 plus 4 u d2 for its own roundings (the band is twice that).  Points inside the band are evaluated
    exactly (ransac_d2_exact) in every order.  At +inf every point whose d2 is not NaN passes, overflowed or not."""
    one = np.asarray(poses).ndim == 2
    P = np.asarray(poses, np.float32).reshape(-1, 3, 4)
    d2_max = float(sqrt_le_max(thresh))
    A = np.asarray(A, np.float32)[:, :3]
    B = np.asarray(B, np.float32)[:, :3]
    P64, A64, B64 = P.astype(np.float64), A.astype(np.float64), B.astype(np.float64)
    with np.errstate(all="ignore"):
        d = B64[None] - (np.einsum("tij,nj->tni", P64[:, :, :3], A64) + P64[:, None, :, 3])
        d2 = (d * d).sum(2)
        E = 8.0 * _U * (np.einsum("tij,nj->tni", np.abs(P64[:, :, :3]), np.abs(A64)) + np.abs(P64[:, None, :, 3]) + np.abs(B64)[None]).max(2)
        band = 2.0 * (2.0 * np.sqrt(d2) * E + E * E + 4.0 * _U * d2)
        if d2_max == float("inf"):
            decision = ~np.isnan(d2)
            near = np.zeros_like(decision)
        else:
            decision = d2 <= d2_max
            near = np.isfinite(d2) & (np.abs(d2 - d2_max) <= band)
    status = np.where(decision, IN, OUT).astype(np.int8)
    for t, i in zip(*np.nonzero(near)):
        k = ransac_d2_exact(P[t], A[i], B[i], "kernel") <= d2_max
        alt = [ransac_d2_exact(P[t], A[i], B[i], o) <= d2_max for o in RANSAC_ORDERS[1:]]
        decision[t, i] = k
        status[t, i] = MARGINAL if any(x != k for x in alt) else (IN if k else OUT)
    return (decision[0], status[0]) if one else (decision, status)


def counts_from_poses(A, B, poses, good, thresh, batch=64):
    """Every trial's inlier count restated under its own float32 pose (poses [T, 3, 4], good [T]): (counts [T] int64, counts of marginal
    points [T] int64).  Trials that are not good count 0."""
    T = len(good)
    counts = np.zeros(T, np.int64)
    marg = np.zeros(T, np.int64)
    g = np.nonzero(np.asarray(good) != 0)[0]
    if len(g) == 0:
        return counts, marg
    P = np.ascontiguousarray(np.asarray(poses, np.float32)[g]).reshape(len(g), 12)
    uniq, inv = np.unique(P.view(np.uint32), axis=0, return_inverse=True)      # trials with bit-equal poses are restated once
    uc, um = np.zeros(len(uniq), np.int64), np.zeros(len(uniq), np.int64)
    for s in range(0, len(uniq), batch):
        dec, st = ransac_classify(uniq[s:s + batch].view(np.float32).reshape(-1, 3, 4), A, B, thresh)
        uc[s:s + batch] = dec.sum(1)
        um[s:s + batch] = (st == MARGINAL).sum(1)
    counts[g] = uc[inv.ravel()]
    marg[g] = um[inv.ravel()]
    return counts, marg


def ransac_winner(counts, good):
    """(max count, lowest trial among those with it) over the good trials, as the device's 64-bit key picks it; (-1, -1) without one."""
    g = np.nonzero(np.asarray(good) != 0)[0]
    if len(g) == 0:
        return -1, -1
    c = np.asarray(counts)[g]
    return int(g[np.argmax(c)]), int(c.max())


def ransac_model_f32(s, d, sweeps=8):
    """k_ransac_model's fit in float32, operation by operation (no fused multiply-adds; rsqrtf and sqrtf correctly rounded): Horn's 4x4
    profile matrix and `sweeps` cyclic Jacobi sweeps.  s, d: [3, 3] float32 samples.  Returns the [3, 4] pose or None (not finite)."""
    f = np.float32
    with np.errstate(all="ignore"):
        s = np.asarray(s, f)
        d = np.asarray(d, f)
        sm = ((s[0] + s[1]) + s[2]) / f(3)
        dm = ((d[0] + d[1]) + d[2]) / f(3)
        S = np.zeros((3, 3), f)
        for k in range(3):
            a, b = s[k] - sm, d[k] - dm
            for i in range(3):
                for j in range(3):
                    S[i, j] = f(S[i, j] + f(a[i] * b[j]))
        N = np.zeros((4, 4), f)
        N[0, 0] = (S[0, 0] + S[1, 1]) + S[2, 2]
        N[0, 1] = N[1, 0] = S[1, 2] - S[2, 1]
        N[0, 2] = N[2, 0] = S[2, 0] - S[0, 2]
        N[0, 3] = N[3, 0] = S[0, 1] - S[1, 0]
        N[1, 1] = (S[0, 0] - S[1, 1]) - S[2, 2]
        N[1, 2] = N[2, 1] = S[0, 1] + S[1, 0]
        N[1, 3] = N[3, 1] = S[2, 0] + S[0, 2]
        N[2, 2] = (-S[0, 0] + S[1, 1]) - S[2, 2]
        N[2, 3] = N[3, 2] = S[1, 2] + S[2, 1]
        N[3, 3] = (-S[0, 0] - S[1, 1]) + S[2, 2]
        V = np.eye(4, dtype=f)
        for _ in range(sweeps):
            off = f(0)
            for p in range(4):
                for r in range(p + 1, 4):
                    off = f(off + f(N[p, r] * N[p, r]))
            if off < f(1e-22):
                break
            for p in range(3):
                for r in range(p + 1, 4):
                    apq = N[p, r]
                    if abs(apq) < f(1e-30):
                        continue
                    theta = f((N[r, r] - N[p, p]) / f(f(2) * apq))
                    t = f((f(1) if theta >= 0 else f(-1)) / f(abs(theta) + np.sqrt(f(f(theta * theta) + f(1)))))
                    c = f(f(1) / np.sqrt(f(f(t * t) + f(1))))
                    sn = f(t * c)
                    for M, rows in ((N, True), (N, False), (V, True)):
                        if rows:      # columns p, r of every row
                            x, y = M[:, p].copy(), M[:, r].copy()
                            M[:, p], M[:, r] = f(c * x) - f(sn * y), f(sn * x) + f(c * y)
                        else:
                            x, y = M[p, :].copy(), M[r, :].copy()
                            M[p, :], M[r, :] = f(c * x) - f(sn * y), f(sn * x) + f(c * y)
        best = 0
        for k in range(1, 4):
            if N[k, k] > N[best, best]:
                best = k
        q = V[:, best]
        qn = f(f(1) / np.sqrt(f(f(f(q[0] * q[0]) + f(q[1] * q[1])) + f(q[2] * q[2])) + f(q[3] * q[3])))
        w, x, y, z = (f(v * qn) for v in q)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]], f)
        if not np.isfinite(R).all():
            return None
        t = (dm - R @ sm).astype(f)
    return np.concatenate([R, t[:, None]], 1).astype(f)


# ---------------------------------------------------------------------------------------------------------------------
def _cloud_point(depth, K, u, v):
    """Frame::depthToCloudAndNormals (/root/reference/src/Frame.cpp:199-233): K^-1 (u d, v d, d), zeros wherever !(d >= 0.1): below
    0.1, negative, -inf and NaN alike (to_camera in frontend.cu)."""
    fx, fy, cx, cy = [np.float32(x) for x in K]
    d = np.float32(depth[v, u])
    if not d >= np.float32(0.1):
        return np.zeros(3, np.float32)
    ifx, ify, icx, icy = np.float32(1) / fx, np.float32(1) / fy, -cx / fx, -cy / fy
    return np.array([ifx * (np.float32(u) * d) + icx * d, ify * (np.float32(v) * d) + icy * d, d], np.float32)


def _round_half_away(x):
    return int(np.floor(abs(float(x)) + 0.5) * (1 if x >= 0 else -1))


def prune_matches(Q, T, knn_idx, K, max_dist, cos_max):
    """SiftManager::pruneMatches (/root/reference/src/FeatureManager.cpp:290-336) for one direction.
    Q, T: dicts with kpts [n,2], depth [H,W], normal [H,W,4], pose [4,4].  Returns list of (q, t, ptQ_cam, ptT_cam)."""
    H, W = Q["depth"].shape
    out = []
    Rq, tq = Q["pose"][:3, :3].astype(np.float32), Q["pose"][:3, 3].astype(np.float32)
    Rt, tt = T["pose"][:3, :3].astype(np.float32), T["pose"][:3, 3].astype(np.float32)
    for q in range(len(Q["kpts"])):
        for t in knn_idx[q]:
            if t < 0:
                continue
            uq, vq = _round_half_away(Q["kpts"][q, 0]), _round_half_away(Q["kpts"][q, 1])
            ut, vt = _round_half_away(T["kpts"][t, 0]), _round_half_away(T["kpts"][t, 1])
            if not (0 <= uq < W and 0 <= vq < H and 0 <= ut < W and 0 <= vt < H):
                continue
            pq, pt = _cloud_point(Q["depth"], K, uq, vq), _cloud_point(T["depth"], K, ut, vt)
            if pq[2] < 0.1 or pt[2] < 0.1:
                continue
            mq, mt = Rq @ pq + tq, Rt @ pt + tt
            nq, nt = Rq @ Q["normal"][vq, uq, :3], Rt @ T["normal"][vt, ut, :3]
            dist = np.float32(np.linalg.norm((mq - mt).astype(np.float32)))
            with np.errstate(invalid="ignore", divide="ignore"):
                dotn = np.float32(np.dot(nq / np.float32(np.linalg.norm(nq)), nt / np.float32(np.linalg.norm(nt))))
            if dist > max_dist or dotn < cos_max:      # NaN dot (zero normal) does NOT reject (FeatureManager.cpp:326)
                continue
            out.append((q, int(t), pq, pt))
            break
    return out


# ---------------------------------------------------------------------------------------------------------------------
GATE_FAIL, GATE_PASS, GATE_MARGINAL = "fail", "pass", "marginal"
# A zero normal normalises to NaN (Eigen 3.2's normalized()), the dot is NaN and `dot < cos_max` is false: the candidate is kept.  Eigen
# 3.3 returns the zero vector instead (dot 0, rejected whenever cos_max > 0); which one the reference ran is open (DESIGN.md §3.2).
ZERO_NORMAL_KEEPS = True
_U = 2.0 ** -24


def _gamma(n):
    return n * _U / (1.0 - n * _U)


class _Exact:
    """Float64 arithmetic that records whether every step was exact in float32 too: every result a float32 value and every float64
    operation exact (TwoSum for additions; a product of two float32 values always is; sqrt and division checked by multiplying back).
    When it stays exact, the kernel's float32 values - fused or not - equal these."""

    def __init__(self):
        self.ok = True

    def _rep(self, x):
        if np.isfinite(x) and float(np.float32(x)) != x:
            self.ok = False
        return x

    def mul(self, a, b):
        return self._rep(a * b)

    def add(self, a, b):
        s = a + b
        bb = s - a
        if np.isfinite(s) and (a - (s - bb)) + (b - bb) != 0.0:
            self.ok = False
        return self._rep(s)

    def sqrt(self, s):
        r = float(np.sqrt(s))
        if r * r != s:
            self.ok = False
        return self._rep(r)

    def div(self, a, b):
        q = a / b
        if q * b != a:
            self.ok = False
        return self._rep(q)


def gate_pixels(Q, T, q, t):
    """std::round (half away from zero) of both keypoints and Utils::isPixelInsideImage on both frames: (uq, vq, ut, vt) or None."""
    H, W = Q["depth"].shape
    uq, vq = _round_half_away(Q["kpts"][q, 0]), _round_half_away(Q["kpts"][q, 1])
    ut, vt = _round_half_away(T["kpts"][t, 0]), _round_half_away(T["kpts"][t, 1])
    if not (0 <= uq < W and 0 <= vq < H and 0 <= ut < W and 0 <= vt < H):
        return None
    return uq, vq, ut, vt


def prune_gate64(Q, T, q, t, K, max_dist, cos_max):
    """One candidate of SiftManager::pruneMatches (FeatureManager.cpp:290-336) in float64 with a float32 error bound.
    Returns (GATE_PASS / GATE_FAIL / GATE_MARGINAL, ptQ_cam, ptT_cam as float32, detail dict).

    Rounding, the in-image test and the depth test (!(d >= 0.1) rejects, NaN included) are exact decisions.  The rest is evaluated in
    float64 in the kernel's operation order from the kernel's float32 inputs (ifx = 1/fx, icx = -cx/fx rounded to float32, the float32
    pose, depth and normals).  When every step is exact in float32 as well (_Exact: dyadic geometry) the decision is exact; otherwise
    a test within its bound E of the threshold is MARGINAL: the float32 kernel may decide it either way.

    Bounds (u = 2^-24; a float32 operation, fused or not, rounds once; n roundings on a term stay within gamma_n = n u / (1 - n u)):
      cloud point  x = ifx (u d) + icx d: at most 3 roundings per term, |dx| <= gamma_3 a_x with a_x = |ifx u d| + |icx d|; z = d exact.
      model point  m_r = ((T_r0 x + T_r1 y) + T_r2 z) + T_r3: at most 4 roundings per term on top of the inputs' errors, so
                   |dm_r| <= gamma_8 M_r with M_r = sum_i |T_ri| (|p_i| + a_i) + |T_r3|.
      difference   |dd_r| <= |dmQ_r| + |dmT_r| + u |d_r|.
      distance     sqrt((d0^2 + d1^2) + d2^2) is 1-Lipschitz in d (moves by <= sum_r |dd_r|); its own 3 squares, 2 additions and the sqrt
                   add at most gamma_4 dist.   E_dist = sum_r (gamma_8 (MQ_r + MT_r) + u |d_r|) + gamma_4 dist.
      normals      w_r = (T_r0 n_x + T_r1 n_y) + T_r2 n_z: |dw_r| <= gamma_3 N_r, N_r = sum_i |T_ri| |n_i|.  w / |w| moves by at most
                   2 |dw|_2 / |w|; the norm (3 squares, 2 adds, sqrt) and the division add gamma_5 per unit component; the dot's 3 products
                   and 2 additions add gamma_3 (its terms sum to <= 1 in magnitude).
                   E_dot = 2 gamma_3 (|N_q|_2 / l_q + |N_t|_2 / l_t) + 2 gamma_5 + gamma_3.
    Both bounds are doubled for the second-order terms and the float64 evaluation itself."""
    H, W = Q["depth"].shape
    px = gate_pixels(Q, T, q, t)
    z3 = np.zeros(3, np.float32)
    if px is None:
        return GATE_FAIL, z3, z3, {"why": "outside"}
    uq, vq, ut, vt = px
    dq, dt = np.float32(Q["depth"][vq, uq]), np.float32(T["depth"][vt, ut])
    if not (dq >= np.float32(0.1) and dt >= np.float32(0.1)):
        return GATE_FAIL, z3, z3, {"why": "depth"}
    pq, pt = _cloud_point(Q["depth"], K, uq, vq), _cloud_point(T["depth"], K, ut, vt)
    fx, fy, cx, cy = [np.float32(x) for x in K]
    ifx, ify, icx, icy = (float(v) for v in (np.float32(1) / fx, np.float32(1) / fy, -cx / fx, -cy / fy))
    ex, exn = _Exact(), _Exact()          # the distance's chain and the normals' chain, each exact or bounded on its own
    out = {}
    for side, (fr, u, v, d) in (("q", (Q, uq, vq, float(dq))), ("t", (T, ut, vt, float(dt)))):
        P = np.asarray(fr["pose"], np.float32).astype(np.float64)
        p = [ex.add(ex.mul(ifx, ex.mul(float(u), d)), ex.mul(icx, d)), ex.add(ex.mul(ify, ex.mul(float(v), d)), ex.mul(icy, d)), d]
        a = [abs(ifx * u * d) + abs(icx * d), abs(ify * v * d) + abs(icy * d), 0.0]
        n = [float(x) for x in np.asarray(fr["normal"][v, u, :3], np.float32)]
        m, M, w, N = [], [], [], []
        for r in range(3):
            m.append(ex.add(ex.add(ex.add(ex.mul(P[r, 0], p[0]), ex.mul(P[r, 1], p[1])), ex.mul(P[r, 2], p[2])), P[r, 3]))
            M.append(sum(abs(P[r, i]) * (abs(p[i]) + a[i]) for i in range(3)) + abs(P[r, 3]))
            w.append(exn.add(exn.add(exn.mul(P[r, 0], n[0]), exn.mul(P[r, 1], n[1])), exn.mul(P[r, 2], n[2])))
            N.append(sum(abs(P[r, i]) * abs(n[i]) for i in range(3)))
        out[side] = (m, M, w, N)
    (mQ, MQ, wq, NQ), (mT, MT, wt, NT) = out["q"], out["t"]
    dd = [ex.add(mQ[r], -mT[r]) for r in range(3)]
    dist = ex.sqrt(ex.add(ex.add(ex.mul(dd[0], dd[0]), ex.mul(dd[1], dd[1])), ex.mul(dd[2], dd[2])))
    e_dist = 2.0 * (sum(_gamma(8) * (MQ[r] + MT[r]) + _U * abs(dd[r]) for r in range(3)) + _gamma(4) * dist)
    lq = exn.sqrt(exn.add(exn.add(exn.mul(wq[0], wq[0]), exn.mul(wq[1], wq[1])), exn.mul(wq[2], wq[2])))
    lt = exn.sqrt(exn.add(exn.add(exn.mul(wt[0], wt[0]), exn.mul(wt[1], wt[1])), exn.mul(wt[2], wt[2])))
    zero_normal = lq == 0.0 or lt == 0.0
    if zero_normal:
        dot, e_dot = float("nan"), 0.0
    else:
        uq3, ut3 = [exn.div(x, lq) for x in wq], [exn.div(x, lt) for x in wt]
        dot = exn.add(exn.add(exn.mul(uq3[0], ut3[0]), exn.mul(uq3[1], ut3[1])), exn.mul(uq3[2], ut3[2]))
        e_dot = 2.0 * (2.0 * _gamma(3) * (np.linalg.norm(NQ) / lq + np.linalg.norm(NT) / lt) + 2.0 * _gamma(5) + _gamma(3))
    if ex.ok:
        e_dist = 0.0
    if exn.ok:
        e_dot = 0.0
    md, cm = float(np.float32(max_dist)), float(np.float32(cos_max))
    detail = {"dist": dist, "e_dist": e_dist, "dot": dot, "e_dot": e_dot, "exact": ex.ok and exn.ok, "zero_normal": zero_normal}
    if zero_normal and not ZERO_NORMAL_KEEPS:
        return GATE_FAIL, pq, pt, detail
    if dist > md + e_dist or (not zero_normal and dot < cm - e_dot):
        return GATE_FAIL, pq, pt, detail
    if dist > md - e_dist or (not zero_normal and dot < cm + e_dot):
        return GATE_MARGINAL, pq, pt, detail
    return GATE_PASS, pq, pt, detail


def prune_options(Q, T, knn_idx, K, max_dist, cos_max):
    """pruneMatches for one direction under prune_gate64: for every query, in order, the outcomes the kernel may produce - the train
    index it keeps, or None - each with its (ptQ, ptT).  A query has one outcome unless a marginal candidate comes before the first
    passing one.  Returns (options [per query: list of (t or None, ptQ, ptT)], marginals [(q, t, detail)])."""
    nT = len(T["kpts"])
    options, marginals = [], []
    for q in range(len(Q["kpts"])):
        opts = []
        decided = False
        for t in knn_idx[q]:
            t = int(t)
            if t < 0 or t >= nT:
                continue
            verdict, pq, pt, detail = prune_gate64(Q, T, q, t, K, max_dist, cos_max)
            if verdict == GATE_FAIL:
                continue
            opts.append((t, pq, pt))
            if verdict == GATE_PASS:
                decided = True
                break
            marginals.append((q, t, detail))
        if not decided:
            opts.append((None, None, None))
        options.append(opts)
    return options, marginals


def _mutual_row(A, B, q, t, pq, pt, direction):
    if direction == 0:
        return np.concatenate([A["kpts"][q], B["kpts"][t], pq, pt]).astype(np.float32)
    return np.concatenate([A["kpts"][t], B["kpts"][q], pt, pq]).astype(np.float32)


def mutual_rows_resolved(A, B, optAB, optBA, got=None, ulps=0):
    """collectMutualMatches' rows under prune_options' outcomes (A->B block, then B->A).  A query with several possible outcomes takes the
    one whose row is `got`'s next row (uv bit-equal, points within `ulps` float32 ulps), else its no-match outcome if it has one.
    Returns (rows [m,10] float32, n_ambiguous_queries)."""
    rows, amb = [], 0
    for direction, opts_all in ((0, optAB), (1, optBA)):
        for q, opts in enumerate(opts_all):
            if len(opts) > 1:
                amb += 1
            pick = opts[-1] if len(opts) == 1 else None
            if pick is None:
                nxt = got[len(rows)] if got is not None and len(rows) < len(got) else None
                pick = opts[-1]
                for o in opts:
                    if o[0] is not None and nxt is not None and rows_match(_mutual_row(A, B, q, o[0], o[1], o[2], direction)[None], nxt[None], ulps):
                        pick = o
                        break
            if pick[0] is not None:
                rows.append(_mutual_row(A, B, q, pick[0], pick[1], pick[2], direction))
    return np.asarray(rows, np.float32).reshape(-1, 10), amb


def rows_match(a, b, ulps=0):
    """(uA, vA, uB, vB) bit-equal and the six point coordinates within `ulps` float32 ulps (0: bit-equal)."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 10)
    b = np.ascontiguousarray(b, np.float32).reshape(-1, 10)
    if a.shape != b.shape:
        return False
    if not np.array_equal(a[:, :4].view(np.uint32), b[:, :4].view(np.uint32)):
        return False
    return bool((ulp_distance(a[:, 4:], b[:, 4:]) <= ulps).all())


def ulp_distance(a, b):
    """|a - b| in float32 ulps along the ordered integer line (+0 and -0 are 0 apart); NaN against anything is far."""
    def key(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    d = np.abs(key(a) - key(b))
    return np.where(np.isnan(a) | np.isnan(b), np.int64(1) << 40, d)


def emit_plan(n_inliers, neighbor, capacity):
    """k_emit_entryj's contract for one call, from each pair's RANSAC inlier count: a pair with fewer than 5 is cleared
    (FeatureManager.cpp:233-241); the pairs are written back to back and cut at `capacity`; the status is the match outcome, not the
    cut's: OK when >= 5 inliers, else FAIL for a neighbour pair (Frame::FAIL, :282-286) and EMPTY otherwise.
    Returns (n_entry, entry_off, total, status) with status 0 / 1 / 2 = BT_PAIR_OK / BT_PAIR_EMPTY / BT_PAIR_FAIL."""
    kept = np.where(np.asarray(n_inliers, np.int64) >= 5, np.asarray(n_inliers, np.int64), 0)
    off = np.concatenate([[0], np.cumsum(kept)[:-1]]).astype(np.int64)
    off_c = np.minimum(off, capacity)
    n_c = np.minimum(off + kept, capacity) - off_c
    status = np.where(kept > 0, 0, np.where(np.asarray(neighbor, bool), 2, 1))
    return n_c.astype(np.int32), off_c.astype(np.int32), int(min(kept.sum(), capacity)), status.astype(np.int32)


def collect_mutual(A, B, mAB, mBA):
    """SiftManager::collectMutualMatches (:338-368): A->B survivors then B->A survivors, duplicates kept.
    Rows: [uA, vA, uB, vB, ptA_cam(3), ptB_cam(3)]."""
    rows = []
    for (q, t, pq, pt) in mAB:
        rows.append(np.concatenate([A["kpts"][q], B["kpts"][t], pq, pt]))
    for (q, t, pq, pt) in mBA:
        rows.append(np.concatenate([A["kpts"][t], B["kpts"][q], pt, pq]))
    return np.asarray(rows, np.float32).reshape(-1, 10)


def find_corres(A, B, K, prune, u3, ransac_inlier_dist, k=5, propagated=None):
    """findCorresbyNN [+ findCorresByMapPoints for a non-neighbour pair] + runRansacBetween for one pair (A newer).
    prune = (max_dist_nn, cos_nn, max_dist_n, cos_n).  propagated: [m,4] (uA,vA,uB,vB) of the map points both frames observe, in
    the order SiftManager::findCorresByMapPoints walks them (/root/reference/src/FeatureManager.cpp:489-520): appended unless an
    existing match has the same (uA,vA) or (uB,vB), with the organised-cloud points at round(u), round(v).
    Returns (mutual rows incl. the appended ones, inlier row ids or None if the pair was dropped)."""
    iAB, _ = knn(A["desc"], B["desc"], k)
    iBA, _ = knn(B["desc"], A["desc"], k)
    neighbor = abs(A["id"] - B["id"]) == 1
    max_dist, cos_max = (prune[2], prune[3]) if neighbor else (prune[0], prune[1])
    rows = collect_mutual(A, B, prune_matches(A, B, iAB, K, max_dist, cos_max), prune_matches(B, A, iBA, K, max_dist, cos_max))
    if propagated is not None and not neighbor and len(propagated):
        H, W = A["depth"].shape
        extra = []
        for uA, vA, uB, vB in np.asarray(propagated, np.float32):
            if len(rows) and (((rows[:, 0] == uA) & (rows[:, 1] == vA)) | ((rows[:, 2] == uB) & (rows[:, 3] == vB))).any():
                continue
            ua, va, ub, vb = _round_half_away(uA), _round_half_away(vA), _round_half_away(uB), _round_half_away(vB)
            pa = _cloud_point(A["depth"], K, ua, va) if (0 <= ua < W and 0 <= va < H) else np.zeros(3, np.float32)
            pb = _cloud_point(B["depth"], K, ub, vb) if (0 <= ub < W and 0 <= vb < H) else np.zeros(3, np.float32)
            extra.append(np.concatenate([[uA, vA, uB, vB], pa, pb]).astype(np.float32))
        if extra:
            rows = np.concatenate([rows.reshape(-1, 10), np.asarray(extra, np.float32)], 0)
    if len(rows) <= 5:
        return rows, None
    PA = rows[:, 4:7] @ A["pose"][:3, :3].T.astype(np.float32) + A["pose"][:3, 3].astype(np.float32)
    PB = rows[:, 7:10] @ B["pose"][:3, :3].T.astype(np.float32) + B["pose"][:3, 3].astype(np.float32)
    ids, best, counts = ransac_pair(PA, PB, u3, ransac_inlier_dist)
    if len(ids) < 5:
        return rows, None
    return rows, ids
